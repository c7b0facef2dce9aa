// A bounded neighbour for tests/test_gpu_shared_device.py: it takes whole SMs away from the library for a fixed time,
// as another job on a shared GPU does.
//
// hold_sms(G, hold_us, wait_ms, &resident) launches G CTAs of one thread on the holder's own non-blocking stream, each
// with the largest dynamic shared memory a CTA may have, so no other CTA that uses shared memory fits on its SM.  Each
// CTA counts itself into a mapped pinned counter and then sleeps on %globaltimer until hold_us microseconds (at most
// 1 s) after its own start, and exits: the holder never waits on anything but the clock, so it always ends by itself.
// The host waits, bounded by wait_ms, until all G CTAs have reported; *resident receives how many did.  A new hold first
// waits for the previous one to end.  hold_end() waits for the last hold to end.
#include <cuda_runtime.h>
#include <stdint.h>

#include <chrono>
#include <thread>

namespace {

constexpr unsigned kMaxHoldUs = 1000000;

__device__ __forceinline__ uint64_t globaltimer_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void hold_kernel(unsigned* running, uint64_t hold_ns)
{
    extern __shared__ unsigned char smem[];
    const uint64_t start = globaltimer_ns();
    smem[0] = 1;
    atomicAdd_system(running, 1u);
    __threadfence_system();
    while (globaltimer_ns() - start < hold_ns) __nanosleep(20000);
}

cudaStream_t g_stream = nullptr;
unsigned* g_host = nullptr;       // mapped pinned counter
unsigned* g_dev = nullptr;
int g_smem = 0;

int init()
{
    if (g_stream) return 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&g_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(hold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_smem);
    if (e == cudaSuccess) e = cudaHostAlloc(reinterpret_cast<void**>(&g_host), sizeof(unsigned), cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&g_dev), g_host, 0);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking);
    return static_cast<int>(e);
}

}  // namespace

// the dynamic shared memory of one holder CTA (bytes), or a negative CUDA error
extern "C" int hold_smem_bytes(void)
{
    const int e = init();
    return e ? -e : g_smem;
}

extern "C" int hold_sms(int ctas, unsigned hold_us, unsigned wait_ms, int* resident)
{
    int e = init();
    if (e) return e;
    if (ctas <= 0 || hold_us == 0 || hold_us > kMaxHoldUs || !resident) return static_cast<int>(cudaErrorInvalidValue);
    e = static_cast<int>(cudaStreamSynchronize(g_stream));       // the previous hold has ended
    if (e) return e;
    *reinterpret_cast<volatile unsigned*>(g_host) = 0;
    hold_kernel<<<ctas, 1, g_smem, g_stream>>>(g_dev, static_cast<uint64_t>(hold_us) * 1000u);
    e = static_cast<int>(cudaGetLastError());
    if (e) return e;
    const volatile unsigned* seen = g_host;
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(wait_ms);
    while (*seen < static_cast<unsigned>(ctas) && std::chrono::steady_clock::now() < deadline)
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    *resident = static_cast<int>(*seen);
    return 0;
}

extern "C" int hold_end(void)
{
    return g_stream ? static_cast<int>(cudaStreamSynchronize(g_stream)) : 0;
}

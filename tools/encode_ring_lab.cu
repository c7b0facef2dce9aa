// encode_ring_lab.cu -- timing bench for the fused word encoder with its streams in a shared-memory ring (K2r,
// word_kernels.cuh) at several shapes {ring bytes, warps, prefetch distance D}, on 1 GiB of uniform bytes:
//   ring_place:   K2r with placement; its blob and directory are checked against K2f's byte for byte, and the ring
//                 waits (a pending stream placed before its offset was seen ready) are counted per chunk;
//   ring_noplace: the step alone: every warp encodes its chunks into its ring and only records their sizes (checked
//                 against K2's), so the output is not a container.
// Against them, in the same process on the same data: the split word encoder (K2, encode into global slots, no
// compaction) and the shipped fused encoder (K2f, with placement).  One JSON line per variant on stdout.  Not part of
// the product.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Iinclude -Iryg_rans_b200/csrc \
//        -o build/encode_ring_lab tools/encode_ring_lab.cu
//   build/encode_ring_lab [--n BYTES] [--chunk SYMS] [--reps K]
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "word_kernels.cuh"

using namespace rb200;

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            std::exit(2);                                                                          \
        }                                                                                          \
    } while (0)

__device__ __forceinline__ uint32_t mix32(uint64_t v)
{
    v ^= v >> 33; v *= 0xff51afd7ed558ccdull; v ^= v >> 33; v *= 0xc4ceb9fe1a85ec53ull; v ^= v >> 33;
    return static_cast<uint32_t>(v);
}
__global__ void gen_uniform_kernel(uint8_t* out, uint64_t n, uint64_t seed)
{
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) out[i] = mix32(i + seed) >> 24;
}

struct NoSpace {
    __device__ __forceinline__ void reserve(uint32_t, uint32_t) {}
};

template <uint32_t RING, uint32_t W, uint32_t D>
__global__ void __launch_bounds__(W * 32, 1)
ring_step_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, const WordEncEntry* __restrict__ g_table,
                 uint32_t* __restrict__ counter, uint32_t* __restrict__ sizes, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];     // [32 KiB table][W rings][W stages]
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<true>(g_table[i / kEncReplicas]);
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tab = smem_addr(s_enc);
    const uint32_t ring = tab + kEncTableBytes + warp * RING, stage = tab + kEncTableBytes + W * RING + warp * kEncStageBytes;
    NoSpace space;
    uint32_t top = 0;
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(counter, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= n_chunks) break;
        const ChunkRange r = chunk_range(chunk, chunk_syms, n);
        const uint32_t produced = word_encode_stream_ring<true, RING, D>(in + r.first, r.m, tab, stage, ring, top, space, status);
        if (lane == 0) sizes[chunk] = produced;
        const uint32_t t = top - ((produced + 15u) & ~15u);
        top = min(t, t + RING);
    }
}

// K2r with placement at a given shape; adds up the warps' ring waits in *waits
template <uint32_t RING, uint32_t W, uint32_t D>
__global__ void __launch_bounds__(W * 32, 1)
ring_place_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, const WordEncEntry* __restrict__ g_table,
                  uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap,
                  uint64_t* __restrict__ offsets, uint32_t* __restrict__ status, unsigned long long* __restrict__ waits)
{
    const uint32_t w = word_encode_ring<true, RING, W, D>(in, n, chunk_syms, g_table, PlaceOut{look, n_chunks, blob, blob_cap, offsets, status},
                                                          counter);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(waits, static_cast<unsigned long long>(w));
}

struct Ctx {
    const uint8_t* in; uint64_t n; uint32_t chunk, n_chunks; const WordEncEntry* table; uint32_t* counter; uint32_t* sizes;
    uint32_t* ref_sizes; uint32_t* status; uint8_t* scratch; uint32_t slot; uint64_t* look; uint8_t* blob; uint64_t* offsets; int sms; int reps;
    uint8_t* ref_blob; uint64_t* ref_offsets; unsigned long long* waits;
};

template <class F>
double time_ms(const Ctx& c, F&& launch, bool zero_counter)
{
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    float total = 0;
    for (int r = -2; r < c.reps; r++) {
        if (zero_counter) {
            CK(cudaMemset(c.counter, 0, 16));
            CK(cudaMemset(c.look, 0, c.n_chunks * sizeof(uint64_t)));
        }
        CK(cudaEventRecord(a));
        launch();
        CK(cudaEventRecord(b));
        CK(cudaEventSynchronize(b));
        CK(cudaGetLastError());
        float ms;
        CK(cudaEventElapsedTime(&ms, a, b));
        if (r >= 0) total += ms;
    }
    CK(cudaEventDestroy(a));
    CK(cudaEventDestroy(b));
    return total / c.reps;
}

template <uint32_t RING, uint32_t W, uint32_t D>
void run_ring(const Ctx& c)
{
    const uint32_t smem = kEncTableBytes + W * (RING + kEncStageBytes);
    auto k = ring_step_kernel<RING, W, D>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CK(cudaMemset(c.sizes, 0, c.n_chunks * 4));
    const double ms = time_ms(c, [&] { k<<<c.sms, W * 32, smem>>>(c.in, c.n, c.chunk, c.n_chunks, c.table, c.counter, c.sizes, c.status); }, true);
    std::vector<uint32_t> got(c.n_chunks), want(c.n_chunks);
    CK(cudaMemcpy(got.data(), c.sizes, c.n_chunks * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(want.data(), c.ref_sizes, c.n_chunks * 4, cudaMemcpyDeviceToHost));
    const bool ok = std::memcmp(got.data(), want.data(), c.n_chunks * 4) == 0;
    std::printf("{\"variant\": \"ring_noplace\", \"ring\": %u, \"warps\": %u, \"D\": %u, \"ms\": %.4f, \"sizes_match_k2\": %s}\n", RING, W, D, ms,
                ok ? "true" : "false");
    std::fflush(stdout);
}

// the blob and directory of K2r against K2f's
bool same_container(const Ctx& c)
{
    std::vector<uint64_t> o(c.n_chunks + 1), ro(c.n_chunks + 1);
    CK(cudaMemcpy(o.data(), c.offsets, o.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ro.data(), c.ref_offsets, ro.size() * 8, cudaMemcpyDeviceToHost));
    if (o != ro) return false;
    std::vector<uint8_t> b(o.back()), rb(o.back());
    CK(cudaMemcpy(b.data(), c.blob, b.size(), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rb.data(), c.ref_blob, rb.size(), cudaMemcpyDeviceToHost));
    return b == rb;
}

template <uint32_t RING, uint32_t W, uint32_t D>
void run_place(const Ctx& c)
{
    const uint32_t smem = kEncTableBytes + W * (RING + kEncStageBytes);
    auto k = ring_place_kernel<RING, W, D>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CK(cudaMemset(c.blob, 0, 2 * c.n));
    CK(cudaMemset(c.offsets, 0, (c.n_chunks + 1) * 8ull));
    CK(cudaMemset(c.waits, 0, 8));
    const double ms = time_ms(c, [&] {
        k<<<c.sms, W * 32, smem>>>(c.in, c.n, c.chunk, c.n_chunks, c.table, c.look, c.counter, c.blob, 2 * c.n, c.offsets, c.status, c.waits);
    }, true);
    unsigned long long waits = 0;
    CK(cudaMemcpy(&waits, c.waits, 8, cudaMemcpyDeviceToHost));
    const bool ok = same_container(c);
    std::printf("{\"variant\": \"ring_place\", \"ring\": %u, \"warps\": %u, \"D\": %u, \"ms\": %.4f, \"waits_per_chunk\": %.4f, "
                "\"same_as_k2f\": %s}\n", RING, W, D, ms, static_cast<double>(waits) / (c.reps + 2) / c.n_chunks, ok ? "true" : "false");
    std::fflush(stdout);
}

int main(int argc, char** argv)
{
    uint64_t n = 1ull << 30;
    uint32_t chunk = 8192;
    int reps = 10;
    for (int i = 1; i + 1 < argc; i += 2) {
        if (!std::strcmp(argv[i], "--n")) n = std::strtoull(argv[i + 1], nullptr, 0);
        else if (!std::strcmp(argv[i], "--chunk")) chunk = static_cast<uint32_t>(std::strtoul(argv[i + 1], nullptr, 0));
        else if (!std::strcmp(argv[i], "--reps")) reps = std::atoi(argv[i + 1]);
    }
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    std::printf("{\"device\": \"%s\", \"sms\": %d, \"n\": %llu, \"chunk\": %u, \"reps\": %d}\n", prop.name, sms,
                static_cast<unsigned long long>(n), chunk, reps);

    // uniform model: every byte has frequency 4096 / 256
    std::vector<WordEncEntry> tab(256);
    int exact = 1;
    for (uint32_t s = 0; s < 256; s++) tab[s] = word_enc32_entry(16, s * 16, &exact);

    Ctx c = {};
    c.n = n; c.chunk = chunk; c.n_chunks = static_cast<uint32_t>((n + chunk - 1) / chunk); c.sms = sms; c.reps = reps;
    c.slot = static_cast<uint32_t>((512 + 2ull * chunk + 15) & ~15ull);
    uint8_t* d_in;
    WordEncEntry* d_tab;
    CK(cudaMalloc(&d_in, n + 16));
    CK(cudaMalloc(&d_tab, 256 * sizeof(WordEncEntry)));
    CK(cudaMemcpy(d_tab, tab.data(), 256 * sizeof(WordEncEntry), cudaMemcpyHostToDevice));
    gen_uniform_kernel<<<sms * 8, 256>>>(d_in, n, 12345);
    CK(cudaGetLastError());
    c.in = d_in; c.table = d_tab;
    CK(cudaMalloc(&c.counter, 16));
    CK(cudaMalloc(&c.sizes, c.n_chunks * 4ull));
    CK(cudaMalloc(&c.ref_sizes, c.n_chunks * 4ull));
    CK(cudaMalloc(&c.status, 4));
    CK(cudaMemset(c.status, 0, 4));
    CK(cudaMalloc(&c.scratch, (static_cast<uint64_t>(c.n_chunks) + 1) * c.slot));
    CK(cudaMalloc(&c.look, c.n_chunks * 8ull));
    CK(cudaMalloc(&c.blob, n * 2));
    CK(cudaMalloc(&c.offsets, (c.n_chunks + 1) * 8ull));
    CK(cudaMalloc(&c.ref_blob, n * 2));
    CK(cudaMalloc(&c.ref_offsets, (c.n_chunks + 1) * 8ull));
    CK(cudaMalloc(&c.waits, 8));

    // K2, the split encoder: encode into global slots, no compaction
    configure_word_kernels();
    {
        const double ms = time_ms(c, [&] {
            word_encode_kernel<true><<<(c.n_chunks + kEncWarps - 1) / kEncWarps, kEncWarps * 32, kEncSmemBytes>>>(
                c.in, c.n, c.chunk, c.n_chunks, c.table, c.scratch, c.slot, c.ref_sizes, c.status);
        }, false);
        std::printf("{\"variant\": \"k2_split_encode\", \"ms\": %.4f}\n", ms);
    }
    // K2f as shipped (2 CTAs x 16 warps per SM, two scratch slots per warp), with placement
    {
        const uint32_t grid = sms * RB200_FUSED_MINBLOCKS;
        const double ms = time_ms(c, [&] {
            word_encode_fused_kernel<true><<<grid, kEncWarps * 32, kEncSmemBytes>>>(c.in, c.n, c.chunk, c.n_chunks, c.table, c.scratch, c.slot,
                                                                                    c.look, c.counter, c.blob, 2 * n, c.offsets, c.status);
        }, true);
        std::printf("{\"variant\": \"k2f_fused_shipped\", \"ms\": %.4f}\n", ms);
        CK(cudaMemcpy(c.ref_blob, c.blob, 2 * n, cudaMemcpyDeviceToDevice));
        CK(cudaMemcpy(c.ref_offsets, c.offsets, (c.n_chunks + 1) * 8ull, cudaMemcpyDeviceToDevice));
    }
    run_place<12800, 15, 1>(c);
    run_place<12800, 15, 2>(c);
    run_place<13312, 14, 1>(c);
    run_place<14336, 13, 2>(c);
    run_place<16384, 11, 4>(c);
    run_ring<16384, 11, 1>(c);
    run_ring<16384, 11, 2>(c);
    run_ring<16384, 11, 4>(c);
    run_ring<14336, 13, 2>(c);
    run_ring<14336, 13, 4>(c);
    run_ring<13312, 14, 1>(c);
    run_ring<13312, 14, 2>(c);
    run_ring<13312, 14, 4>(c);
    run_ring<12800, 15, 1>(c);
    run_ring<12800, 15, 2>(c);
    run_ring<12800, 15, 4>(c);
    uint32_t st = 0;
    CK(cudaMemcpy(&st, c.status, 4, cudaMemcpyDeviceToHost));
    std::printf("{\"status\": %u}\n", st);
    return 0;
}

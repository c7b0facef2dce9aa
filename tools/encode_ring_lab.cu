// encode_ring_lab.cu -- timing bench for the fused word encoder with its streams in a shared-memory ring (K2r,
// word_kernels.cuh) at several shapes {ring bytes, warps, prefetch distance D}, on 1 GiB of uniform bytes or of bytes
// drawn from a histogram (--hist tests/golden/book1_hist.json: text-like):
//   ring_place:   K2r with placement; its blob and directory are checked against K2f's byte for byte.  Per chunk: the
//                 ring waits (a placement that waited for its offset), the pending streams spilled whole to the spill
//                 slot (pieces of at most spill_pending bytes), and the bytes spilled.  spill_pending 0: a pending
//                 stream waits for its offset instead;
//   ring_noplace: the step alone: every warp encodes its chunks into its ring and only records their sizes (checked
//                 against K2's), so the output is not a container.
// Against them, in the same process on the same data: the split word encoder (K2, encode into global slots, no
// compaction) and the shipped fused encoder (K2f, with placement).  One JSON line per variant on stdout.  Not part of
// the product.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Iinclude -Iryg_rans_b200/csrc \
//        -o build/encode_ring_lab tools/encode_ring_lab.cu
//   build/encode_ring_lab [--n BYTES] [--chunk SYMS] [--reps K] [--hist FILE]
#include <cuda_runtime.h>

#include <algorithm>
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
// byte i = slot_sym[a 12-bit hash of i]: symbols drawn from the model's own distribution
__global__ void gen_kernel(uint8_t* out, uint64_t n, uint64_t seed, const uint8_t* __restrict__ slot_sym)
{
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) out[i] = slot_sym[mix32(i + seed) >> 20];
}

struct NoSpace {
    __device__ __forceinline__ void reserve(uint32_t, uint32_t) {}
    __device__ __forceinline__ uint32_t emitted(uint32_t e) const { return e; }
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

// K2r with placement at a given shape; adds up the warps' RingStats in stats[0..2]
template <uint32_t RING, uint32_t W, uint32_t D, uint32_t SP>
__global__ void __launch_bounds__(W * 32, 1)
ring_place_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, const WordEncEntry* __restrict__ g_table,
                  uint8_t* __restrict__ spill, uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob,
                  uint64_t blob_cap, uint64_t* __restrict__ offsets, uint32_t* __restrict__ status, unsigned long long* __restrict__ stats)
{
    const RingStats s = word_encode_ring<true, RING, W, D, SP>(in, n, chunk_syms, g_table, spill,
                                                               PlaceOut{look, n_chunks, blob, blob_cap, offsets, status}, counter);
    if ((threadIdx.x & 31) == 0) {
        if (s.waits) atomicAdd(stats, static_cast<unsigned long long>(s.waits));
        if (s.pend_spills) atomicAdd(stats + 1, static_cast<unsigned long long>(s.pend_spills));
        if (s.spilled_bytes) atomicAdd(stats + 2, static_cast<unsigned long long>(s.spilled_bytes));
    }
}

struct Ctx {
    const uint8_t* in; uint64_t n; uint32_t chunk, n_chunks; const WordEncEntry* table; uint32_t* counter; uint32_t* sizes;
    uint32_t* ref_sizes; uint32_t* status; uint8_t* scratch; uint32_t slot; uint64_t* look; uint8_t* blob; uint64_t* offsets; int sms; int reps;
    uint8_t* ref_blob; uint64_t* ref_offsets; unsigned long long* stats; uint8_t* spill;
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

template <uint32_t RING, uint32_t W, uint32_t D, uint32_t SP>
void run_place(const Ctx& c)
{
    static_assert(kEncTableBytes + W * (RING + kEncStageBytes) <= 227 * 1024, "shared memory");
    const uint32_t smem = kEncTableBytes + W * (RING + kEncStageBytes);
    auto k = ring_place_kernel<RING, W, D, SP>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CK(cudaMemset(c.blob, 0, 2 * c.n));
    CK(cudaMemset(c.offsets, 0, (c.n_chunks + 1) * 8ull));
    CK(cudaMemset(c.stats, 0, 24));
    const double ms = time_ms(c, [&] {
        k<<<c.sms, W * 32, smem>>>(c.in, c.n, c.chunk, c.n_chunks, c.table, c.spill, c.look, c.counter, c.blob, 2 * c.n, c.offsets, c.status,
                                   c.stats);
    }, true);
    unsigned long long st[3] = {};
    CK(cudaMemcpy(st, c.stats, 24, cudaMemcpyDeviceToHost));
    const bool ok = same_container(c);
    const double per = 1.0 / (c.reps + 2) / c.n_chunks;
    std::printf("{\"variant\": \"ring_place\", \"ring\": %u, \"warps\": %u, \"D\": %u, \"spill_pending\": %u, \"ms\": %.4f, "
                "\"waits_per_chunk\": %.4f, \"pending_spills_per_chunk\": %.4f, \"spilled_bytes_per_chunk\": %.1f, \"same_as_k2f\": %s}\n",
                RING, W, D, SP, ms, st[0] * per, st[1] * per, st[2] * per, ok ? "true" : "false");
    std::fflush(stdout);
}

int main(int argc, char** argv)
{
    uint64_t n = 1ull << 30;
    uint32_t chunk = 8192;
    int reps = 10;
    const char* hist = nullptr;
    for (int i = 1; i + 1 < argc; i += 2) {
        if (!std::strcmp(argv[i], "--n")) n = std::strtoull(argv[i + 1], nullptr, 0);
        else if (!std::strcmp(argv[i], "--chunk")) chunk = static_cast<uint32_t>(std::strtoul(argv[i + 1], nullptr, 0));
        else if (!std::strcmp(argv[i], "--reps")) reps = std::atoi(argv[i + 1]);
        else if (!std::strcmp(argv[i], "--hist")) hist = argv[i + 1];
    }
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    // the card's power limit, read in the same process as the timings
    char power[64] = "unknown";
    if (FILE* smi = popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader -i 0", "r")) {
        if (std::fgets(power, sizeof power, smi)) power[std::strcspn(power, "\n")] = 0;
        pclose(smi);
    }
    std::printf("{\"power_limit_and_max_sm_clock\": \"%s\"}\n", power);
    std::printf("{\"device\": \"%s\", \"sms\": %d, \"n\": %llu, \"chunk\": %u, \"reps\": %d, \"data\": \"%s\"}\n", prop.name, sms,
                static_cast<unsigned long long>(n), chunk, reps, hist ? hist : "uniform");

    // the model: uniform (every byte 4096 / 256), or the "counts" of a histogram file scaled to 4096 (each seen byte
    // at least 1, the rounding error on the most frequent one)
    std::vector<uint32_t> freq(256, 16);
    if (hist) {
        FILE* f = std::fopen(hist, "rb");
        if (!f) { std::fprintf(stderr, "cannot open %s\n", hist); return 2; }
        std::string text;
        char buf[4096];
        for (size_t got; (got = std::fread(buf, 1, sizeof buf, f)) > 0;) text.append(buf, got);
        std::fclose(f);
        const size_t at = text.find("\"counts\"");
        if (at == std::string::npos) { std::fprintf(stderr, "no counts in %s\n", hist); return 2; }
        const char* q = std::strchr(text.c_str() + at, '[') + 1;
        std::vector<double> cnt(256);
        double total = 0;
        for (int s = 0; s < 256; s++) {
            char* e;
            cnt[s] = std::strtod(q, &e);
            q = e + 1;
            total += cnt[s];
        }
        uint32_t sum = 0, top = 0;
        for (int s = 0; s < 256; s++) {
            freq[s] = cnt[s] > 0 ? std::max<uint32_t>(1, static_cast<uint32_t>(cnt[s] / total * 4096)) : 0;
            sum += freq[s];
            if (freq[s] > freq[top]) top = s;
        }
        freq[top] += 4096 - sum;
    }
    std::vector<WordEncEntry> tab(256);
    std::vector<uint8_t> slot_sym(4096);
    int exact = 1;
    for (uint32_t s = 0, cum = 0; s < 256; cum += freq[s], s++) {
        tab[s] = word_enc32_entry(freq[s], cum, &exact);
        for (uint32_t j = 0; j < freq[s]; j++) slot_sym[cum + j] = static_cast<uint8_t>(s);
    }

    Ctx c = {};
    c.n = n; c.chunk = chunk; c.n_chunks = static_cast<uint32_t>((n + chunk - 1) / chunk); c.sms = sms; c.reps = reps;
    c.slot = static_cast<uint32_t>((512 + 2ull * chunk + 15) & ~15ull);
    uint8_t* d_in;
    WordEncEntry* d_tab;
    CK(cudaMalloc(&d_in, n + 16));
    CK(cudaMalloc(&d_tab, 256 * sizeof(WordEncEntry)));
    CK(cudaMemcpy(d_tab, tab.data(), 256 * sizeof(WordEncEntry), cudaMemcpyHostToDevice));
    uint8_t* d_slot_sym;
    CK(cudaMalloc(&d_slot_sym, 4096));
    CK(cudaMemcpy(d_slot_sym, slot_sym.data(), 4096, cudaMemcpyHostToDevice));
    gen_kernel<<<sms * 8, 256>>>(d_in, n, 12345, d_slot_sym);
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
    CK(cudaMalloc(&c.stats, 24));
    CK(cudaMalloc(&c.spill, static_cast<uint64_t>(sms) * 32 * kEncRingSpillBytes));     // up to 32 warps per CTA

    // K2, the split encoder: encode into global slots, no compaction
    configure_word_kernels();
    {
        const double ms = time_ms(c, [&] {
            word_encode_kernel<true><<<(c.n_chunks + kEncWarps - 1) / kEncWarps, kEncWarps * 32, kEncSmemBytes>>>(
                c.in, c.n, c.chunk, c.n_chunks, c.table, c.scratch, c.slot, c.ref_sizes, c.status, nullptr, nullptr);
        }, false);
        std::printf("{\"variant\": \"k2_split_encode\", \"ms\": %.4f}\n", ms);
    }
    // K2f as shipped (2 CTAs x 16 warps per SM, two scratch slots per warp), with placement
    {
        const uint32_t grid = sms * RB200_FUSED_MINBLOCKS;
        const double ms = time_ms(c, [&] {
            word_encode_fused_kernel<true><<<grid, kEncWarps * 32, kEncSmemBytes>>>(c.in, c.n, c.chunk, c.n_chunks, c.table, c.scratch, c.slot,
                                                                                    c.look, c.counter, c.blob, 2 * n, c.offsets, c.status, nullptr, nullptr);
        }, true);
        std::printf("{\"variant\": \"k2f_fused_shipped\", \"ms\": %.4f}\n", ms);
        CK(cudaMemcpy(c.ref_blob, c.blob, 2 * n, cudaMemcpyDeviceToDevice));
        CK(cudaMemcpy(c.ref_offsets, c.offsets, (c.n_chunks + 1) * 8ull, cudaMemcpyDeviceToDevice));
    }
    // shapes by occupancy (32 KiB + W x (ring + 512) <= 227 KiB; a ring of at least half a slot, so 20 warps at most)
    // and how an unpublished pending stream is spilled (bytes per step of making room; 0: wait for its offset instead);
    // two alternated passes with placement
    for (int pass = 0; pass < 2; pass++) {
        run_place<12800, 15, 2, kEncRingSlotBytes>(c);
        run_place<10240, 18, 1, kEncRingSlotBytes>(c);
        run_place<9472, 20, 1, kEncRingSlotBytes>(c);
        run_place<9472, 20, 1, 2048>(c);
        run_place<9472, 20, 1, 1024>(c);
        run_place<9472, 20, 1, 0>(c);
        run_place<9472, 20, 2, kEncRingSlotBytes>(c);
    }
    // the step alone.  A stream longer than the ring wraps over its own start (harmless here) and its size no longer
    // matches K2's.
    run_ring<12800, 15, 1>(c);
    run_ring<9472, 20, 1>(c);
    run_ring<8560, 22, 1>(c);
    run_ring<7808, 24, 1>(c);
    uint32_t st = 0;
    CK(cudaMemcpy(&st, c.status, 4, cudaMemcpyDeviceToHost));
    std::printf("{\"status\": %u}\n", st);
    return 0;
}

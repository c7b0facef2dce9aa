// block_kernels.cuh -- device model construction and the per-block-model variants of the
// word-coder kernels (BASELINE config 5: many independent blocks, each with its own
// 256-entry frequency table, scale_bits 12).
//
//   histogram_kernel       SymbolStats::count_freqs   (main.cpp:59-66) on the device
//   block_model_kernel     count_freqs + calc_cum_freqs + normalize_freqs (main.cpp:59-129)
//                          per block, bit-exact, one warp running the order-dependent
//                          "steal a slot" loop with a warp-wide arg-min
//   block_encode_fused_kernel  K5f: model (optional), encoder reciprocal table in shared memory, 32-way encode,
//                          directory and placement in one persistent launch
// The split per-block encoder and the per-block decoders of every coder are in block_coder_kernels.cuh.
#pragma once
#include "device_utils.cuh"
#include "tables.h"
#include "word_decode_tma.cuh"   // WordDecoder
#include "word_kernels.cuh"

namespace rb200 {

// ---------------------------------------------------------------------------
// K7: byte histogram
// ---------------------------------------------------------------------------
constexpr int kHistWarps = 8;

// One histogram copy per LANE, bin-major: counter (bin, lane) lives at word bin * 32 + lane, i.e. in bank `lane`.
// The 32 lanes of a shared-memory atomic therefore never share a bank -- whatever the symbols are: uniform data no
// longer pays the ~3.5 wavefronts of 32 random banks, skewed data no longer serialises on one hot counter (round 1's
// per-warp copies did both and ran at 2.6 TB/s).  All warps of the CTA add into the same 32 KiB.
// GEOM (rb200_container_model_encode_varlen_async): the length from the record (VarlenGeom), on the grid of n_max.
template <bool GEOM = false>
__global__ void __launch_bounds__(kHistWarps * 32)
histogram_kernel(const uint8_t* __restrict__ in, uint64_t n, unsigned long long* __restrict__ counts, const VarlenGeom* __restrict__ geom)
{
    if (GEOM) {
        if (!geom->go) return;
        n = geom->n;
    }
    __shared__ uint32_t s_h[256 * 32];
    for (uint32_t i = threadIdx.x; i < 256 * 32; i += blockDim.x) s_h[i] = 0;
    __syncthreads();
    uint32_t* h = s_h + (threadIdx.x & 31);

    // unaligned head (< 16 bytes) and tail (< 16 bytes) go to block 0, the 16-byte body is grid-strided
    const uint64_t head = min(n, static_cast<uint64_t>((16 - (reinterpret_cast<uintptr_t>(in) & 15)) & 15));
    const uint64_t nvec = (n - head) / 16;
    const uint4* body = reinterpret_cast<const uint4*>(in + head);
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    uint64_t v = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    auto count16 = [&](const uint4& q) {
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            atomicAdd(&h[(w[j] & 0xff) * 32], 1u);
            atomicAdd(&h[((w[j] >> 8) & 0xff) * 32], 1u);
            atomicAdd(&h[((w[j] >> 16) & 0xff) * 32], 1u);
            atomicAdd(&h[(w[j] >> 24) * 32], 1u);
        }
    };
    for (; v + stride < nvec; v += 2 * stride) {             // two loads in flight per thread
        const uint4 q0 = ldg_stream_u128(body + v), q1 = ldg_stream_u128(body + v + stride);
        count16(q0);
        count16(q1);
    }
    if (v < nvec) count16(ldg_stream_u128(body + v));
    if (blockIdx.x == 0) {
        const uint64_t tail_lo = head + nvec * 16;
        for (uint64_t i = threadIdx.x; i < head; i += blockDim.x) atomicAdd(&h[in[i] * 32u], 1u);
        for (uint64_t i = tail_lo + threadIdx.x; i < n; i += blockDim.x) atomicAdd(&h[in[i] * 32u], 1u);
    }
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < 256; s += blockDim.x) {
        unsigned long long t = 0;
#pragma unroll
        for (uint32_t l = 0; l < 32; l++) t += s_h[s * 32 + ((l + s) & 31)];      // rotated: the 32 threads of a warp read 32 banks
        if (t) atomicAdd(&counts[s], t);
    }
}

// geom set: the GEOM instance, with n = n_max sizing the grid
inline void launch_histogram(cudaStream_t stream, uint32_t sms, const uint8_t* d_in, uint64_t n, unsigned long long* d_counts,
                             const VarlenGeom* geom = nullptr)
{
    const uint64_t want = (n / 16 + kHistWarps * 32 - 1) / (kHistWarps * 32);
    // keep each block's per-bin count below 2^32: >= 1 block per 2^31 bytes is plenty
    uint64_t grid = static_cast<uint64_t>(sms) * 8;
    if (want < grid) grid = want ? want : 1;
    auto kernel = geom ? histogram_kernel<true> : histogram_kernel<false>;
    kernel<<<static_cast<uint32_t>(grid), kHistWarps * 32, 0, stream>>>(d_in, n, d_counts, geom);
}

// ---------------------------------------------------------------------------
// per-block model: histogram + normalize_freqs(4096), one CTA per block
// ---------------------------------------------------------------------------
constexpr int kModelWarps = 8;

// calc_cum_freqs + normalize_freqs(target) (main.cpp:68-129) on 256 counts in shared memory, run by ONE warp, bit-exact:
// s_cnt = the counts (their sum below 2^32), s_cum / s_w = 257 / 256 words of workspace (s_w 16-byte aligned); the
// normalised frequencies end up in s_w and in dst[0..256).  target <= 65536: the resample product target * cum is below
// 2^48 and the arg-min key (width << 8 | symbol) below 2^25.  When no symbol can give up a slot (main.cpp:104) it ORs
// fail_bit into the status word.  The per-block callers pass compile-time constants (4096, kStatStream).
template <class T>
__device__ __forceinline__ void block_normalize(const uint32_t* s_cnt, uint32_t* s_cum, uint32_t* s_w, T* __restrict__ dst, uint32_t target,
                                                uint32_t fail_bit, uint32_t* __restrict__ status)
{
    const uint32_t lane = threadIdx.x & 31;
    // calc_cum_freqs (main.cpp:68-73): lane l owns symbols 8l .. 8l+7
    uint32_t run = 0, local[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { local[j] = run; run += s_cnt[8 * lane + j]; }
    uint32_t incl = run;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= static_cast<uint32_t>(d)) incl += v;
    }
    const uint32_t base = incl - run;
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);      // == block_size
    // resample, main.cpp:83-84 (cum[0] stays 0)
#pragma unroll
    for (int j = 0; j < 8; j++)
        s_cum[8 * lane + j] = static_cast<uint32_t>((static_cast<uint64_t>(target) * (base + local[j])) / total);
    if (lane == 31) s_cum[256] = target;                           // target * total / total
    __syncwarp();

    // main.cpp:90-116, symbols in order.  Moving the boundaries between donor and taker by one changes exactly
    // two widths (donor - 1, taker + 1), so the loop runs on widths; the arg-min over 256 widths is warp-wide
    // with the key (width << 8 | symbol): lowest width first, lowest symbol on ties, as the reference's scan.
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const uint32_t t = 8 * lane + j;
        s_w[t] = s_cum[t + 1] - s_cum[t];
    }
    __syncwarp();
    bool failed = false;
    for (uint32_t s = 0; s < 256; s++) {
        if (s_cnt[s] == 0 || s_w[s] != 0) continue;                // warp-uniform
        uint32_t key = 0xffffffffu;
        const uint4 lo = *reinterpret_cast<const uint4*>(&s_w[8 * lane]);
        const uint4 hi = *reinterpret_cast<const uint4*>(&s_w[8 * lane + 4]);
        const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (w[j] > 1) key = min(key, (w[j] << 8) | (8 * lane + j));
        key = __reduce_min_sync(0xffffffffu, key);
        if (key == 0xffffffffu) { failed = true; break; }           // main.cpp:104
        __syncwarp();
        if (lane == 0) {
            s_w[key & 0xffu] -= 1;                                  // main.cpp:107-113 in terms of widths
            s_w[s] += 1;
        }
        __syncwarp();
    }
    if (failed && lane == 0) atomicOr(status, fail_bit);
#pragma unroll
    for (int j = 0; j < 8; j++) dst[8 * lane + j] = static_cast<T>(s_w[8 * lane + j]);            // main.cpp:127
}

// Shared-memory workspace of the per-block model build.
struct BlockModelSmem {
    uint32_t h[kModelWarps][256];     // one private histogram per (warp & 7); h[0] is reused for the 256 widths
    uint32_t cnt[256];
    uint32_t cum[257];
};

// count_freqs + calc_cum_freqs + normalize_freqs(target) (main.cpp:59-129) of one block by the whole CTA, bit-exact.
// The CTA must call it convergently; on return (after a CTA barrier) dst[0..256) holds the normalised frequencies.
// target <= 32768 (the frequencies are u16); the word coder's callers pass the constant 4096.
__device__ __forceinline__ void block_model_build(const uint8_t* __restrict__ blk, uint32_t block_size, BlockModelSmem& sm,
                                                  uint16_t* __restrict__ dst, uint32_t* __restrict__ status, uint32_t target)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (uint32_t i = tid; i < kModelWarps * 256; i += blockDim.x) (&sm.h[0][0])[i] = 0;
    __syncthreads();
    {   // count_freqs, main.cpp:59-66 (more copies per warp were measured slower: the copies share banks)
        uint32_t* h = sm.h[warp & (kModelWarps - 1)];
        const uint32_t head = min(block_size, static_cast<uint32_t>((16 - (reinterpret_cast<uintptr_t>(blk) & 15)) & 15));
        const uint32_t nvec = (block_size - head) / 16;
        const uint4* body = reinterpret_cast<const uint4*>(blk + head);
        for (uint32_t v = tid; v < nvec; v += blockDim.x) {
            const uint4 q = ldg_stream_u128(body + v);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                atomicAdd(&h[w[j] & 0xff], 1u);
                atomicAdd(&h[(w[j] >> 8) & 0xff], 1u);
                atomicAdd(&h[(w[j] >> 16) & 0xff], 1u);
                atomicAdd(&h[w[j] >> 24], 1u);
            }
        }
        for (uint32_t i = tid; i < head; i += blockDim.x) atomicAdd(&h[blk[i]], 1u);
        for (uint32_t i = head + nvec * 16 + tid; i < block_size; i += blockDim.x) atomicAdd(&h[blk[i]], 1u);
    }
    __syncthreads();
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        uint32_t t = 0;
#pragma unroll
        for (int w = 0; w < kModelWarps; w++) t += sm.h[w][s];
        sm.cnt[s] = t;
    }
    __syncthreads();
    if (warp == 0) block_normalize(sm.cnt, sm.cum, sm.h[0], dst, target, kStatStream, status);      // h[0] is reused for the 256 widths
    __syncthreads();
}

// count_freqs of one block by the whole CTA with the bank-private histogram of histogram_kernel (one copy per lane, 32
// KiB at `hist`): no bank conflicts and no hot-counter serialisation.  The CTA must call it convergently; on return
// (after a CTA barrier) s_cnt[0..256) holds the counts and `hist` is free.
__device__ __forceinline__ void block_histogram_wide(const uint8_t* __restrict__ blk, uint32_t block_size, uint32_t* hist, uint32_t* s_cnt)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    for (uint32_t i = tid; i < 256 * 32; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    {   // count_freqs, main.cpp:59-66
        uint32_t* h = hist + lane;
        const uint32_t head = min(block_size, static_cast<uint32_t>((16 - (reinterpret_cast<uintptr_t>(blk) & 15)) & 15));
        const uint32_t nvec = (block_size - head) / 16;
        const uint4* body = reinterpret_cast<const uint4*>(blk + head);
        for (uint32_t v = tid; v < nvec; v += blockDim.x) {
            const uint4 q = ldg_stream_u128(body + v);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                atomicAdd(&h[(w[j] & 0xff) * 32], 1u);
                atomicAdd(&h[((w[j] >> 8) & 0xff) * 32], 1u);
                atomicAdd(&h[((w[j] >> 16) & 0xff) * 32], 1u);
                atomicAdd(&h[(w[j] >> 24) * 32], 1u);
            }
        }
        for (uint32_t i = tid; i < head; i += blockDim.x) atomicAdd(&h[blk[i] * 32u], 1u);
        for (uint32_t i = head + nvec * 16 + tid; i < block_size; i += blockDim.x) atomicAdd(&h[blk[i] * 32u], 1u);
    }
    __syncthreads();
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        uint32_t t = 0;
#pragma unroll
        for (uint32_t l = 0; l < 32; l++) t += hist[s * 32 + ((l + s) & 31)];
        s_cnt[s] = t;
    }
    __syncthreads();
}

// block_model_build on the bank-private histogram (block_histogram_wide).  Used by the fused per-block encoder, where
// the 32 KiB are the (not yet built) encoder table.  s_cnt / s_cum / s_w: 256 / 257 / 256 words.  target as for
// block_model_build.
__device__ __forceinline__ void block_model_build_wide(const uint8_t* __restrict__ blk, uint32_t block_size, uint32_t* hist, uint32_t* s_cnt,
                                                       uint32_t* s_cum, uint32_t* s_w, uint16_t* __restrict__ dst,
                                                       uint32_t* __restrict__ status, uint32_t target)
{
    const uint32_t warp = threadIdx.x >> 5;
    block_histogram_wide(blk, block_size, hist, s_cnt);
    if (warp == 0) block_normalize(s_cnt, s_cum, s_w, dst, target, kStatStream, status);
    __syncthreads();
}

__global__ void __launch_bounds__(kModelWarps * 32)
block_model_kernel(const uint8_t* __restrict__ in, uint32_t block_size, uint16_t* __restrict__ block_freqs,
                   uint32_t* __restrict__ status)
{
    __shared__ uint32_t s_hist[256 * 32];
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];      // block_normalize reads it 16 bytes at a time
    block_model_build_wide(in + static_cast<uint64_t>(blockIdx.x) * block_size, block_size, s_hist, s_cnt, s_cum, s_w,
                           block_freqs + static_cast<uint64_t>(blockIdx.x) * 256, status, kWordSlots);
}

inline void launch_block_models(cudaStream_t stream, const uint8_t* d_in, uint32_t n_blocks, uint32_t block_size,
                                uint16_t* d_freqs, uint32_t* status)
{
    block_model_kernel<<<n_blocks, kModelWarps * 32, 0, stream>>>(d_in, block_size, d_freqs, status);
}

// ---------------------------------------------------------------------------
// K5: per-block decode / encode.  One CTA per block, one warp per chunk of the block (block_coder_kernels.cuh).
// ---------------------------------------------------------------------------
constexpr int kMaxBlockWarps = 32;

// cum[s] for the block's frequencies (u16 from global memory, or the u32 widths the model build left in shared
// memory); returns false if they do not sum to target (the word coder's callers pass the constant 4096)
template <class F>
__device__ __forceinline__ bool block_prefix(const F* freqs, uint32_t* s_cum, uint32_t* s_bad, uint32_t target)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) *s_bad = 0;
    __syncthreads();
    if (tid < 32) {
        uint32_t run = 0, local[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { local[j] = run; run += freqs[8 * lane + j]; }
        uint32_t incl = run;
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= static_cast<uint32_t>(d)) incl += v;
        }
#pragma unroll
        for (int j = 0; j < 8; j++) s_cum[8 * lane + j] = incl - run + local[j];
        if (lane == 31) {
            s_cum[256] = incl;
            if (incl != target) *s_bad = 1;
        }
    }
    __syncthreads();
    return *s_bad == 0;
}

// RansWordTablesInitSymbol for every slot (rans_word_sse41.h:64-72) from the cumulative table in s_cum.  Each thread
// owns a run of consecutive slots: one binary search over the cumulative table for the first, then it walks forward,
// so the work is balanced however skewed the model is.  Sets *s_wide when one symbol takes all 4096 slots.  The
// caller puts a CTA barrier between this and the first read of s_tab.
__device__ __forceinline__ void block_fill_slots(const uint32_t* s_cum, uint32_t* s_tab, uint32_t* s_wide)
{
    const uint32_t per = kWordSlots / blockDim.x;                // blockDim is a power of two between 128 and 1024
    uint32_t slot = threadIdx.x * per;
    uint32_t lo = 0, hi = 256;                                   // largest s with cum[s] <= slot
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (s_cum[mid] <= slot) lo = mid; else hi = mid;
    }
    for (uint32_t j = 0; j < per; j++, slot++) {
        while (slot >= s_cum[lo + 1]) lo++;                      // also steps over zero-width symbols
        const uint32_t f = s_cum[lo + 1] - s_cum[lo];
        if (f == kWordSlots) *s_wide = 1;
        s_tab[slot] = ((f & 0xfffu) << 20) | ((slot - s_cum[lo]) << 8) | lo;
    }
}

// The block's encoder table (8x replicated {magic, x_max | shift, start, 4096 - freq}) from its cumulative table in
// s_cum; returns whether the 32-bit reciprocal is exact for every symbol of this model (tables.h: enc32), which
// selects the kernel variant for the block.  Ends with a CTA barrier.
__device__ __forceinline__ bool block_build_enc_table(const uint32_t* s_cum, bool ok, uint4* s_tab)
{
    const uint32_t tid = threadIdx.x;
    bool exact32 = true;
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        const uint32_t f = ok ? s_cum[s + 1] - s_cum[s] : 0;
        if (f > 1) {
            uint32_t sh = 0;
            while ((1u << sh) < f) sh++;
            const uint64_t pow = 1ull << (31 + sh), M32 = (pow + f - 1) / f;
            if (M32 >> 32 || ((static_cast<uint64_t>(f) << 20) - 1) * (M32 * f - pow) >= pow) exact32 = false;
        }
    }
    const bool r32 = __syncthreads_and(exact32) != 0;
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        const uint32_t f = ok ? s_cum[s + 1] - s_cum[s] : 0;
        WordEncEntry e = {0u, kEncBadSymbol};
        if (f) {
            uint32_t sh = 0;
            while ((1u << sh) < f) sh++;
            if (!r32) {
                const uint64_t M = ((1ull << (32 + sh)) + f - 1) / f;      // in [2^32, 2^33): keep the low word
                e.magic = static_cast<uint32_t>(M);
                e.packed = f | (s_cum[s] << 13) | (sh << 25);
            } else if (f == 1) {
                e.magic = 0xffffffffu;
                e.packed = f | (s_cum[s] << 13);
            } else {
                e.magic = static_cast<uint32_t>(((1ull << (31 + sh)) + f - 1) / f);
                e.packed = f | (s_cum[s] << 13) | ((sh - 1) << 25);
            }
        }
        const uint4 x = r32 ? word_enc_expand<true>(e) : word_enc_expand<false>(e);
#pragma unroll
        for (uint32_t r = 0; r < kEncReplicas; r++) s_tab[s * kEncReplicas + r] = x;
    }
    __syncthreads();
    return r32;
}

// The block's model in s_cum: BUILD, count_freqs + normalize_freqs(M) of the block (block_model_build_wide over the 32
// KiB at hist, written to freqs); else freqs, the caller's row.  Returns block_prefix's verdict (s_bad its flag).
template <bool BUILD>
__device__ __forceinline__ bool block_model_prefix(const uint8_t* __restrict__ blk, uint32_t block_size, uint16_t* __restrict__ freqs,
                                                   uint32_t* hist, uint32_t* s_cnt, uint32_t* s_cum, uint32_t* s_w, uint32_t* s_bad,
                                                   uint32_t* __restrict__ status, uint32_t M)
{
    if (!BUILD) return block_prefix(static_cast<const uint16_t*>(freqs), s_cum, s_bad, M);
    block_model_build_wide(blk, block_size, hist, s_cnt, s_cum, s_w, freqs, status, M);
    return block_prefix(s_w, s_cum, s_bad, M);                    // the widths are still in shared memory
}

// K5f: per-block encode in ONE persistent launch -- model (optional), tables, encode, directory, placement.
//
// CTA 0 only hosts the scanner warp (placement.cuh).  Every other CTA takes block ids from an atomic counter
// (so chunks start in order), builds the block's model when BUILD (count_freqs + normalize_freqs, written to
// block_freqs) or reads it, builds the encoder table in shared memory, and its warps encode the block's chunks into
// kBlockFusedSlots per-warp scratch slots (a SlotQueue) exactly as the fused word encoder does: publish the padded size,
// place the chunk of the PREVIOUS block once the scanner has turned the published sizes into end offsets.  The second
// pass over the block's 64 KiB (histogram first, then encode) is served by the L2.
constexpr uint32_t kBlockFusedSlots = 2;        // scratch slots per worker warp
template <bool BUILD>
__device__ __forceinline__ void block_encode_fused(const uint8_t* __restrict__ in, uint32_t n_blocks, uint32_t block_size,
                                                   uint16_t* __restrict__ block_freqs, uint32_t chunk_syms, uint8_t* __restrict__ scratch,
                                                   uint32_t slot_bytes, uint64_t* __restrict__ look, uint32_t* __restrict__ counter,
                                                   uint8_t* __restrict__ blob, uint64_t blob_cap, uint64_t* __restrict__ offsets,
                                                   uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];          // [32 KiB: histogram copies, then the table][warps x 1 KiB stage + ring]
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];      // block_normalize reads it 16 bytes at a time
    __shared__ uint32_t s_flag[1];
    __shared__ uint32_t s_block;
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t per_block = block_size / chunk_syms;
    const uint32_t n_chunks = n_blocks * per_block;
    if (blockIdx.x == 0) {
        if (warp == 0) fused_scanner(look, n_chunks, lane, status);
        return;
    }
    const uint32_t warps = blockDim.x >> 5;
    const uint32_t tab = smem_addr(s_enc), wsm = tab + kEncTableBytes + warp * kEncWarpSmem;
    const PlaceOut out = {look, n_chunks, blob, blob_cap, offsets, status};
    SlotQueue<kBlockFusedSlots> q(scratch, (blockIdx.x - 1) * warps + warp, slot_bytes);
    for (;;) {
        __syncthreads();                                   // the previous block's table is no longer in use
        if (tid == 0) s_block = atomicAdd(counter, 1u);
        __syncthreads();
        const uint32_t block = s_block;
        if (block >= n_blocks) break;
        const uint8_t* blk = in + static_cast<uint64_t>(block) * block_size;
        uint16_t* freqs = block_freqs + static_cast<uint64_t>(block) * 256;
        const bool ok = block_model_prefix<BUILD>(blk, block_size, freqs, reinterpret_cast<uint32_t*>(s_enc), s_cnt, s_cum, s_w, &s_flag[0],
                                                  status, kWordSlots);
        const bool r32 = block_build_enc_table(s_cum, ok, s_tab);
        if (warp < per_block) {
            const uint8_t* src = blk + static_cast<uint64_t>(warp) * chunk_syms;
            const uint32_t produced = r32 ? encode_stream(src, chunk_syms, WordEncoder<true>{tab}, wsm, q.next_end(), status)
                                          : encode_stream(src, chunk_syms, WordEncoder<false>{tab}, wsm, q.next_end(), status);
            q.finish(out, block * per_block + warp, produced, lane);
        }
    }
    q.drain(out, lane);
}

// GATED (rb200_container_blocks_model_encode_auto_async, with BUILD): runs only when the choice record (CoderChoice,
// device_utils.cuh) names `group`; otherwise every CTA, the scanner's included, exits at entry, before it touches the
// counter, look[] or scratch, which the host zeroes before every launch all the same.
// GEOM (rb200_container_blocks_model_encode_varlen_async, with GATED): on the grid the host plans for n_blocks_max, with
// the block count from the record (BlocksVarlenGeom; 0 when the plan failed, and then every CTA exits at entry).  The
// body takes the count as an argument, so the scanner warp follows the record's chunks and workers past the count find
// no block and drain.  `blob` is the container and blob_cap its capacity; the directory and the blob's place in it are
// worked out here from the count and per_block (= block_size / chunk_syms), as the plan kernel lays them out, rather
// than read from the record: values this cheap to derive from one register are recomputed where they are used instead
// of held, which keeps the 8-warp instance at the spill of the shipped one whose body it runs.
template <bool BUILD, int WARPS, bool GATED = false, bool GEOM = false>
__global__ void __launch_bounds__(WARPS * 32, WARPS <= 8 ? 5 : 1)
block_encode_fused_kernel(const uint8_t* __restrict__ in, uint32_t n_blocks, uint32_t block_size, uint16_t* __restrict__ block_freqs,
                          uint32_t chunk_syms, uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint64_t* __restrict__ look,
                          uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap, uint64_t* __restrict__ offsets,
                          uint32_t* __restrict__ status, const CoderChoice* __restrict__ choice, uint32_t group,
                          const BlocksVarlenGeom* __restrict__ geom, uint32_t per_block)
{
    if (GEOM) n_blocks = geom->n_blocks;
    if ((GEOM && !n_blocks) || (GATED && choice->group != group)) return;      // the same for the whole grid
    if (GEOM) {
        const uint64_t entries = static_cast<uint64_t>(n_blocks) * per_block + 1;     // the directory's
        const uint64_t dir_off = 64 + 512ull * n_blocks, blob_off = dir_off + ((entries + 1) >> 1) * 16;
        offsets = reinterpret_cast<uint64_t*>(blob + dir_off);
        blob += blob_off;
        blob_cap -= blob_off;
    }
    block_encode_fused<BUILD>(in, n_blocks, block_size, block_freqs, chunk_syms, scratch, slot_bytes, look, counter, blob, blob_cap, offsets,
                              status);
}

inline uint32_t block_threads(uint32_t block_size, uint32_t chunk_syms)
{
    uint32_t warps = 4;                // table construction wants a few warps even for 1-chunk blocks;
    while (warps < block_size / chunk_syms) warps <<= 1;   // power of two so 4096 slots split evenly
    return warps * 32;
}

// dynamic shared memory of the per-block encoders (K5f; K5 adds the alias coder's remap) at `threads` threads: the
// table, then 1 KiB per warp
inline uint32_t block_encode_smem(uint32_t threads) { return kEncTableBytes + (threads / 32) * kEncWarpSmem; }

// the instance of the fused per-block encoder for blocks of block_threads() = `threads`: (BUILD, GATED, GEOM) =
// (build, 0, 0) for the fixed calls, (1, 1, 0) for the auto encode, (1, 1, 1) for the device-count encode
using BlockEncodeFusedKernel = decltype(&block_encode_fused_kernel<true, 8>);
template <int WARPS>
inline BlockEncodeFusedKernel block_encode_fused_warps(bool build, bool gated, bool geom)
{
    if (geom) return block_encode_fused_kernel<true, WARPS, true, true>;
    if (gated) return block_encode_fused_kernel<true, WARPS, true>;
    return build ? block_encode_fused_kernel<true, WARPS> : block_encode_fused_kernel<false, WARPS>;
}
inline BlockEncodeFusedKernel block_encode_fused_for(bool build, bool gated, bool geom, uint32_t threads)
{
    return threads <= 256 ? block_encode_fused_warps<8>(build, gated, geom) : block_encode_fused_warps<32>(build, gated, geom);
}

}  // namespace rb200

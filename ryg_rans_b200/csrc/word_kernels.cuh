// word_kernels.cuh -- sm_90a kernels for the word coder (rans_word_sse41.h semantics):
// 32-bit state, 16-bit renormalisation, L = 1 << 16, scale_bits = 12.
//
// One warp = one chunk = one 32-way interleaved stream; lane k owns rANS state k.
// This is the warp-wide form of the reference's SSE4.1 design (README:27-30):
//   RansSimdDecSym    (rans_word_sse41.h:151-179)  -> one shared-memory gather + IMAD
//   RansSimdDecRenorm (rans_word_sse41.h:182-227)  -> __ballot_sync + popc(mask & lanemask_lt)
//                                                     replaces movemask + pshufb LUT
//   RansWordEncPut    (rans_word_sse41.h:81-93)    -> ballot + popc(mask & lanemask_gt),
//                                                     exact division by reciprocal multiply
#pragma once
#include "device_utils.cuh"
#include "encode_stream.cuh"
#include "placement.cuh"
#include "tables.h"

namespace rb200 {

constexpr uint32_t kWordL = 1u << 16;       // RANS_WORD_L, rans_word_sse41.h:35
constexpr uint32_t kWordScaleBits = 12;     // RANS_WORD_SCALE_BITS, :37
constexpr uint32_t kWordSlots = 1u << kWordScaleBits;

// ---------------------------------------------------------------------------
// K2: 32-way word-coder encode into per-chunk worst-case slots of a scratch buffer
// (stage, ring and flush: encode_stream.cuh; the word coder's step: WordEncoder below)
// ---------------------------------------------------------------------------
// build-time switches of the encoders (A/B runs: nvcc -DNAME=value into a second .so, loaded with RB200_LIB)
// The fused word encoder's scratch is live data: (resident warps) x (slots per warp) x (one chunk's stream, 8.3 KB at
// chunks of 8192).  2 CTAs x 16 warps per SM with two slots bring it down to about the 50 MB L2 of an H100 (3 x 16 warps
// with three slots: 100-150 MB), and the evict_last hint then keeps most of it there, so a stream is not read back from
// HBM before it is placed.  H100 SXM at 700 W, 1 GiB uniform bytes, chunks of 8192, ms per encode call
// {CTAs per SM, slots, hint}: {3, 3, no} 1.79 | {3, 2, no} 1.76 | {3, 2, yes} 1.71 | {2, 3, no} 1.67 | {2, 2, no} 1.66 |
// {2, 2, yes} 1.62.  Fewer warps lose more encode throughput than they save traffic (2 x 11 warps, {2, yes}: 1.71), and
// 32-40 warps per SM in other shapes (3 x 12, 3 x 10, 2 x 20, 4 x 8) measured the same as 2 x 16 within noise (on a
// 400 W card: 1.70-1.72 ms against 1.84-1.86 ms for {3, 3, no}).
// Dropping a placed stream's lines from L2 (discard.global.L2, so they are never written back) was slower: 1.66 ms.
#ifndef RB200_FUSED_SLOTS
#define RB200_FUSED_SLOTS 2            // scratch slots per worker warp of the fused word encoder: a chunk is placed SLOTS - 1 chunks late
#endif
constexpr uint32_t kFusedSlots = RB200_FUSED_SLOTS;
#ifndef RB200_FUSED_MINBLOCKS
#define RB200_FUSED_MINBLOCKS 2        // CTAs per SM of the fused word encoder (its grid is SMs x this)
#endif
#ifndef RB200_ENC_KEEP_HINT
#define RB200_ENC_KEEP_HINT true       // evict_last hint on the fused encoder's scratch stores (see enc_flush)
#endif
#ifndef RB200_ENC_ASM_RENORM
#define RB200_ENC_ASM_RENORM 1
#endif
constexpr int kEncWarps = 16;

// {magic, x_max | shift, start, 4096 - freq}
//   x_max = freq << 20 in 32-bit arithmetic (rans_word_sse41.h:85; wraps to 0 for freq 4096, as the
//   reference does); its low 20 bits are zero, so the 4-bit reciprocal shift rides in them:
//   x >= x_max  <=>  (x | 31) >= (x_max | shift), and the funnel shift only looks at the low 5 bits.
// R32: `e` comes from the 32-bit-reciprocal table (tables.h: enc32).  mulhi(x, 2^32 - 1) = x - 1 for the
// freq-1 entries, so their `start` carries the missing (4096 - 1).
template <bool R32>
__device__ __forceinline__ uint4 word_enc_expand(WordEncEntry e)
{
    const uint32_t freq = e.packed & 0x1fffu, start = (e.packed >> 13) & 0xfffu, shift = (e.packed >> 25) & 0xfu;
    const uint32_t fix = (R32 && freq == 1) ? kWordSlots - 1 : 0;
    return make_uint4(e.magic, (freq << 20) | shift, start + fix, kWordSlots - freq);    // freq 0 (bad symbol) <=> w == 4096
}

__device__ __forceinline__ uint32_t funnel_shr_wrap(uint32_t lo, uint32_t hi, uint32_t n)
{
    uint32_t r;
    asm("shf.r.wrap.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(lo), "r"(hi), "r"(n));
    return r;
}

// The word coder for encode_stream (encode_stream.cuh).  step = RansWordEncPut for 32 lanes (rans_word_sse41.h:81-93);
// wpos is the ring position of the next word = 510 - 2 * words_emitted; flags bit 12 set <=> a symbol with freq 0.
template <bool R32>
struct WordEncoder {
    using X = uint32_t;
    static constexpr uint32_t kUnit = 2, kMaxEmit = 2, kBadBit = kWordSlots;
    static constexpr X kInit = kWordL;                 // RansWordEncInit, rans_word_sse41.h:75-78
    uint32_t tab;                                      // shared address of the 8x replicated uint4 table

    template <bool FULL>
    __device__ __forceinline__ void step(EncState<X>& st, uint32_t sym, uint32_t tab_lane, uint32_t ring, uint32_t gt, bool active) const
    {
        bool need = false;
        uint4 e = make_uint4(0, 0, 0, 0);
        if (active) {
            e = lds_u128_ro(tab_lane + sym * (kEncReplicas * 16));
            st.flags |= e.w;
            need = (st.x | 31u) >= e.y;                                   // x >= ((L >> 12) << 16) * freq, :85
        }
#if RB200_ENC_ASM_RENORM
        // the same renormalisation as below with ONE predicate feeding the vote, the store and the shift (the
        // compiler otherwise evaluates the comparison twice and copies x before shifting it)
        if (FULL) {
            asm volatile(
                "{\n\t"
                ".reg .pred p;\n\t"
                ".reg .b32 m, r, a;\n\t"
                "setp.ge.u32 p, %2, %3;\n\t"
                "vote.sync.ballot.b32 m, p, 0xffffffff;\n\t"
                "and.b32 r, m, %4;\n\t"
                "popc.b32 r, r;\n\t"
                "shl.b32 r, r, 1;\n\t"
                "sub.u32 a, %1, r;\n\t"
                "and.b32 a, a, %5;\n\t"
                "or.b32 a, a, %6;\n\t"
                "@p st.shared.u16 [a], %0;\n\t"
                "@p shr.u32 %0, %0, 16;\n\t"
                "popc.b32 m, m;\n\t"
                "shl.b32 m, m, 1;\n\t"
                "sub.u32 %1, %1, m;\n\t"
                "}"
                : "+r"(st.x), "+r"(st.wpos)
                : "r"(st.x | 31u), "r"(e.y), "r"(gt), "n"(kEncRingBytes - 1), "r"(ring)
                : "memory");
        } else
#endif
        {
        const uint32_t mask = __ballot_sync(0xffffffffu, need);
        if (need) {
            sts_u16(ring | ((st.wpos - 2u * __popc(mask & gt)) & (kEncRingBytes - 1)), st.x);   // :86-87, lanes 31..0 downwards
            st.x >>= 16;                                                                        // :88
        }
        st.wpos -= 2u * __popc(mask);
        }
        if (active) {
            uint32_t q;
            if (R32) {
                // x < freq << 20 here, where the 32-bit reciprocal is exact: q = mulhi(x, M32) >> shift
                q = funnel_shr_wrap(__umulhi(st.x, e.x), 0u, e.y);
            } else {
                // q = x / freq exactly for any x: M = 2^32 + magic = ceil(2^(32+shift) / freq), q = (x + mulhi(x, magic)) >> shift
                const uint32_t hi = __umulhi(st.x, e.x);
                const uint32_t lo = st.x + hi;
                q = funnel_shr_wrap(lo, lo < hi ? 1u : 0u, e.y);
            }
            st.x = st.x + e.z + q * e.w;                       // ((x / freq) << 12) + x % freq + start, :92
        }
    }
};

#ifndef RB200_ENC_MINBLOCKS
#define RB200_ENC_MINBLOCKS 3
#endif
template <bool R32>
__global__ void __launch_bounds__(kEncWarps * 32, RB200_ENC_MINBLOCKS)
word_encode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                   const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                   uint32_t* __restrict__ sizes, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];     // [32 KiB table][warps x 1 KiB]
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<R32>(g_table[i / kEncReplicas]);
    __syncthreads();

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * kEncWarps + warp;
    if (chunk >= n_chunks) return;
    const ChunkRange r = chunk_range(chunk, chunk_syms, n);
    encode_chunk_split(in + r.first, r.m, chunk, WordEncoder<R32>{smem_addr(s_enc)}, smem_addr(s_enc) + kEncTableBytes + warp * kEncWarpSmem,
                       scratch, slot_bytes, sizes, status);
}
// dynamic shared memory of both word encoders (K2, K2f)
constexpr uint32_t kEncSmemBytes = kEncTableBytes + kEncWarps * kEncWarpSmem;

// ---------------------------------------------------------------------------
// K2f: persistent encode with the directory and the compaction fused in (the protocol: placement.cuh).
// ---------------------------------------------------------------------------
// Grid = resident capacity (SMs x RB200_FUSED_MINBLOCKS CTAs, sized by the host's encode plan).  Warp 0 of CTA 0 is the
// scanner, every other warp is a worker with kFusedSlots scratch slots (encode_chunks_fused).
template <bool R32>
__global__ void __launch_bounds__(kEncWarps * 32, RB200_FUSED_MINBLOCKS)
word_encode_fused_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                         const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                         uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap,
                         uint64_t* __restrict__ offsets, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];     // [32 KiB table][warps x 1 KiB]
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<R32>(g_table[i / kEncReplicas]);
    __syncthreads();

    const uint32_t tab = smem_addr(s_enc), wsm = tab + kEncTableBytes + (threadIdx.x >> 5) * kEncWarpSmem;
    encode_chunks_fused<kFusedSlots, kEncWarps, RB200_ENC_KEEP_HINT>(in, n, chunk_syms, WordEncoder<R32>{tab}, wsm, scratch, slot_bytes,
                                                                     PlaceOut{look, n_chunks, blob, blob_cap, offsets, status}, counter);
}

// ---------------------------------------------------------------------------
// K6: directory + compaction of the per-chunk slots into the final blob
//
// offsets[c] = E_c - sizes[c], E_c = sum_{j<=c} round_up_16(sizes[j]); offsets[n_chunks] = E_last.
// Pass 1 (scan_tiles_kernel, one CTA per 4096 chunks): tile-local inclusive ends into offsets[],
// tile totals into tile_sums[].  Pass 2 (compact_kernel): every CTA adds the totals of the tiles
// before its own (a handful of values), finalises its directory entries and moves its streams.
// ---------------------------------------------------------------------------
constexpr uint32_t kScanTile = 4096;

__global__ void __launch_bounds__(1024)
scan_tiles_kernel(const uint32_t* __restrict__ sizes, uint32_t n_chunks, uint64_t* __restrict__ offsets,
                  uint64_t* __restrict__ tile_sums)
{
    __shared__ uint64_t s_warp[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t c0 = blockIdx.x * kScanTile + tid * 4;
    uint32_t pad[4];
    uint64_t sum = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        pad[j] = (c0 + j < n_chunks) ? ((sizes[c0 + j] + 15u) & ~15u) : 0u;
        sum += pad[j];
    }
    uint64_t incl = sum;
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= static_cast<uint32_t>(d)) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = s_warp[lane];
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t v = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= static_cast<uint32_t>(d)) w += v;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    uint64_t run = incl - sum + (warp ? s_warp[warp - 1] : 0);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        run += pad[j];
        if (c0 + j < n_chunks) offsets[c0 + j] = run;
    }
    if (tid == 1023) tile_sums[blockIdx.x] = s_warp[31];
}

// for very large directories: turn tile_sums into exclusive prefixes once, so compact CTAs read one value
__global__ void __launch_bounds__(1024)
tile_prefix_kernel(uint64_t* __restrict__ tile_sums, uint32_t n_tiles)
{
    __shared__ uint64_t s_warp[32];
    __shared__ uint64_t s_carry;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n_tiles; base += 1024) {
        const uint32_t i = base + tid;
        const uint64_t v = i < n_tiles ? tile_sums[i] : 0;
        uint64_t incl = v;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= static_cast<uint32_t>(d)) incl += u;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint64_t w = s_warp[lane];
            for (int d = 1; d < 32; d <<= 1) {
                const uint64_t u = __shfl_up_sync(0xffffffffu, w, d);
                if (lane >= static_cast<uint32_t>(d)) w += u;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const uint64_t excl = s_carry + (warp ? s_warp[warp - 1] : 0) + incl - v;
        if (i < n_tiles) tile_sums[i] = excl;
        __syncthreads();
        if (tid == 0) s_carry += s_warp[31];
        __syncthreads();
    }
}

constexpr int kCopyWarps = 8;
constexpr uint32_t kTilePrefixThreshold = 256;   // above this many tiles, tile_prefix_kernel runs first

// one warp moves one chunk stream from the end of its scratch slot to blob[offsets[c]..E_c)
__global__ void __launch_bounds__(kCopyWarps * 32)
compact_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
               uint64_t* __restrict__ offsets, const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed,
               uint32_t n_chunks, uint8_t* __restrict__ blob, uint64_t blob_cap, uint32_t* __restrict__ status)
{
    __shared__ uint64_t s_base;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk0 = blockIdx.x * kCopyWarps;
    if (warp == 0) {      // all chunks of this CTA live in one scan tile (kScanTile % kCopyWarps == 0)
        const uint32_t tile = chunk0 / kScanTile;
        uint64_t acc = 0;
        if (tiles_prefixed) {
            acc = tile_sums[tile];
        } else {
            for (uint32_t t = lane; t < tile; t += 32) acc += tile_sums[t];
            for (int d = 16; d; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
        }
        if (lane == 0) s_base = acc;
    }
    __syncthreads();
    const uint32_t chunk = chunk0 + warp;
    if (chunk >= n_chunks) return;
    const uint32_t size = sizes[chunk];
    const uint64_t end = s_base + offsets[chunk];          // E_c, multiple of 16 (tile-local value from pass 1)
    const uint64_t off = end - size;
    __syncwarp();
    if (lane == 0) {
        offsets[chunk] = off;
        if (chunk == n_chunks - 1) {
            offsets[n_chunks] = end;
            if (end > blob_cap) atomicOr(status, kStatSpace);
        }
    }
    if (end <= blob_cap) place_stream<false>(scratch + static_cast<uint64_t>(chunk + 1) * slot_bytes, size, blob, end, lane);
}

inline void configure_word_kernels()
{
    cudaFuncSetAttribute(word_encode_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
    cudaFuncSetAttribute(word_encode_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
    cudaFuncSetAttribute(word_encode_fused_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
    cudaFuncSetAttribute(word_encode_fused_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
}

}  // namespace rb200

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
#include "container_format.h"
#include "device_utils.cuh"
#include "encode_ring.cuh"
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
// The instances of rb200_container_model_encode_async and its device-length form (model_kernels.cuh), which the flags
// select; with both off, gate and geom are unused.
//   GATED: run only when *gate (the model kernel's r32) names this instance.  The host launches both instances, and
//          the other one exits at entry, before it touches shared memory, the counter, look[] or scratch.
//   GEOM:  n, the chunk count, and on the fused path the blob's place in the container `blob` and its capacity come from
//          the record (VarlenGeom), on a grid sized for n_max; nothing runs when geom->go == 0.  A split-path CTA past
//          the real chunks exits before it stages its table.
template <bool R32, bool GATED = false, bool GEOM = false>
__global__ void __launch_bounds__(kEncWarps * 32, RB200_ENC_MINBLOCKS)
word_encode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                   const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                   uint32_t* __restrict__ sizes, uint32_t* __restrict__ status, const uint32_t* __restrict__ gate,
                   const VarlenGeom* __restrict__ geom)
{
    if (GEOM) n_chunks = geom->n_chunks;
    if ((GEOM && !geom->go) || (GATED && *gate != (R32 ? 1u : 0u)) || (GEOM && blockIdx.x * kEncWarps >= n_chunks)) return;
    extern __shared__ __align__(1024) uint8_t s_enc[];     // [32 KiB table][warps x 1 KiB]
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<R32>(g_table[i / kEncReplicas]);
    __syncthreads();

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * kEncWarps + warp;
    if (chunk >= n_chunks) return;
    if (GEOM) n = geom->n;
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
// scanner, every other warp is a worker with kFusedSlots scratch slots (encode_chunks_fused).  GATED, GEOM: as
// word_encode_kernel; with GEOM every CTA runs.
template <bool R32, bool GATED = false, bool GEOM = false>
__global__ void __launch_bounds__(kEncWarps * 32, RB200_FUSED_MINBLOCKS)
word_encode_fused_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                         const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                         uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap,
                         uint64_t* __restrict__ offsets, uint32_t* __restrict__ status, const uint32_t* __restrict__ gate,
                         const VarlenGeom* __restrict__ geom)
{
    if ((GEOM && !geom->go) || (GATED && *gate != (R32 ? 1u : 0u))) return;     // the same for the whole grid
    extern __shared__ __align__(1024) uint8_t s_enc[];     // [32 KiB table][warps x 1 KiB]
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<R32>(g_table[i / kEncReplicas]);
    __syncthreads();

    const uint32_t tab = smem_addr(s_enc), wsm = tab + kEncTableBytes + (threadIdx.x >> 5) * kEncWarpSmem;
    if (GEOM) {
        n = geom->n;
        n_chunks = geom->n_chunks;
        blob += geom->blob_off;
        blob_cap = geom->blob_cap;
    }
    encode_chunks_fused<kFusedSlots, kEncWarps, RB200_ENC_KEEP_HINT>(in, n, chunk_syms, WordEncoder<R32>{tab}, wsm, scratch, slot_bytes,
                                                                     PlaceOut{look, n_chunks, blob, blob_cap, offsets, status}, counter);
}

// ---------------------------------------------------------------------------
// K2r: the fused word encoder with its streams in shared memory (the chunk loop and placement: encode_ring.cuh).
// Every warp encodes into its own shared-memory stream ring of RING bytes; a finished stream stays there until its end
// offset is published and is then stored to the blob with TMA bulk copies, so no stream goes through global scratch.
// The step loads its symbol 2 D steps and its table entry D steps ahead, so only the state arithmetic is on the chain.
// ---------------------------------------------------------------------------

// shared address of ring position pos, pos in [-RING, RING) (as uint32_t)
template <uint32_t RING>
__device__ __forceinline__ uint32_t ring_addr(uint32_t ring, uint32_t pos)
{
    if constexpr ((RING & (RING - 1)) == 0) return ring + (pos & (RING - 1));
    else return ring + min(pos, pos + RING);
}

// x = ((x / freq) << 12) + x % freq + start for a renormalised x (RansWordEncPut, rans_word_sse41.h:92), e = word_enc_expand
template <bool R32>
__device__ __forceinline__ uint32_t word_enc_fold(uint32_t x, const uint4 e)
{
    uint32_t q;
    if (R32) {
        q = funnel_shr_wrap(__umulhi(x, e.x), 0u, e.y);
    } else {
        const uint32_t hi = __umulhi(x, e.x);
        const uint32_t lo = x + hi;
        q = funnel_shr_wrap(lo, lo < hi ? 1u : 0u, e.y);
    }
    return x + e.z + q * e.w;
}

// one full-warp step on a prefetched table entry: WordEncoder::step's renormalisation, with the word stored at ring
// position wpos - 2 * popc(mask & gt) modulo RING (wpos in [-RING, RING) on entry)
template <bool R32, uint32_t RING>
__device__ __forceinline__ void word_ring_step(uint32_t& x, uint32_t& wpos, uint32_t& flags, const uint4 e, uint32_t ring, uint32_t gt)
{
    flags |= e.w;
    if constexpr ((RING & (RING - 1)) == 0) {
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
            "add.u32 a, a, %6;\n\t"
            "@p st.shared.u16 [a], %0;\n\t"
            "@p shr.u32 %0, %0, 16;\n\t"
            "popc.b32 m, m;\n\t"
            "shl.b32 m, m, 1;\n\t"
            "sub.u32 %1, %1, m;\n\t"
            "}"
            : "+r"(x), "+r"(wpos)
            : "r"(x | 31u), "r"(e.y), "r"(gt), "n"(RING - 1), "r"(ring)
            : "memory");
    } else {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            ".reg .b32 m, r, a, b;\n\t"
            "setp.ge.u32 p, %2, %3;\n\t"
            "vote.sync.ballot.b32 m, p, 0xffffffff;\n\t"
            "and.b32 r, m, %4;\n\t"
            "popc.b32 r, r;\n\t"
            "shl.b32 r, r, 1;\n\t"
            "sub.u32 a, %1, r;\n\t"
            "add.u32 b, a, %5;\n\t"
            "min.u32 a, a, b;\n\t"
            "add.u32 a, a, %6;\n\t"
            "@p st.shared.u16 [a], %0;\n\t"
            "@p shr.u32 %0, %0, 16;\n\t"
            "popc.b32 m, m;\n\t"
            "shl.b32 m, m, 1;\n\t"
            "sub.u32 %1, %1, m;\n\t"
            "}"
            : "+r"(x), "+r"(wpos)
            : "r"(x | 31u), "r"(e.y), "r"(gt), "n"(RING), "r"(ring)
            : "memory");
    }
    x = word_enc_fold<R32>(x, e);
}

// Encode m symbols (one warp) as one 32-way stream that ends at ring position `top` (16-byte aligned) and grows
// downwards, modulo RING; the bytes of encode_stream's stream, preceded by zeros up to a 16-byte boundary.  Returns the
// stream size in bytes (warp-uniform); the stream then fills [top - round_up_16(size), top) of the ring.
//   stage = this warp's 512 B input stage; tab = the shared address of the 8x replicated uint4 table
//   space.reserve(emitted, need): returns once `need` more bytes below the `emitted` ones (counted modulo RING) are
//   free to write; space.emitted(emitted): the stream's emitted bytes from their count modulo RING
template <bool R32, uint32_t RING, uint32_t D, class Space>
__device__ __forceinline__ uint32_t word_encode_stream_ring(const uint8_t* __restrict__ chunk_in, uint32_t m, uint32_t tab, uint32_t stage,
                                                            uint32_t ring, uint32_t top, Space& space, uint32_t* __restrict__ status)
{
    static_assert(D == 1 || D == 2 || D == 4, "the prefetch registers rotate with the 16-step stage block");
    static_assert(RING % 16 == 0 && RING > 2048, "16-byte aligned stream ends; a 16-step block (<= 1 KiB) wraps at most once");
    constexpr uint32_t D2 = 2 * D;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t tab_lane = tab + (lane & (kEncReplicas - 1)) * 16;
    const uint32_t gt = lanemask_gt();
    auto entry = [&](uint32_t s) { return lds_u128_ro(tab_lane + s * (kEncReplicas * 16)); };
    auto emitted = [&](uint32_t w) { const uint32_t d = top - 2u - w; return min(d, d + RING); };
    auto wrap = [](uint32_t w) { return min(w, w + RING); };      // back into [0, RING)

    uint32_t x = kWordL, wpos = top - 2u, flags = 0;
    const uint32_t steps = m >> 5, rem = m & 31;
    const uint32_t nblk = steps >> 4;
    const bool vec_ok = (reinterpret_cast<uintptr_t>(chunk_in) & 15) == 0;
    uint4 parked = make_uint4(0, 0, 0, 0);
    auto fetch = [&](uint32_t b) {               // block b's 512 symbols into registers, one 16-byte vector per lane
        if (vec_ok) parked = ldg_stream_u128(reinterpret_cast<const uint4*>(chunk_in + b * kEncStageBytes) + lane);
    };
    auto fill = [&](uint32_t b) {                // block b into the stage (row j = step 16 b + j)
        if (vec_ok) {
            sts_u128(stage + lane * 16, parked);
        } else {
            const uint8_t* p = chunk_in + b * kEncStageBytes + lane;
#pragma unroll
            for (int j = 0; j < 16; j++) sts_u8(stage + j * 32 + lane, p[j * 32]);
        }
    };

    // symbols are walked last to first (main_simd.cpp:294): the ragged tail first, read directly
    if (nblk) fetch(nblk - 1);
    space.reserve(0, (steps - nblk * 16 + 1) * 64);
    if (rem) {
        const bool active = lane < rem;
        const uint4 e = active ? entry(chunk_in[static_cast<uint64_t>(steps) * 32 + lane]) : make_uint4(0, 0, 0, 0);
        const bool need = active && (x | 31u) >= e.y;
        const uint32_t mask = __ballot_sync(0xffffffffu, need);
        if (need) {
            sts_u16(ring_addr<RING>(ring, wpos - 2u * __popc(mask & gt)), x);
            x >>= 16;
        }
        wpos -= 2u * __popc(mask);
        if (active) {
            flags |= e.w;
            x = word_enc_fold<R32>(x, e);
        }
    }
    for (uint32_t g = steps; g > nblk * 16; g--)
        word_ring_step<R32, RING>(x, wpos, flags, entry(chunk_in[static_cast<uint64_t>(g - 1) * 32 + lane]), ring, gt);
    wpos = wrap(wpos);

    if (nblk) {
        // the software pipeline: during step t the symbol of step t - 2D and the table entry of step t - D are loaded;
        // sy[t % 2D] and en[t % D] hold them (16 % 2D == 0, so the rotation is the same in every block)
        uint32_t sy[D2];
        uint4 en[D];
        __syncwarp();
        fill(nblk - 1);
        if (nblk > 1) fetch(nblk - 2);
        __syncwarp();
#pragma unroll
        for (int j = 15; j >= 16 - static_cast<int>(D2); j--) sy[j % D2] = lds_u8(stage + j * 32 + lane);
#pragma unroll
        for (int j = 15; j >= 16 - static_cast<int>(D); j--) en[j % D] = entry(sy[j % D2]);
        for (uint32_t b = nblk; b-- > 0;) {
            space.reserve(emitted(wpos), 16 * 64);
#pragma unroll
            for (int j = 15; j >= 0; j--) {
                const uint4 e = en[j % D];
                if (j == static_cast<int>(D2) - 1 && b) {      // every row of block b has been read: the stage takes block b - 1
                    __syncwarp();
                    fill(b - 1);
                    if (b > 1) fetch(b - 2);
                    __syncwarp();
                }
                // in block 0 the rows below 0 read stale stage bytes: valid table indices, never used
                sy[j % D2] = lds_u8(stage + ((j - static_cast<int>(D2)) & 15) * 32 + lane);
                en[j % D] = entry(sy[(j - static_cast<int>(D)) & (D2 - 1)]);
                word_ring_step<R32, RING>(x, wpos, flags, e, ring, gt);
            }
            wpos = wrap(wpos);
        }
    }

    // the final states for lanes 31..0 (RansWordEncFlush, main_simd.cpp:298-299), then zeros down to a 16-byte boundary
    space.reserve(emitted(wpos), 32 * 4 + 16);
    const uint32_t hpos = wpos - 4u * (31u - lane);
    sts_u16(ring_addr<RING>(ring, hpos), x >> 16);
    sts_u16(ring_addr<RING>(ring, hpos - 2u), x);
    const uint32_t produced = space.emitted(emitted(wpos)) + 32 * 4;
    const uint32_t gap = ((produced + 15u) & ~15u) - produced;
    if (2u * lane < gap) sts_u16(ring_addr<RING>(ring, wpos - 32u * 4 - 2u * lane), 0);     // wpos - 126 = top - produced, modulo RING
    if (__any_sync(0xffffffffu, (flags & kWordSlots) != 0) && lane == 0) atomicOr(status, kStatSymbol);
    return produced;
}

// K2r's shape: one CTA of RB200_RING_WARPS warps per SM, each with a ring of RB200_RING_BYTES and a 512 B stage, and the
// table: 32 KiB + 20 x (9472 + 512) B = 227 KiB, all the shared memory a CTA can have.  The ring no longer holds a
// worst-case stream (12 480 B at chunks of 8192) and the pending one before it: what does not fit goes to the warp's
// spill slots (encode_ring.cuh).  Occupancy is what pays: 20 warps at 96 registers, no local-memory spills.  At 22 and
// 24 warps ptxas allocates 80 registers (-Xptxas -v) and spills to local memory.
// H100 80GB HBM3 at 700 W, 1 GiB, chunks of 8192, ms per call with placement (tools/encode_ring_lab.cu, two alternated
// passes; D = prefetch distance; P = RB200_RING_PEND_PIECE, 16512 = a pending stream spilled whole, 0 = its offset
// waited for; spilled = bytes per chunk that went through a spill slot):
//   uniform bytes: {12800, 15, 2} 1.355-1.358 | {10240, 18, 1, P 16512} 1.259-1.270, 2.7 KB spilled |
//   {9472, 20, 1, P 16512} 1.246-1.283, 4.4 KB spilled | {9472, 20, 1, P 2048} 1.237-1.241, 1.8 KB |
//   {9472, 20, 1, P 1024} 1.212-1.214, 0.96 KB, a pending stream spilled from in 94 % of chunks |
//   {9472, 20, 2, P 16512} 1.257-1.267 | {9472, 20, 1, P 0} 2.79-3.21 | {8560, 22, 2} 1.505 and {8560, 22, 1} 1.92
//   (register spills); K2f 1.574.  The step alone: {12800, 15, 1} 1.158-1.166 | {10240, 18, 1} 1.039-1.050 |
//   {9472, 20, 1} 0.981-0.988 | {8560, 22, 1} 0.942-0.950 | {7808, 24, 1} 0.908-0.917.
//   text-like bytes (book1 histogram, nothing spilled at 20 warps): {12800, 15, 2} 1.358-1.365 | {10240, 18, 1}
//   1.215-1.227 | {9472, 20, 1} 1.155-1.163 for every P but 0 (1.193-1.196) | {9472, 20, 2} 1.152-1.158 |
//   {8560, 22, 2} 1.182-1.186 | {7808, 24, 2} 1.395-1.400 (with 12 480 B slots); K2f 1.200.
// The sweep of the 15-warp design, H100 SXM at 400 W, 1 GiB uniform bytes, chunks of 8192, ms per call of the step alone (no placement:
// tools/encode_ring_lab.cu), {ring bytes, warps, D}: {16384, 11, 1} 2.00 | {16384, 11, 2} 1.73 | {16384, 11, 4} 1.60 |
// {14336, 13, 2} 1.32 | {14336, 13, 4} 1.33 | {13312, 14, 1} 1.23 | {13312, 14, 2} 1.24 | {13312, 14, 4} 1.26 |
// {12800, 15, 1} 1.18 | {12800, 15, 2} 1.25 | {12800, 15, 4} 1.27; the split encoder (K2, 16 warps x 3 CTAs, streams
// through global slots) 1.23, the shipped K2f with placement 1.71.  At 11 warps the step is latency bound and the
// prefetch distance pays; at 14-15 warps the warps hide the latency and D = 1 issues least.  With placement
// (encode_ring.cuh) the order changes: {12800, 15, 2} 1.37-1.38 | {12800, 15, 1} 1.59-1.75 | {13312, 14, 1} 1.41-1.42 |
// {14336, 13, 2} 1.50-1.51 | {16384, 11, 4} 1.76-1.77, against 1.70-1.71 for K2f in the same runs (two sessions).
#ifndef RB200_RING_BYTES
#define RB200_RING_BYTES 9472
#endif
#ifndef RB200_RING_WARPS
#define RB200_RING_WARPS 20
#endif
#ifndef RB200_RING_PEND_PIECE
#define RB200_RING_PEND_PIECE 1024     // bytes of an unpublished pending stream spilled per step of making room (encode_ring.cuh)
#endif
#ifndef RB200_RING_AHEAD
#define RB200_RING_AHEAD 1             // D: table entries loaded D steps ahead, symbols 2 D steps ahead
#endif
constexpr uint32_t kEncRingStreamBytes = RB200_RING_BYTES, kEncRingWarps = RB200_RING_WARPS;
constexpr uint32_t kEncRingMaxChunk = 8192;     // chunks of at most this many symbols: a spill slot holds any of their streams
constexpr uint32_t kEncRingSmemBytes = kEncTableBytes + kEncRingWarps * (kEncRingStreamBytes + kEncStageBytes);

// Each worker warp's two spill slots (encode_ring.cuh), one worst-case stream each; the host sizes the workspace as
// grid x kEncRingWarps of them (including the scanner warp's, unused).
// A slot holds any stream of a chunk of kEncRingMaxChunk symbols, also one whose frequency-0 symbols make every step
// emit a word (2 x 8192 + 128 B): such a call fails with kStatSymbol, but its spills stay inside the warp's own slots.
constexpr uint32_t kEncRingSlotBytes = 2 * kEncRingMaxChunk + 128;
constexpr uint32_t kEncRingSpillBytes = 2 * kEncRingSlotBytes;

// The body of K2r at a given shape (the kernels below use RB200_RING_*): dynamic shared memory
// [32 KiB table][W rings of RING bytes][W stages of 512 B], and kEncRingSpillBytes per warp at `spill`.  Returns what
// this warp's ring did (encode_ring.cuh).
template <bool R32, uint32_t RING, uint32_t W, uint32_t D, uint32_t PEND_PIECE = RB200_RING_PEND_PIECE>
__device__ __forceinline__ RingStats word_encode_ring(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms,
                                                      const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ spill,
                                                      const PlaceOut& out, uint32_t* __restrict__ counter)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) s_tab[i] = word_enc_expand<R32>(g_table[i / kEncReplicas]);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, tab = smem_addr(s_enc);
    const uint32_t ring = tab + kEncTableBytes + warp * RING, stage = tab + kEncTableBytes + W * RING + warp * kEncStageBytes;
    uint8_t* slots = spill + (static_cast<uint64_t>(blockIdx.x) * W + warp) * kEncRingSpillBytes;
    uint32_t* status = out.status;
    using Ring = StreamRing<RING, kEncRingSlotBytes, PEND_PIECE>;
    return encode_chunks_ring<RING, kEncRingSlotBytes, PEND_PIECE>(in, n, chunk_syms, ring, slots, out, counter,
                                                                   [=](const uint8_t* chunk_in, uint32_t m, Ring& q) {
        return word_encode_stream_ring<R32, RING, D>(chunk_in, m, tab, stage, ring, q.top, q, status);
    });
}

// Grid = min(SMs, what the chunks need), sized by the host's encode plan; chunk_syms <= kEncRingMaxChunk; spill: grid x
// kEncRingWarps x kEncRingSpillBytes bytes.
template <bool R32>
__global__ void __launch_bounds__(kEncRingWarps * 32, 1)
word_encode_ring_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                        const WordEncEntry* __restrict__ g_table, uint8_t* __restrict__ spill, uint64_t* __restrict__ look,
                        uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap, uint64_t* __restrict__ offsets,
                        uint32_t* __restrict__ status)
{
    word_encode_ring<R32, kEncRingStreamBytes, kEncRingWarps, RB200_RING_AHEAD>(in, n, chunk_syms, g_table, spill,
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

// GEOM (the device-length and device-count encodes): grids sized for the bound, the chunk count and the directory's and
// blob's places in the container from the record (VarlenGeom, device_utils.cuh), with `offsets` (scan) and `blob`
// (compaction) the container; CTAs past the real tiles or chunks exit at entry.  The host fixes whether
// tile_prefix_kernel runs from the bound's tile count; the prefix and the compaction then both use the device's, which
// gives the same sums as either choice.
// GATED (rb200_container_model_encode_auto_async): the three kernels run only when the choice record (CoderChoice,
// device_utils.cuh) names `group`, the launch group whose split encoder they finish; otherwise they exit at entry.
template <bool GEOM, bool GATED>
__device__ __forceinline__ void scan_tiles(const uint32_t* __restrict__ sizes, uint32_t n_chunks, uint64_t* __restrict__ offsets,
                                           uint64_t* __restrict__ tile_sums, const VarlenGeom* __restrict__ geom,
                                           const CoderChoice* __restrict__ choice, uint32_t group)
{
    if (GATED && choice->group != group) return;
    if (GEOM) {
        n_chunks = geom->n_chunks;
        if (!geom->go || blockIdx.x * kScanTile >= n_chunks) return;
        offsets = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(offsets) + geom->dir_off);
    }
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

template <bool GEOM = false, bool GATED = false>
__global__ void __launch_bounds__(1024)
scan_tiles_kernel(const uint32_t* __restrict__ sizes, uint32_t n_chunks, uint64_t* __restrict__ offsets,
                  uint64_t* __restrict__ tile_sums, const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice,
                  uint32_t group)
{
    scan_tiles<GEOM, GATED>(sizes, n_chunks, offsets, tile_sums, geom, choice, group);
}

// for very large directories: turn tile_sums into exclusive prefixes once, so compact CTAs read one value
template <bool GEOM = false, bool GATED = false>
__global__ void __launch_bounds__(1024)
tile_prefix_kernel(uint64_t* __restrict__ tile_sums, uint32_t n_tiles, const VarlenGeom* __restrict__ geom,
                   const CoderChoice* __restrict__ choice, uint32_t group)
{
    if (GATED && choice->group != group) return;
    if (GEOM) {
        if (!geom->go) return;
        n_tiles = (geom->n_chunks + kScanTile - 1) / kScanTile;
    }
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

// The blocks rb200_container_blocks_stored_encode_async stores: the input, chunks of chunk_syms symbols, per_block to a
// block, and blocks_store_kernel's verdict per block (nonzero: stored).  rb200_container_stored_encode_async: one chunk
// per "block" and chunks_store_kernel's verdicts, with the input's length n for its ragged last chunk.
struct StoredBlocks {
    const uint8_t* in;
    const uint32_t* stored;
    uint32_t per_block, chunk_syms;
    uint64_t n;
};

// one warp moves one chunk stream from the end of its scratch slot to blob[offsets[c]..E_c)
// STORED (rb200_container_blocks_stored_encode_async): a chunk of a stored block is its symbols from the input instead,
// with zero padding (place_stored); its size is already round16(chunk_syms).  RAGGED (with STORED,
// rb200_container_stored_encode_async): a stored chunk has m_c symbols, fewer than chunk_syms when it is the last of
// st.n, and its size is round16(m_c); nothing at or past in + n is read.
template <bool GEOM, bool GATED, bool STORED = false, bool RAGGED = false>
__device__ __forceinline__ void compact(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
                                        uint64_t* __restrict__ offsets, const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed,
                                        uint32_t n_chunks, uint8_t* __restrict__ blob, uint64_t blob_cap, uint32_t* __restrict__ status,
                                        const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice, uint32_t group,
                                        const StoredBlocks& st = StoredBlocks{})
{
    if (GATED && choice->group != group) return;
    if (GEOM) {
        n_chunks = geom->n_chunks;
        if (!geom->go || blockIdx.x * kCopyWarps >= n_chunks) return;
        offsets = reinterpret_cast<uint64_t*>(blob + geom->dir_off);
        blob += geom->blob_off;
        blob_cap = geom->blob_cap;
    }
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
    if (end <= blob_cap) {
        if (STORED && st.stored[chunk / st.per_block])
            place_stored(st.in + static_cast<uint64_t>(chunk) * st.chunk_syms,
                         RAGGED ? container_chunk_symbols(chunk, st.chunk_syms, st.n) : st.chunk_syms, blob + (end - size), lane);
        else
            place_stream<false>(scratch + static_cast<uint64_t>(chunk + 1) * slot_bytes, size, blob, end, lane);
    }
}

template <bool GEOM = false, bool GATED = false>
__global__ void __launch_bounds__(kCopyWarps * 32)
compact_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
               uint64_t* __restrict__ offsets, const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed,
               uint32_t n_chunks, uint8_t* __restrict__ blob, uint64_t blob_cap, uint32_t* __restrict__ status,
               const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice, uint32_t group)
{
    compact<GEOM, GATED>(scratch, slot_bytes, sizes, offsets, tile_sums, tiles_prefixed, n_chunks, blob, blob_cap, status, geom, choice, group);
}

// the STORED compaction of rb200_container_blocks_stored_encode_async (ungated, every length by value)
__global__ void __launch_bounds__(kCopyWarps * 32)
compact_stored_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
                      uint64_t* __restrict__ offsets, const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed,
                      uint32_t n_chunks, uint8_t* __restrict__ blob, uint64_t blob_cap, uint32_t* __restrict__ status, StoredBlocks st)
{
    compact<false, false, true>(scratch, slot_bytes, sizes, offsets, tile_sums, tiles_prefixed, n_chunks, blob, blob_cap, status, nullptr,
                                nullptr, 0, st);
}

// the compaction of rb200_container_stored_encode_async: STORED and RAGGED, one chunk per verdict (ungated, every length
// by value)
__global__ void __launch_bounds__(kCopyWarps * 32)
chunks_stored_compaction_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
                                uint64_t* __restrict__ offsets, const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed,
                                uint32_t n_chunks, uint8_t* __restrict__ blob, uint64_t blob_cap, uint32_t* __restrict__ status, StoredBlocks st)
{
    compact<false, false, true, true>(scratch, slot_bytes, sizes, offsets, tile_sums, tiles_prefixed, n_chunks, blob, blob_cap, status,
                                      nullptr, nullptr, 0, st);
}

// The GEOM instances of the two stored compactions (rb200_container_blocks_stored_encode_varlen_async and
// rb200_container_stored_encode_varlen_async): on the grid of the bound, with `blob` the container, the chunk count,
// the directory and the blob from the record; the version 6 one also takes the input's length, for its ragged last
// chunk, from there.
__global__ void __launch_bounds__(kCopyWarps * 32)
compact_stored_varlen_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
                             const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed, uint8_t* __restrict__ blob,
                             uint32_t* __restrict__ status, const VarlenGeom* __restrict__ geom, StoredBlocks st)
{
    compact<true, false, true>(scratch, slot_bytes, sizes, nullptr, tile_sums, tiles_prefixed, 0, blob, 0, status, geom, nullptr, 0, st);
}

__global__ void __launch_bounds__(kCopyWarps * 32)
chunks_stored_compaction_varlen_kernel(const uint8_t* __restrict__ scratch, uint32_t slot_bytes, const uint32_t* __restrict__ sizes,
                                       const uint64_t* __restrict__ tile_sums, uint32_t tiles_prefixed, uint8_t* __restrict__ blob,
                                       uint32_t* __restrict__ status, const VarlenGeom* __restrict__ geom, StoredBlocks st)
{
    st.n = geom->n;
    compact<true, false, true, true>(scratch, slot_bytes, sizes, nullptr, tile_sums, tiles_prefixed, 0, blob, 0, status, geom, nullptr, 0,
                                     st);
}

// the K2 and K2f instances: (R32, GATED, GEOM) = (r32, 0, 0) for an rb200_model, (r32, 1, 0) and (r32, 1, 1) for the
// model encodes
template <bool R32, bool GATED, bool GEOM>
inline void configure_word_encode()
{
    for (const void* k : {reinterpret_cast<const void*>(word_encode_kernel<R32, GATED, GEOM>),
                          reinterpret_cast<const void*>(word_encode_fused_kernel<R32, GATED, GEOM>)}) {
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncSmemBytes);
    }
}

inline void configure_word_kernels()
{
    configure_word_encode<false, false, false>(); configure_word_encode<true, false, false>();
    configure_word_encode<false, true, false>(); configure_word_encode<true, true, false>();
    configure_word_encode<false, true, true>(); configure_word_encode<true, true, true>();
    cudaFuncSetAttribute(word_encode_ring_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_ring_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncRingSmemBytes);
    cudaFuncSetAttribute(word_encode_ring_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_encode_ring_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kEncRingSmemBytes);
}

}  // namespace rb200

// block_coder_kernels.cuh -- the split encoder and the decoder of every per-block coder: the word coder
// (rans_word_sse41.h) at scale_bits 12, and the byte (main.cpp), rans64 (main64.cpp) and alias (main_alias.cpp) coders
// at scale_bits 8..15.  One CTA per block, one warp per chunk, at most 32 chunks per block, each block's model
// normalised to 1 << scale_bits.
//
//   block_coder_encode_kernel<CODER, SB, BUILD>
//                          BUILD: count_freqs + normalize_freqs(1 << sb) of the block (block_model_build_wide, bit-exact,
//                          written to block_freqs); else the caller's row.  Then the block's encoder table in shared
//                          memory: the word coder's reciprocal table (block_build_enc_table, WordEncoder<r32>), or the
//                          tables.h formulas (byte_enc_entry / rans64_enc_entry, 8x replicated as K8 / K9 stage it), and
//                          encode_chunk_split per warp with AliasEncoder<false, SB> / Rans64Encoder: the split path's
//                          slots, followed by K6's tile scan and compaction.  The word coder has the flags-off instance
//                          only: a word encode that builds its models runs K5f (block_encode_fused_kernel).
//   block_decode_kernel<CODER, SB>
//                          the block's decode table in shared memory (block_decode_table: the word coder's 4096 slot
//                          entries, RansWordTablesInitSymbol of rans_word_sse41.h:64-72; cum2sym[1 << sb], then
//                          byte_dec_symbol x 256 or rans64's 16x replicated {start, freq}), then each warp's chunk
//                          (block_decode_chunk: decode_window_chunk with WordDecoder<WIDE> / ByteDecoder<SB> / Rans64Decoder).
//                          container_decode.cuh's block_decode_planned_kernel runs the same two steps per block.
//   CODER = RB200_CODER_ALIAS  the block's alias table built by the CTA (block_alias_tables, over the coding table's place),
//                          then AliasEncoder<true, SB> with the remap (block_alias_remap, after the warps' stages) or
//                          AliasDecoder<SB, lean> on kAliasDecReplicas copies of the 256 bucket entries
//
// A block whose frequencies do not sum to 1 << sb: the encoder codes it with an empty model (every symbol flagged,
// RB200_E_SYMBOL), the decoder flags kStatStream and decodes nothing of it.
#pragma once
#include "alias_kernels.cuh"
#include "block_kernels.cuh"
#include "rans64_kernels.cuh"
#include "tables.h"

namespace rb200 {

// the largest scale_bits of a per-block model: its frequencies are u16, and 1 << 15 holds a one-symbol block
constexpr uint32_t kBlockCoderMaxScaleBits = 15;

// ---------------------------------------------------------------------------
// make_alias_table (main_alias.cpp:147-237) of one block, built by the CTA: bit-exact with alias_tables_core and
// rb200_alias_tables_build (tables.h, model_host.cpp), which stay the host builders.
// ---------------------------------------------------------------------------
// The outputs of alias_tables_core, and the per-symbol records of the pairing that phase 2 turns into them.  12.5 KiB:
// the per-block alias kernels place it over their (not yet built) 32 KiB coding table.
struct AliasBuildSmem {
    uint32_t divider[256];
    uint32_t slot_adjust[512];
    uint32_t slot_freqs[512];
    uint32_t rest[256];         // phase 1: what each symbol still has to hand out (main_alias.cpp's rest)
    uint32_t own[256];          // the part of bucket s that s keeps (divider[s] before :219)
    uint32_t lend_base[256];    // taker s: what its donor had lent to earlier takers (= earlier buckets)
    uint32_t own_base[256];     // what s had lent to buckets below s: given[s] when bucket s is handed out (:217)
    uint32_t lent[256];         // everything s lent
    uint32_t dst[512];          // remap: where bucket s's own part [2s] and its partner's part [2s + 1] start, minus k
    uint8_t sym_id[512];
};

// Phase 1 (main_alias.cpp:159-204) on warp 0, phase 2 (:207-232) on the CTA, from the block's s_cum[257] (sum M, a
// multiple of 256).  Every thread of the CTA calls it; it ends with a CTA barrier and returns what alias_tables_core
// returns: false when some symbol is not handed exactly its frequency (never for a table that sums to M).
//
// Phase 1 is a chain of at most 256 (taker, donor) steps.  Each step needs "the first index >= p whose rest is below
// (taker) / at least (donor) the bucket".  Lane l keeps bit k of `under` for symbol 32k + l, so one ballot over bit k
// is word k of the 256-bit predicate rest < bucket, and a query is one ballot per word from p's word on (usually one).
// Only the donor's rest changes in a step, so only its bit is updated.
// Phase 2 needs given[] in bucket order.  A donor's run of steps is contiguous and its takers come in increasing bucket
// order (the first may be the previous donor, which lies below the resume point; the rest come from the resume scan),
// so what a donor lent before taker t is a running sum over its run (lend_base), and what it lent below its own bucket
// is that sum at the first taker above it (own_base).  Then every bucket's entries are independent.
__device__ __forceinline__ bool block_alias_tables(const uint32_t* s_cum, uint32_t M, AliasBuildSmem& a)
{
    const uint32_t tid = threadIdx.x, lane = tid & 31, bucket = M >> 8;
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        a.rest[s] = s_cum[s + 1] - s_cum[s];
        a.own[s] = bucket;
        a.lend_base[s] = 0;
        a.own_base[s] = 0;
        a.lent[s] = 0;
        a.sym_id[2 * s] = a.sym_id[2 * s + 1] = static_cast<uint8_t>(s);
    }
    __syncthreads();
    if (tid < 32) {
        uint32_t under = 0;
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) under |= static_cast<uint32_t>(a.rest[32 * k + lane] < bucket) << k;
        // the first index >= p (p <= 257) with rest < bucket (want_under) or rest >= bucket, 256 if none
        auto next = [&](uint32_t p, bool want_under) {
            const uint32_t bits = want_under ? under : ~under;
            for (uint32_t k = p >> 5; k < 8; k++) {
                uint32_t w = __ballot_sync(0xffffffffu, (bits >> k) & 1u);
                if (k == (p >> 5)) w &= ~0u << (p & 31);
                if (w) return 32 * k + __ffs(w) - 1;
            }
            return 256u;
        };
        uint32_t donor = next(0, false), taker = next(0, true);   // :172-175
        uint32_t resume = taker + 1;                              // :179
        uint32_t rd = donor < 256 ? a.rest[donor] : 0;            // the donor's rest
        uint32_t before = 0;                                      // what the donor lent in its earlier steps
        bool crossed = false;                                     // the donor has had a taker above its own bucket
        while (donor < 256 && taker < 256) {                      // :183
            const uint32_t rt = a.rest[taker], give = bucket - rt;
            if (lane == 0) {
                a.sym_id[2 * taker] = static_cast<uint8_t>(donor);     // :185
                a.own[taker] = rt;                                     // :186
                a.lend_base[taker] = before;
                if (!crossed && taker > donor) a.own_base[donor] = before;
            }
            crossed |= taker > donor;
            before += give;
            rd -= give;                                           // :189
            a.rest[donor] = rd;                                   // every lane stores it, so every lane reads it back
            const bool low = rd < bucket;
            if (low && lane == (donor & 31)) under |= 1u << (donor >> 5);
            if (!low || resume <= donor) {                        // :192
                taker = next(resume, true);
                resume = taker + 1;
            } else {
                taker = donor;                                    // :199 (donor became a taker behind us)
            }
            if (low) {                                            // :202-203: the donor's run ends
                if (lane == 0) {
                    if (!crossed) a.own_base[donor] = before;
                    a.lent[donor] = before;
                }
                before = 0;
                crossed = false;
                donor = next(donor + 1, false);
                rd = donor < 256 ? a.rest[donor] : 0;             // never a donor before: its rest is its frequency
            }
        }
        if (donor < 256 && lane == 0) {
            if (!crossed) a.own_base[donor] = before;
            a.lent[donor] = before;
        }
    }
    __syncthreads();
    bool bad = false;
    for (uint32_t s = tid; s < 256; s += blockDim.x) {            // :207-232, one bucket per thread
        const uint32_t other = a.sym_id[2 * s], own = a.own[s], lo = s * bucket, f = s_cum[s + 1] - s_cum[s];
        const uint32_t own_base = a.own_base[s];
        const uint32_t other_base = other == s ? own_base : a.lend_base[s] + (other < s ? a.own[other] : 0);
        a.divider[s] = lo + own;                                  // :219
        a.slot_freqs[2 * s + 1] = f;                              // :221
        a.slot_freqs[2 * s] = s_cum[other + 1] - s_cum[other];    // :222
        a.slot_adjust[2 * s + 1] = lo - own_base;                 // :223
        a.slot_adjust[2 * s] = lo - (other_base - own);           // :224
        a.dst[2 * s] = s_cum[s] + own_base - lo;
        a.dst[2 * s + 1] = s_cum[other] + other_base - lo - own;
        bad |= own + a.lent[s] != f;                              // :235-236 (given[s] = own + what s lent)
    }
    return __syncthreads_or(bad) == 0;
}

// alias_remap (main_alias.cpp:225-228) as u16 from a pairing that block_alias_tables accepted, one slot per thread:
// slot j of bucket s = j / bucket goes to s's own part or to its partner's, after what earlier buckets gave that
// symbol.  The caller puts a CTA barrier between this and the first read of remap.
__device__ __forceinline__ void block_alias_remap(const AliasBuildSmem& a, uint32_t M, uint16_t* remap)
{
    const uint32_t lb = __ffs(M >> 8) - 1;                        // log2(bucket)
    for (uint32_t j = threadIdx.x; j < M; j += blockDim.x) {
        const uint32_t s = j >> lb;
        remap[a.dst[2 * s + (j - (s << lb) >= a.own[s])] + j] = static_cast<uint16_t>(j);
    }
}

// dynamic shared memory of the split per-block encoder: the 32 KiB table, then 1 KiB per warp (as K5f's); the alias
// coder's remap (u16, 1 << sb entries) after them
inline uint32_t block_coder_encode_smem(uint32_t coder, uint32_t sb, uint32_t threads)
{
    return block_encode_smem(threads) + (coder == RB200_CODER_ALIAS ? (2u << sb) : 0u);
}

// dynamic shared memory of the per-block decoders: 1 KiB of stream window per warp, then the table: the word coder's
// 4096 slot entries, the alias coder's bucket entries, or cum2sym and the symbol entries
__host__ __device__ constexpr uint32_t block_coder_sym_bytes(uint32_t coder)
{
    return coder == RB200_CODER_BYTE ? 256 * 4 : kRans64DecSymBytes;
}
inline uint32_t block_coder_decode_smem(uint32_t coder, uint32_t sb, uint32_t threads)
{
    if (coder == RB200_CODER_WORD) return (threads / 32) * kRingBytes + kWordSlots * 4;
    if (coder == RB200_CODER_ALIAS) return (threads / 32) * kRingBytes + 256 * kAliasDecReplicas * 16;   // the bucket table
    return (threads / 32) * kRingBytes + (1u << sb) + block_coder_sym_bytes(coder);
}

template <uint32_t CODER, uint32_t SB, bool BUILD>
__device__ __forceinline__ void block_coder_encode(const uint8_t* __restrict__ in, uint32_t block_size, uint16_t* __restrict__ block_freqs,
                                                   uint32_t sb_rt, uint32_t chunk_syms, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                                                   uint32_t* __restrict__ sizes, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_benc[];         // [32 KiB: histogram copies (BUILD), then the table][warps x 1 KiB]
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];                 // block_normalize reads it 16 bytes at a time
    __shared__ uint32_t s_flag[1];
    const uint32_t sb = SB ? SB : sb_rt, M = 1u << sb;
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const uint8_t* blk = in + static_cast<uint64_t>(blockIdx.x) * block_size;
    uint16_t* freqs = block_freqs + static_cast<uint64_t>(blockIdx.x) * 256;
    bool ok = block_model_prefix<BUILD>(blk, block_size, freqs, reinterpret_cast<uint32_t*>(s_benc), s_cnt, s_cum, s_w, &s_flag[0], status, M);
    const uint32_t warps = blockDim.x >> 5;
    const uint32_t remap = smem_addr(s_benc) + kEncTableBytes + warps * kEncWarpSmem;
    if (CODER == RB200_CODER_ALIAS && ok) {
        // the pairing and the remap, in the table's place; a table that sums to M always pairs
        AliasBuildSmem& a = *reinterpret_cast<AliasBuildSmem*>(s_benc);
        ok = block_alias_tables(s_cum, M, a);
        if (ok) block_alias_remap(a, M, reinterpret_cast<uint16_t*>(s_benc + kEncTableBytes + warps * kEncWarpSmem));
        __syncthreads();
    }
    uint4* s_tab = reinterpret_cast<uint4*>(s_benc);
    bool r32 = false;
    if (CODER == RB200_CODER_WORD) {
        r32 = block_build_enc_table(s_cum, ok, s_tab);              // ends with a CTA barrier
    } else {
        // the encoder table as K8 / K9 stage theirs: one 16-byte entry per symbol, kEncReplicas copies
        for (uint32_t s = tid; s < 256; s += blockDim.x) {
            const uint32_t f = ok ? s_cum[s + 1] - s_cum[s] : 0, cum = ok ? s_cum[s] : 0;
            uint4 x;
            if (CODER == RB200_CODER_ALIAS) {
                // a symbol outside the model: freq 1 keeps the step well defined, the flag reports it (as K4 stages it)
                const AliasEncEntry e = alias_enc_entry(f, cum);      // {magic, freq, cum, shift}
                x = f ? make_uint4(e.magic, e.freq, e.cum, e.shift) : make_uint4(0, 1, 0, kEncBadSymbol);
            } else if (CODER == RB200_CODER_BYTE) {
                const AliasEncEntry e = byte_enc_entry(f, cum, sb);   // {x_max, rcp_freq, bias, cmpl_freq | rcp_shift << 16}
                x = make_uint4(e.magic, e.freq, e.cum, e.shift);
            } else {
                uint32_t e[8];
                rans64_enc_entry(f, cum, sb, e);                      // {rcp_lo, rcp_hi, freq, bias}, {cmpl_freq, shift | bad}
                x = make_uint4(e[0], e[1], e[3], (e[4] & 0xfffffu) | ((e[5] & 63u) << 20) | (e[5] & kEncBadSymbol));
            }
#pragma unroll
            for (uint32_t r = 0; r < kEncReplicas; r++) s_tab[s * kEncReplicas + r] = x;
        }
        __syncthreads();
    }

    const uint32_t per_block = block_size / chunk_syms;
    if (warp >= per_block) return;
    const uint32_t chunk = blockIdx.x * per_block + warp;
    const uint8_t* src = blk + static_cast<uint64_t>(warp) * chunk_syms;
    const uint32_t tab = smem_addr(s_benc), wsm = tab + kEncTableBytes + warp * kEncWarpSmem;
    if (CODER == RB200_CODER_WORD && r32)
        encode_chunk_split(src, chunk_syms, chunk, WordEncoder<true>{tab}, wsm, scratch, slot_bytes, sizes, status);
    else if (CODER == RB200_CODER_WORD)
        encode_chunk_split(src, chunk_syms, chunk, WordEncoder<false>{tab}, wsm, scratch, slot_bytes, sizes, status);
    else if (CODER == RB200_CODER_ALIAS)
        encode_chunk_split(src, chunk_syms, chunk, AliasEncoder<true, SB>{tab, remap, sb}, wsm, scratch, slot_bytes, sizes, status);
    else if (CODER == RB200_CODER_BYTE)
        encode_chunk_split(src, chunk_syms, chunk, AliasEncoder<false, SB>{tab, 0, sb}, wsm, scratch, slot_bytes, sizes, status);
    else
        encode_chunk_split(src, chunk_syms, chunk, Rans64Encoder{tab, sb}, wsm, scratch, slot_bytes, sizes, status);
}

// GATED (rb200_container_blocks_model_encode_auto_async, with BUILD): runs only when the choice record (CoderChoice,
// device_utils.cuh) names `group`, and then at the record's scale_bits (the generic instances; the specialised ones are
// only ever named at their own).
// GEOM (rb200_container_blocks_model_encode_varlen_async, with GATED): on the grid of n_blocks_max, the CTAs at or past
// the record's count (BlocksVarlenGeom) exit at entry, as every CTA does when the plan failed (the count is then 0).
template <uint32_t CODER, uint32_t SB, bool BUILD, bool GATED = false, bool GEOM = false>
__global__ void __launch_bounds__(kMaxBlockWarps * 32)
block_coder_encode_kernel(const uint8_t* __restrict__ in, uint32_t block_size, uint16_t* __restrict__ block_freqs, uint32_t sb_rt,
                    uint32_t chunk_syms, uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint32_t* __restrict__ sizes,
                    uint32_t* __restrict__ status, const CoderChoice* __restrict__ choice, uint32_t group,
                    const BlocksVarlenGeom* __restrict__ geom)
{
    if ((GATED && choice->group != group) || (GEOM && blockIdx.x >= geom->n_blocks)) return;   // the group is the same for the whole grid
    block_coder_encode<CODER, SB, BUILD>(in, block_size, block_freqs, GATED ? choice->scale_bits : sb_rt, chunk_syms, scratch, slot_bytes,
                                         sizes, status);
}

// A block's decode table in shared memory at s_tab, from its cumulative frequencies (s_cum[257], M = 1 << sb): cum2sym[M],
// then the symbol entries.  Every thread of the CTA takes part; the caller synchronises before the table is read.
template <uint32_t CODER>
__device__ __forceinline__ void block_coder_decode_table(const uint32_t* s_cum, uint8_t* s_tab, uint32_t M)
{
    const uint32_t tid = threadIdx.x;
    // cum2sym, 4 slots (one u32) at a time: one binary search per 4 slots for the largest s with cum[s] <= slot, then a
    // walk that also steps over zero-width symbols; the cost per slot does not depend on how skewed the model is, and
    // consecutive threads store consecutive words
    uint32_t* c2s = reinterpret_cast<uint32_t*>(s_tab);
    for (uint32_t q = tid; q < M / 4; q += blockDim.x) {
        uint32_t lo = 0, hi = 256;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s_cum[mid] <= 4 * q) lo = mid; else hi = mid;
        }
        uint32_t packed = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            while (4 * q + k >= s_cum[lo + 1]) lo++;
            packed |= lo << (8 * k);
        }
        c2s[q] = packed;
    }
    if (CODER == RB200_CODER_BYTE) {
        uint32_t* syms = reinterpret_cast<uint32_t*>(s_tab + M);
        for (uint32_t s = tid; s < 256; s += blockDim.x) syms[s] = byte_dec_symbol(s_cum[s], s_cum[s + 1] - s_cum[s]);
    } else {
        uint2* syms = reinterpret_cast<uint2*>(s_tab + M);
        for (uint32_t i = tid; i < 256 * kRans64DecReplicas; i += blockDim.x) {
            const uint32_t s = i / kRans64DecReplicas;
            syms[i] = make_uint2(s_cum[s], s_cum[s + 1] - s_cum[s]);
        }
    }
}

// A block's alias decode table in shared memory at s_tab, from its cumulative frequencies (s_cum[257], M = 1 << sb): the
// pairing (block_alias_tables) in the table's place, each thread's bucket entries (at most 2: blockDim >= 128) in
// registers, then kAliasDecReplicas copies of the 256 entries over it (lean for SB > 8).  Every thread of the CTA takes
// part and gets the same result: false when the pairing fails (never for a table that sums to M), with nothing written
// over the pairing.  The caller synchronises before the table is read.
template <uint32_t SB>
__device__ __forceinline__ bool block_alias_decode_table(const uint32_t* s_cum, uint8_t* s_tab, uint32_t M)
{
    const uint32_t tid = threadIdx.x;
    const AliasBuildSmem& a = *reinterpret_cast<AliasBuildSmem*>(s_tab);
    if (!block_alias_tables(s_cum, M, *reinterpret_cast<AliasBuildSmem*>(s_tab))) return false;
    uint4 e[2];
#pragma unroll
    for (uint32_t i = 0; i < 2; i++) {
        const uint32_t b = tid + i * blockDim.x;
        if (b >= 256) continue;
        const AliasDecEntry d = alias_dec_entry(b, a.divider, a.slot_adjust, a.slot_freqs, a.sym_id);
        if (kAliasLean && SB > 8) e[i] = alias_lean_entry<(SB > 8 ? SB : 9)>(d, b);
        else e[i] = make_uint4(d.divider, d.alt0, d.alt1, d.adjust);
    }
    __syncthreads();
    uint4* s_dec = reinterpret_cast<uint4*>(s_tab);
#pragma unroll
    for (uint32_t i = 0; i < 2; i++) {
        const uint32_t b = tid + i * blockDim.x;
        if (b >= 256) continue;
#pragma unroll
        for (uint32_t r = 0; r < kAliasDecReplicas; r++) s_dec[b * kAliasDecReplicas + r] = e[i];
    }
    return true;
}

// A block's decode table in dynamic shared memory after the `warps` 1 KiB stream windows at s_dyn, from its model (freqs:
// 256 x u16, summing to M = 1 << sb), for block_decode_chunk:
// the word coder's slot table, with s_flag[1] set when one symbol takes all 4096 slots (the WIDE decoder); the alias
// coder's bucket entries; cum2sym and the symbol entries otherwise.  s_flag[0] is block_prefix's.  Every thread of the
// CTA takes part and gets the same result: false when the model does not sum to M (or, alias, does not pair), with no
// table built; true after a CTA barrier.
template <uint32_t CODER, uint32_t SB>
__device__ __forceinline__ bool block_decode_table(const uint16_t* freqs, uint32_t M, uint32_t* s_cum, uint32_t* s_flag, uint8_t* s_dyn,
                                                   uint32_t warps)
{
    if (CODER == RB200_CODER_WORD && threadIdx.x == 0) s_flag[1] = 0;
    if (!block_prefix(freqs, s_cum, &s_flag[0], M)) return false;
    uint8_t* s_tab = s_dyn + warps * kRingBytes;
    if (CODER == RB200_CODER_WORD)
        block_fill_slots(s_cum, reinterpret_cast<uint32_t*>(s_tab), &s_flag[1]);
    else if (CODER == RB200_CODER_ALIAS && !block_alias_decode_table<SB>(s_cum, s_tab, M))
        return false;
    else if (CODER != RB200_CODER_ALIAS)
        block_coder_decode_table<CODER>(s_cum, s_tab, M);
    __syncthreads();
    return true;
}

// One chunk of a block through the warp's 1 KiB stream window at shared address ring, on the table block_decode_table
// built at shared address tab; wide: its s_flag[1] (word coder only).
template <uint32_t CODER, uint32_t SB>
__device__ __forceinline__ void block_decode_chunk(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets,
                                                   uint32_t chunk, uint32_t ring, uint32_t tab, uint32_t sb, bool wide, uint8_t* __restrict__ dst,
                                                   uint32_t chunk_syms, uint32_t* __restrict__ status)
{
    const uint32_t lane = threadIdx.x & 31;
    if (CODER == RB200_CODER_WORD && wide)
        decode_window_chunk(WordDecoder<true>{tab, 0}, blob, blob_size, offsets, chunk, ring, dst, chunk_syms, status);
    else if (CODER == RB200_CODER_WORD)
        decode_window_chunk(WordDecoder<false>{tab, 0}, blob, blob_size, offsets, chunk, ring, dst, chunk_syms, status);
    else if (CODER == RB200_CODER_ALIAS)
        decode_window_chunk(AliasDecoder<SB, kAliasLean>{tab + (lane & (kAliasDecReplicas - 1)) * 16, sb}, blob, blob_size, offsets, chunk,
                            ring, dst, chunk_syms, status);
    else if (CODER == RB200_CODER_BYTE)
        decode_window_chunk(ByteDecoder<SB>{tab, sb}, blob, blob_size, offsets, chunk, ring, dst, chunk_syms, status);
    else
        decode_window_chunk(Rans64Decoder{tab, tab + (1u << sb) + (lane & (kRans64DecReplicas - 1)) * 8, sb}, blob, blob_size, offsets, chunk,
                            ring, dst, chunk_syms, status);
}

// K5: one CTA per block, launched by the host
template <uint32_t CODER, uint32_t SB>
__global__ void __launch_bounds__(kMaxBlockWarps * 32)
block_decode_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets,
                    const uint16_t* __restrict__ block_freqs, uint32_t sb_rt, uint32_t block_size, uint32_t chunk_syms,
                    uint8_t* __restrict__ out, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_bdec[];         // [warps x 1 KiB rings][the block's decode table]
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[2];                              // [0] bad model, [1] wide (word coder)
    const uint32_t sb = SB ? SB : sb_rt;
    const uint32_t tid = threadIdx.x, warp = tid >> 5, warps = blockDim.x >> 5;
    if (!block_decode_table<CODER, SB>(block_freqs + static_cast<uint64_t>(blockIdx.x) * 256, 1u << sb, s_cum, s_flag, s_bdec, warps)) {
        if (tid == 0) atomicOr(status, kStatStream);
        return;
    }
    const uint32_t per_block = block_size / chunk_syms;
    if (warp >= per_block) return;
    uint8_t* dst = out + static_cast<uint64_t>(blockIdx.x) * block_size + static_cast<uint64_t>(warp) * chunk_syms;
    block_decode_chunk<CODER, SB>(blob, blob_size, offsets, blockIdx.x * per_block + warp, smem_addr(s_bdec) + warp * kRingBytes,
                                  smem_addr_pinned(s_bdec + warps * kRingBytes), sb, CODER == RB200_CODER_WORD && s_flag[1], dst, chunk_syms,
                                  status);
}

// Every per-block instance, in the order of the planned decoders' ids (container_decoder): the word coder at scale_bits
// 12; the byte coder specialised for scale_bits 14 (main.cpp) and 12, generic otherwise, as K8; rans64 generic; the
// alias coder at the byte coder's scale_bits.
#define RB200_BLOCK_SB_DISPATCH(C, sb, CALL)                                             \
    if (sb == 14) {                                                                      \
        constexpr uint32_t CODER = C, SB = 14; CALL;                                     \
    } else if (sb == 12) {                                                               \
        constexpr uint32_t CODER = C, SB = 12; CALL;                                     \
    } else {                                                                             \
        constexpr uint32_t CODER = C, SB = 0; CALL;                                      \
    }
#define RB200_BLOCK_DISPATCH(coder, sb, CALL)                                            \
    if (coder == RB200_CODER_WORD) {                                                     \
        constexpr uint32_t CODER = RB200_CODER_WORD, SB = kWordScaleBits; CALL;          \
    } else if (coder == RB200_CODER_RANS64) {                                            \
        constexpr uint32_t CODER = RB200_CODER_RANS64, SB = 0; CALL;                     \
    } else if (coder == RB200_CODER_ALIAS) {                                             \
        RB200_BLOCK_SB_DISPATCH(RB200_CODER_ALIAS, sb, CALL)                             \
    } else {                                                                             \
        RB200_BLOCK_SB_DISPATCH(RB200_CODER_BYTE, sb, CALL)                              \
    }

// The split encoder instance of (CODER, SB): (BUILD, GATED, GEOM) = (build, 0, 0) for the fixed calls, (1, 1, 0) for the
// auto encode, (1, 1, 1) for the device-count encode.  The word coder has only (0, 0, 0), null for any other flags: its
// model-building encodes run K5f (plan_blocks_encode).
using BlockEncodeKernel = decltype(&block_coder_encode_kernel<RB200_CODER_BYTE, 0, false>);
template <uint32_t CODER, uint32_t SB>
inline BlockEncodeKernel block_encode_for(bool build, bool gated, bool geom)
{
    if constexpr (CODER == RB200_CODER_WORD) return build || gated || geom ? nullptr : block_coder_encode_kernel<CODER, SB, false>;
    else if (geom) return block_coder_encode_kernel<CODER, SB, true, true, true>;
    else if (gated) return block_coder_encode_kernel<CODER, SB, true, true>;
    else return build ? block_coder_encode_kernel<CODER, SB, true> : block_coder_encode_kernel<CODER, SB, false>;
}

template <uint32_t CODER, uint32_t SB>
inline void configure_block_coder()
{
    for (const BlockEncodeKernel k : {block_encode_for<CODER, SB>(true, false, false), block_encode_for<CODER, SB>(false, false, false),
                                      block_encode_for<CODER, SB>(true, true, false), block_encode_for<CODER, SB>(true, true, true)}) {
        if (!k) continue;
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             block_coder_encode_smem(CODER, kBlockCoderMaxScaleBits, kMaxBlockWarps * 32));
    }
    cudaFuncSetAttribute(block_decode_kernel<CODER, SB>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(block_decode_kernel<CODER, SB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         block_coder_decode_smem(CODER, kBlockCoderMaxScaleBits, kMaxBlockWarps * 32));
}

// every per-block kernel: the instances of RB200_BLOCK_DISPATCH and K5f's
inline void configure_block_kernels()
{
    configure_block_coder<RB200_CODER_WORD, kWordScaleBits>();
    configure_block_coder<RB200_CODER_BYTE, 14>();
    configure_block_coder<RB200_CODER_BYTE, 12>();
    configure_block_coder<RB200_CODER_BYTE, 0>();
    configure_block_coder<RB200_CODER_RANS64, 0>();
    configure_block_coder<RB200_CODER_ALIAS, 14>();
    configure_block_coder<RB200_CODER_ALIAS, 12>();
    configure_block_coder<RB200_CODER_ALIAS, 0>();
    for (const uint32_t threads : {8u * 32, 32u * 32})
        for (const BlockEncodeFusedKernel k : {block_encode_fused_for(true, false, false, threads), block_encode_fused_for(false, false, false, threads),
                                               block_encode_fused_for(true, true, false, threads), block_encode_fused_for(true, true, true, threads)}) {
            cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, block_encode_smem(threads));
        }
}

// one CTA per block of block_threads() threads; smem = block_coder_encode_smem(coder, sb, threads).  choice set: the
// GATED instance of (coder, sb)'s dispatch, with models built, where sb is the largest scale_bits of the launch group,
// which sizes the alias coder's remap, and the kernel takes the chosen one from the record; geom set as well: the GEOM
// instance, on a grid of n_blocks = n_blocks_max CTAs.
inline void launch_block_encode(cudaStream_t stream, uint32_t coder, uint32_t sb, bool build, uint32_t n_blocks, uint32_t threads,
                                uint32_t smem, const uint8_t* d_in, uint32_t block_size, uint16_t* d_freqs, uint32_t chunk_syms,
                                uint8_t* scratch, uint32_t slot_bytes, uint32_t* sizes, uint32_t* status,
                                const CoderChoice* choice = nullptr, uint32_t group = 0, const BlocksVarlenGeom* geom = nullptr)
{
    RB200_BLOCK_DISPATCH(coder, sb, (block_encode_for<CODER, SB>(build, choice != nullptr, geom != nullptr)
                                     <<<n_blocks, threads, smem, stream>>>(d_in, block_size, d_freqs, sb, chunk_syms, scratch, slot_bytes, sizes,
                                                                           status, choice, group, geom)))
}

inline void launch_block_decode(cudaStream_t stream, uint32_t coder, uint32_t sb, const uint8_t* blob, uint64_t blob_size,
                                const uint64_t* offsets, const uint16_t* d_freqs, uint32_t n_blocks, uint32_t block_size,
                                uint32_t chunk_syms, uint8_t* out, uint32_t* status)
{
    const uint32_t threads = block_threads(block_size, chunk_syms);
    const uint32_t smem = block_coder_decode_smem(coder, sb, threads);
    RB200_BLOCK_DISPATCH(coder, sb, (block_decode_kernel<CODER, SB><<<n_blocks, threads, smem, stream>>>(
                                        blob, blob_size, offsets, d_freqs, sb, block_size, chunk_syms, out, status)))
}

}  // namespace rb200

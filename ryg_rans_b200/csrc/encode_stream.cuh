// encode_stream.cuh -- the per-warp chunk encoder shared by every coder: one warp turns one chunk of symbols into one
// 32-way interleaved stream.
//
// Per warp: a 512 B input stage (16 steps of symbols, filled by one coalesced 128-bit load per lane issued a block
// ahead) and a 512 B output ring (emitted units are placed with ballot/popc compaction by the coder's step and flushed
// to the slot as whole 16-byte vectors).  The per-symbol parameters come from ONE conflict-free LDS.128: the 256-entry
// table is replicated 8x so that the 8 lanes of a quarter-warp always hit different 16-byte bank groups.
//
// A coder is a small value type that holds its operands (`tab`, the shared address of its 8x replicated table, and the
// slot remap or scale_bits where it needs them) and provides:
//   X                      state type (uint32_t or uint64_t)
//   kUnit                  renormalisation unit in bytes (1, 2 or 4)
//   kMaxEmit               most bytes one lane emits in one step
//   kBadBit                bit of EncState::flags that marks a symbol outside the model
//   kInit                  initial state
//   step<FULL>(st, sym, tab_lane, ring, gt, active)
//                          one encode step for the warp: renormalise (units placed in the ring below st.wpos, lanes
//                          31..0 downwards), then fold `sym` in; tab_lane = this lane's replica of the table.  FULL: all
//                          32 lanes take part (active == true); only the ragged first step of a chunk is not FULL.
#pragma once
#include <type_traits>

#include "device_utils.cuh"

namespace rb200 {

#ifndef RB200_ENC_UNIFORM_FLUSH
#define RB200_ENC_UNIFORM_FLUSH 1      // vote on the (warp-uniform) flush test so that ptxas emits a uniform branch
#endif
constexpr uint32_t kEncReplicas = 8;
constexpr uint32_t kEncStageBytes = 512;     // 16 steps x 32 symbols
constexpr uint32_t kEncRingBytes = 512;
constexpr uint32_t kEncTableBytes = 256 * kEncReplicas * 16;                 // 32 KiB
constexpr uint32_t kEncWarpSmem = kEncStageBytes + kEncRingBytes;            // 1 KiB per warp

template <class X>
struct EncState {
    X x;               // rANS state
    uint32_t wpos;     // un-wrapped ring position of the next unit = kEncRingBytes - kUnit - bytes_emitted
    uint32_t flags;    // OR of the table's flag words: the coder's kBadBit set <=> a symbol outside the model was met
};

// flush every complete 16-byte vector of the ring; *flushed = bytes already written below slot_end.
// KEEP: the destination is a scratch slot that is read back soon (fused paths): ask the L2 to hold on to it.
template <bool KEEP = false>
__device__ __forceinline__ void enc_flush(uint32_t produced, uint32_t& flushed, uint32_t ring, uint8_t* slot_end, uint32_t lane)
{
    const uint32_t nvec = (produced - flushed) >> 4;
    __syncwarp();
    if (lane < nvec) {
        const uint32_t v = (flushed >> 4) + lane + 1;                 // vector v ends 16 * (v - 1) bytes below slot_end
        const uint4 q = lds_u128(ring + ((0u - 16u * v) & (kEncRingBytes - 1)));
        if (KEEP) stg_hint_u128(reinterpret_cast<uint4*>(slot_end - 16ull * v), q, l2_policy_keep());
        else stg_stream_u128(reinterpret_cast<uint4*>(slot_end - 16ull * v), q);
    }
    flushed += nvec << 4;
    __syncwarp();
}

// one renormalisation unit from / to the ring
template <uint32_t U>
__device__ __forceinline__ uint32_t lds_unit(uint32_t addr)
{
    if constexpr (U == 1) return lds_u8(addr);
    else if constexpr (U == 2) return lds_u16(addr);
    else return lds_u32(addr);
}
template <uint32_t U>
__device__ __forceinline__ void sts_unit(uint32_t addr, uint32_t v)
{
    if constexpr (U == 1) sts_u8(addr, v);
    else if constexpr (U == 2) sts_u16(addr, v);
    else asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// Encode m symbols (one warp) as one 32-way stream that ENDS at slot_end (16-byte aligned) and grows
// downwards; returns the stream size in bytes (warp-uniform).
//   wsm  = shared address of this warp's 1 KiB (stage, then ring; 512-byte aligned)
//   KEEP = the slot is scratch that is read back soon (see enc_flush)
template <bool KEEP = false, class Coder>
__device__ __forceinline__ uint32_t encode_stream(const uint8_t* __restrict__ chunk_in, uint32_t m, const Coder coder, uint32_t wsm,
                                                  uint8_t* __restrict__ slot_end, uint32_t* __restrict__ status)
{
    constexpr uint32_t U = Coder::kUnit, S = sizeof(typename Coder::X);
    constexpr int kCheck = 256 / (32 * Coder::kMaxEmit);   // steps that emit at most 256 bytes: the ring is looked at after each group
    using Unit = std::conditional_t<U == 1, uint8_t, std::conditional_t<U == 2, uint16_t, uint32_t>>;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t stage = wsm, ring = wsm + kEncStageBytes;
    const uint32_t tab_lane = coder.tab + (lane & (kEncReplicas - 1)) * 16;     // this lane's replica of the table
    const uint32_t gt = lanemask_gt();

    EncState<typename Coder::X> st;
    st.x = Coder::kInit;                        // RansWordEncInit / RansEncInit / Rans64EncInit
    st.wpos = kEncRingBytes - U;
    st.flags = 0;
    uint32_t flushed = 0;
    const uint32_t steps = m >> 5, rem = m & 31;
    const uint32_t nblk = steps >> 4;           // full 16-step blocks, staged; the rest is read directly
    const bool vec_ok = (reinterpret_cast<uintptr_t>(chunk_in) & 15) == 0;

    // symbols are walked last to first (main_simd.cpp:294): ragged tail first
    uint4 parked = make_uint4(0, 0, 0, 0);
    if (nblk && vec_ok) parked = ldg_stream_u128(reinterpret_cast<const uint4*>(chunk_in + (nblk - 1) * kEncStageBytes) + lane);
    if (rem) {
        const bool active = lane < rem;
        const uint32_t s = active ? chunk_in[static_cast<uint64_t>(steps) * 32 + lane] : 0;
        coder.template step<false>(st, s, tab_lane, ring, gt, active);
    }
    for (uint32_t g = steps; g > nblk * 16; g--) {
        const uint32_t s = chunk_in[static_cast<uint64_t>(g - 1) * 32 + lane];
        coder.template step<true>(st, s, tab_lane, ring, gt, true);
        if (((g - 1) & (kCheck - 1)) == 0) enc_flush<KEEP>(kEncRingBytes - U - st.wpos, flushed, ring, slot_end, lane);
    }
    enc_flush<KEEP>(kEncRingBytes - U - st.wpos, flushed, ring, slot_end, lane);

    for (uint32_t b = nblk; b-- > 0;) {
        __syncwarp();
        if (vec_ok) {
            sts_u128(stage + lane * 16, parked);
            if (b) parked = ldg_stream_u128(reinterpret_cast<const uint4*>(chunk_in + (b - 1) * kEncStageBytes) + lane);
        } else {                                 // unaligned input: byte loads into the stage
            const uint8_t* p = chunk_in + b * kEncStageBytes + lane;
#pragma unroll
            for (int j = 0; j < 16; j++) sts_u8(stage + j * 32 + lane, p[j * 32]);
        }
        __syncwarp();
#pragma unroll
        for (int grp = 16 / kCheck - 1; grp >= 0; grp--) {
#pragma unroll
            for (int j = kCheck - 1; j >= 0; j--)
                coder.template step<true>(st, lds_u8(stage + (grp * kCheck + j) * 32 + lane), tab_lane, ring, gt, true);
            // <= 256 bytes per group; flushing whenever >= 256 are pending keeps the 512-byte ring safe.  The test is
            // warp-uniform; voting on it tells ptxas so (a uniform branch: no convergence check before the next ballot)
#if RB200_ENC_UNIFORM_FLUSH
            if (__any_sync(0xffffffffu, kEncRingBytes - U - st.wpos - flushed >= 256))
#else
            if (kEncRingBytes - U - st.wpos - flushed >= 256)
#endif
                enc_flush<KEEP>(kEncRingBytes - U - st.wpos, flushed, ring, slot_end, lane);
        }
    }

    // the final states for lanes 31..0 (RansWordEncFlush, main_simd.cpp:298-299; RansEncFlush, rans_byte.h:93-105;
    // Rans64EncFlush, rans64.h:96-103): lane 31's most significant unit is written first (highest address), lane 0's
    // least significant unit ends up first in memory.  < 16 bytes are pending, so the 32 x S header fits the ring.
    enc_flush<KEEP>(kEncRingBytes - U - st.wpos, flushed, ring, slot_end, lane);     // < 16 bytes stay pending
    const uint32_t hpos = st.wpos - S * (31 - lane);
#pragma unroll
    for (uint32_t j = 0; j < S / U; j++)
        sts_unit<U>(ring | ((hpos - U * j) & (kEncRingBytes - 1)), static_cast<uint32_t>(st.x >> (8 * (S - U * (j + 1)))));
    st.wpos -= 32 * S;
    const uint32_t produced = kEncRingBytes - U - st.wpos;           // total stream bytes
    enc_flush<KEEP>(produced, flushed, ring, slot_end, lane);
    const uint32_t left = produced - flushed;                        // < 16, whole units: head of the stream, not vector aligned
    if (U * lane < left) {
        const uint32_t off = flushed + U * lane + U;                 // bytes below slot_end
        *reinterpret_cast<Unit*>(slot_end - off) = static_cast<Unit>(lds_unit<U>(ring | ((0u - off) & (kEncRingBytes - 1))));
    }
    if (__any_sync(0xffffffffu, (st.flags & Coder::kBadBit) != 0) && lane == 0) atomicOr(status, kStatSymbol);
    return produced;
}

// The symbols of chunk `chunk` of in[0, n): in[first, first + m), m = chunk_syms except for a ragged last chunk.
struct ChunkRange {
    uint64_t first;
    uint32_t m;
};
__device__ __forceinline__ ChunkRange chunk_range(uint32_t chunk, uint32_t chunk_syms, uint64_t n)
{
    const uint64_t first = static_cast<uint64_t>(chunk) * chunk_syms;
    return {first, static_cast<uint32_t>(min(static_cast<uint64_t>(chunk_syms), n - first))};
}

// The split path's store (K6 compacts after it): encode chunk `chunk` (m symbols at chunk_in) into the end of its own
// worst-case slot of `scratch` and record its size in sizes[chunk].
template <class Coder>
__device__ __forceinline__ void encode_chunk_split(const uint8_t* __restrict__ chunk_in, uint32_t m, uint32_t chunk, const Coder coder,
                                                   uint32_t wsm, uint8_t* __restrict__ scratch, uint32_t slot_bytes,
                                                   uint32_t* __restrict__ sizes, uint32_t* __restrict__ status)
{
    const uint32_t produced = encode_stream(chunk_in, m, coder, wsm, scratch + static_cast<uint64_t>(chunk + 1) * slot_bytes, status);
    if ((threadIdx.x & 31) == 0) sizes[chunk] = produced;
}

}  // namespace rb200

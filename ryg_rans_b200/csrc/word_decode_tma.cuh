// word_decode_tma.cuh -- the word coder's decode steps (WordDecoder) and K1p: persistent 32-way word-coder decode with
// TMA-fed stream rings (sm_90a).  The chunk loops are decode_stream.cuh's.
//
// The step is RansSimdDecSym + RansSimdDecRenorm (rans_word_sse41.h:151-227) as one warp; the plumbing of K1p:
//   * persistent grid: CTAs stay resident, every warp pulls chunk ids from an atomic counter; the 16 KiB
//     RansWordTables image (rans_word_sse41.h:58-72, fused to one u32 per slot) is staged ONCE per CTA by one
//     cp.async.bulk (TMA 1-D bulk copy, SASS UBLKCP) completing on an mbarrier;
//   * the per-warp stream window is a ring of 512-byte units filled by cp.async.bulk straight from the blob:
//     no LDG -> register -> STS hop, no parked registers, no LSU wavefronts for refills.  One mbarrier per
//     ring slot; lane 0 arms it (arrive.expect_tx) and issues the copy, the warp waits with try_wait.parity
//     one unit before the cursor gets there;
//   * optional 64-byte mirror after the ring (a second small bulk copy of the unit that lands in slot 0), so
//     the per-step refill read needs no wrap mask;
//   * warp-uniform bookkeeping (cursor, fill state, loop control) is derived from shuffle-broadcast values so
//     ptxas keeps the control flow uniform (no BRA.DIV convergence checks in the hot loop).
//
// The policy struct carries the experiment switches of tools/decode_lab.cu (texture-pipe offload of every k-th
// table gather, ablations that remove one term of the step).  The shipped configuration is kDecShip below.
#pragma once
#include "decode_stream.cuh"
#include "device_utils.cuh"
#include "tables.h"
#include "word_kernels.cuh"

namespace rb200 {

__device__ __forceinline__ void mul_wide_u32(uint32_t a, uint32_t b, uint32_t& lo, uint32_t& hi)
{
    asm("{\n\t"
        ".reg .u64 t;\n\t"
        "mul.wide.u32 t, %2, %3;\n\t"
        "mov.b64 {%0, %1}, t;\n\t"
        "}"
        : "=r"(lo), "=r"(hi)
        : "r"(a), "r"(b));
}


// The word coder for the decode drivers (decode_stream.cuh): RansWordDecSym + RansWordDecRenorm for 32 lanes.
// tab = shared address of the packed table freq << 20 | bias << 8 | symbol (kept live in a register by the caller).
template <bool WIDE>
struct WordDecoder {
    using X = uint32_t;
    static constexpr uint32_t kHeaderBytes = rb200::kHeaderBytes, kUnit = 2, kMaxBytes = 2;
    static constexpr X kL = kWordL;                    // RansWordEncInit, rans_word_sse41.h:75-78
    uint32_t tab;
    cudaTextureObject_t tex;                           // the table as a texture (DecPolicy::kTexEvery), or 0

    // RansWordDecInit x 32 (rans_word_sse41.h:109-120): lane k's state is the k-th u32
    template <class At>
    __device__ __forceinline__ X read_header(At at, uint32_t lane) const
    {
        return lds_u16(at(4 * lane)) | (lds_u16(at(4 * lane + 2)) << 16);
    }

    __device__ __forceinline__ static uint32_t table_freq(uint32_t e)
    {
        uint32_t f = e >> 20;
        if (WIDE) f = f ? f : kWordSlots;   // single-symbol model: freq 4096 stored as 0
        return f;
    }

    // window step (decode_window_chunk)
    template <bool FULL>
    __device__ __forceinline__ void step(uint32_t& x, uint32_t& cursor, uint32_t ring, uint8_t* o, uint32_t lt, bool active) const
    {
        bool need = false;
        if (active) {
            const uint32_t e = lds_u32_ro(mad_u32(x & (kWordSlots - 1), 4u, tab));  // rans_word_sse41.h:126
            x = table_freq(e) * (x >> kWordScaleBits) + ((e >> 8) & 0xfffu);      // :129
            *o = static_cast<uint8_t>(e);                                       // :130
            need = x < kWordL;                                                  // :137
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, need);
        const uint32_t a = mad_u32(__popc(mask & lt), 2u, cursor);              // lane order within the step
        const uint32_t w = lds_u16(ring | (a & (kRingBytes - 1)));
        if (need) x = (x << 16) | w;                                            // :138
        cursor = mad_u32(__popc(mask), 2u, cursor);                             // :139
    }

    // persistent step (decode_persistent), rans_word_sse41.h:123-141.
    //   kWideMul: x * 2^20 as a 64-bit product gives q = x >> 12 in the high word and slot << 20 in the low one, from
    //   which ptxas forms the table address with ONE LEA.HI; e * 2^12 likewise gives freq in the high word and bias << 20
    //   in the low one.  Two IMAD.WIDE + one shift replace five shift/mask instructions (16 instead of 18 per step) --
    //   but they run on the FMA-heavy pipe, which the four IMADs of the step already load, and measured slower than the
    //   shift form (tools/decode_lab.cu); the shipped configuration uses shifts.
    template <class P>
    __device__ __forceinline__ void step_p(uint32_t& x, uint32_t& cur, uint8_t* o, uint32_t lt, uint32_t lane, int j, bool active) const
    {
        const bool via_tex = P::kTexEvery > 0 && j >= 0 && (j % (P::kTexEvery > 0 ? P::kTexEvery : 1)) == 0;
        if (active) {
            uint32_t q, f, b, e;
            if ((P::kWideMul & 1) && !via_tex) {
                uint32_t lo;
                mul_wide_u32(x, 1u << 20, lo, q);                                  // q = x >> 12, lo = (x & 4095) << 20
                if (P::kAblate & kAblGatherConflictFree) e = lds_u32_ro(mad_u32(lo >> 25, 128u, tab + lane * 4));   // bank = lane
                else e = lds_u32_ro(tab + (lo >> 18));                             // rans_word_sse41.h:126
            } else {
                uint32_t slot = x & (kWordSlots - 1);
                if (P::kAblate & kAblGatherConflictFree) slot = (x & 0xfe0u) | lane;
                q = x >> kWordScaleBits;
                if (via_tex) e = tex1Dfetch<unsigned int>(tex, static_cast<int>(slot));
                else e = lds_u32_ro(tab + slot * 4);
            }
            if (P::kWideMul & 2) {
                uint32_t lo;
                mul_wide_u32(e, 1u << 12, lo, f);                                  // f = e >> 20, lo = e << 12
                b = lo >> 20;
            } else {
                f = e >> 20;
                b = (e >> 8) & 0xfffu;
            }
            if (WIDE) f = f ? f : kWordSlots;                                      // single-symbol model: freq 4096 stored as 0
            x = mad_u32(f, q, b);                                                  // :129
            if (!(P::kAblate & kAblNoSymbolStore)) *o = static_cast<uint8_t>(e);   // :130
        }
        // RansWordDecRenorm for 32 lanes with ONE predicate feeding the vote and the merge (:134-141; the warp-wide form of
        // the movemask + pshufb compaction of RansSimdDecRenorm, :182-227): lane k takes the popc(mask & lanemask_lt)-th word.
        const uint32_t xr = active ? x : kWordL;                                   // an inactive lane never refills
        uint32_t xo = x;
        if (P::kAblate & kAblNoRingRead) {
            asm volatile(
                "{\n\t"
                ".reg .pred p;\n\t"
                ".reg .b32 m, r, a;\n\t"
                "setp.lt.u32 p, %2, 65536;\n\t"
                "vote.sync.ballot.b32 m, p, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "mad.lo.u32 a, r, 2, %1;\n\t"
                "and.b32 r, a, 0xffff;\n\t"
                "@p mad.lo.u32 %0, %0, 65536, r;\n\t"
                "popc.b32 m, m;\n\t"
                "mad.lo.u32 %1, m, 2, %1;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt));
        } else if (P::kIadd3) {
            asm volatile(
                "{\n\t"
                ".reg .pred p;\n\t"
                ".reg .b32 m, r, a;\n\t"
                ".reg .b16 h;\n\t"
                "setp.lt.u32 p, %2, 65536;\n\t"
                "vote.sync.ballot.b32 m, p, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, r, r;\n\t"
                "add.u32 a, a, %1;\n\t"
                "ld.shared.u16 h, [a];\n\t"
                "cvt.u32.u16 r, h;\n\t"
                "@p mad.lo.u32 %0, %0, 65536, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt));
        } else {
            asm volatile(
                "{\n\t"
                ".reg .pred p;\n\t"
                ".reg .b32 m, r, a;\n\t"
                ".reg .b16 h;\n\t"
                "setp.lt.u32 p, %2, 65536;\n\t"
                "vote.sync.ballot.b32 m, p, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "mad.lo.u32 a, r, 2, %1;\n\t"
                "ld.shared.u16 h, [a];\n\t"
                "cvt.u32.u16 r, h;\n\t"
                "@p mad.lo.u32 %0, %0, 65536, r;\n\t"
                "popc.b32 m, m;\n\t"
                "mad.lo.u32 %1, m, 2, %1;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt));
        }
        x = xo;
    }
};

template <class P, bool WIDE>
__global__ void __launch_bounds__(P::kWarps * 32, P::kMinBlocks)
word_decode_tma_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets,
                       const uint32_t* __restrict__ g_table, uint8_t* __restrict__ out, uint64_t n, uint32_t chunk_syms,
                       uint32_t n_chunks, DecodeWork* __restrict__ work, uint32_t* __restrict__ status, cudaTextureObject_t tex)
{
    extern __shared__ __align__(1024) uint8_t s_dec[];     // [16 KiB table][table mbarrier][kWarps x (ring, mirror, mbarriers)]
    const uint32_t tab = smem_addr_pinned(s_dec);
    const uint32_t bar_tab = tab + kWordSlots * 4;
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);       // warp-uniform for ptxas
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t ring = tab + P::kWarpsOff + warp * P::kWarpStride;

    if (threadIdx.x == 0) mbar_init(bar_tab, 1);
    if (lane == 0 && P::kRefill == kRefillTma)
        for (uint32_t j = 0; j < kTmaUnits; j++) mbar_init(ring + P::kBarsOff + 8 * j, 1);
    mbar_fence_init();
    __syncthreads();
    if (threadIdx.x == 0) {                                // RansWordTables for the whole CTA: one 16 KiB bulk copy
        mbar_arrive_expect_tx(bar_tab, kWordSlots * 4);
        bulk_g2s(tab, g_table, kWordSlots * 4, bar_tab);
    }
    {
        uint32_t spins = 0;
        while (!mbar_try_wait(bar_tab, 0))
            if (++spins > kTmaSpinLimit) {
                if (threadIdx.x == 0) atomicOr(status, kStatStall);
                return;
            }
    }
    __syncwarp();
    decode_persistent<P>(WordDecoder<WIDE>{tab, tex}, ring, blob, blob_size, offsets, out, n, chunk_syms, n_chunks, work, lane, status);
}

// The configuration the C-ABI launches (tools/decode_lab.cu measures the alternatives):
// 2 CTAs of 32 warps per SM, fill check / ring wrap every 8 steps, ring of 4 x 512 B filled by cp.async (LDGSTS),
// table by one TMA bulk copy, freq / bias by one IMAD.WIDE, slot and x >> 12 by shift / mask.
using DecShip = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, 0, false>;

inline void configure_word_decode_tma()
{
    cudaFuncSetAttribute(word_decode_tma_kernel<DecShip, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_decode_tma_kernel<DecShip, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DecShip::kSmemBytes);
    cudaFuncSetAttribute(word_decode_tma_kernel<DecShip, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(word_decode_tma_kernel<DecShip, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DecShip::kSmemBytes);
}

}  // namespace rb200

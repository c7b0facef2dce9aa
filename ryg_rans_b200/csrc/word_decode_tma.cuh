// word_decode_tma.cuh -- K1p: persistent 32-way word-coder decode with TMA-fed stream rings (sm_90a).
//
// Same decode step as word_kernels.cuh (RansSimdDecSym + RansSimdDecRenorm, rans_word_sse41.h:151-227, as one
// warp), different plumbing:
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
#include "device_utils.cuh"
#include "tables.h"
#include "word_kernels.cuh"

namespace rb200 {

// ---------------------------------------------------------------------------
// mbarrier + bulk-copy primitives (PTX ISA 8.x, sm_90+)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok;
}
// global -> shared bulk copy; bytes is a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}

// the two words of per-launch work state (zero between launches: the last warp out resets them)
struct DecodeWork {
    uint32_t next_chunk;
    uint32_t warps_done;
};

constexpr uint32_t kTmaUnits = 4;                  // ring slots per warp
constexpr uint32_t kTmaSpinLimit = 1u << 20;       // a bug must not hang the GPU
constexpr uint32_t kTmaSeqBase = 1u << 12;         // first unit sequence number (a multiple of 2 * kTmaUnits: parity 0)

// ablation bits (tools/decode_lab.cu): each removes ONE term of the step; the output is then garbage
constexpr int kAblGatherConflictFree = 1;   // gather address forced to bank = lane: same instructions + 1, no bank conflicts
constexpr int kAblNoSymbolStore = 2;        // drop the STG.U8
constexpr int kAblNoRingRead = 4;           // refill word = the address instead of LDS.U16 [address]
constexpr int kAblNoRefill = 8;             // never wait for / issue ring units

// how ring units are fetched
constexpr int kRefillTma = 0;       // cp.async.bulk (UBLKCP) by one elected lane, mbarrier per slot
constexpr int kRefillCpAsync = 1;   // cp.async.cg 16 bytes per lane (LDGSTS), commit/wait groups

template <int kWarps_, int kMinBlocks_, int kGroup_, int kRefill_ = kRefillTma, int kUnitLog_ = 9, int kWideMul_ = 0, int kTexEvery_ = 0,
          int kAblate_ = 0, bool kIadd3_ = false, uint32_t kTableBytes_ = kWordSlots * 4>
struct DecPolicy {
    static constexpr uint32_t kTableBytes = kTableBytes_;   // decode table at the start of the CTA's shared memory
    static constexpr bool kIadd3 = kIadd3_;           // refill address / cursor update as cur + r + r (IADD3, ALU pipe) instead of IMAD
    static constexpr int kWarps = kWarps_;            // warps per CTA
    static constexpr int kMinBlocks = kMinBlocks_;    // CTAs per SM the register budget is sized for
    static constexpr int kGroup = kGroup_;            // steps between two fill checks / ring wraps (<= 8)
    static constexpr int kRefill = kRefill_;
    static constexpr int kWideMul = kWideMul_;        // field extraction by IMAD.WIDE: bit 0 for the state, bit 1 for the table entry
    static constexpr int kTexEvery = kTexEvery_;      // 0: every gather from shared memory; k: every k-th through the TEX pipe
    static constexpr int kAblate = kAblate_;
    static constexpr uint32_t kUnit = 1u << kUnitLog_;                    // bytes per ring unit (512 or 1024)
    static constexpr uint32_t kRing = kTmaUnits * kUnit;
    static constexpr uint32_t kNeed = kGroup_ * 64 + 62;                  // bytes a group may touch from its first cursor
    static constexpr uint32_t kMirror = (kNeed + 15u) & ~15u;             // copy of the ring's first bytes behind its end
    static constexpr uint32_t kBarsOff = kRing + kMirror;                 // per warp: [ring][mirror][kTmaUnits mbarriers]
    static constexpr uint32_t kWarpStride = kBarsOff + 8 * kTmaUnits;
    static constexpr uint32_t kWarpsOff = kTableBytes_ + 16;              // [table][table mbarrier]
    static constexpr uint32_t kSmemBytes = kWarpsOff + kWarps_ * kWarpStride;
    static_assert(kGroup_ >= 1 && kGroup_ * 64 <= 512, "one advance per group must be enough");
    static_assert(kNeed <= (kTmaUnits - 2) * kUnit + 2, "a group must fit between the cursor's unit and the slot being refilled");
    static_assert(kWarpStride % 16 == 0, "bulk-copy destinations are 16-byte aligned");
};

// Per-warp decode cursor + fill state.  Every member is warp-uniform (except src in cp.async mode: + 16 * lane).
//   pos = cur + (seq_ready * kUnit - kNeed - limit) is the ring-linear (never wrapping) byte position of the cursor;
//   pos / kUnit is the sequence
//   number of the unit under it; sequence number s lives in slot s % 4 and its mbarrier completes phase s / 4.
//   cur itself is a shared-memory ADDRESS inside [ring, ring + kRing) at the start of a group and may run up to kNeed
//   bytes past the ring's end during one (the mirror holds a copy of the ring's first kMirror bytes there).
//   Units below seq_ready have landed; unit seq_ready is in flight (issued), nothing beyond it is.
struct TmaWindow {
    uint32_t ring;         // shared address of the ring
    uint32_t cur;          // shared address the next refill word is read from
    uint32_t limit;        // the fast-path test "pos + kNeed > seq_ready * kUnit" as "cur > limit"
    uint32_t seq_ready;
    uint32_t end_pos;      // ring-linear position of the stream's (16-byte aligned) end
    uint64_t src;          // global address of ring-linear position 0: unit s is fetched from src + kUnit * s
};

// Fetch unit `seq` of the current stream into its slot (and its share of the mirror).  The chunk's last unit is cut
// at the stream end (a multiple of 16), so no copy ever reads past the blob.
//   TMA: one elected lane arms the slot's mbarrier with the byte count and issues the bulk copies.
//   cp.async: lane k copies bytes [16k, 16k + 16) of every 512; the caller commits the group.
template <class P>
__device__ __forceinline__ void tma_issue(const TmaWindow& w, uint32_t seq, uint32_t lane)
{
    const uint32_t slot = seq & (kTmaUnits - 1);
    const uint32_t dst = w.ring + slot * P::kUnit;
    const uint64_t src = w.src + static_cast<uint64_t>(seq) * P::kUnit;
    // The slot was last read (by other lanes too) more than a unit ago; the warp-level fence makes that ordering formal
    // for the asynchronous writes that follow (compute-sanitizer racecheck is clean with it).
    __syncwarp();
    if (P::kRefill == kRefillCpAsync) {
#pragma unroll
        for (uint32_t part = 0; part < P::kUnit; part += 512) {
            const uint32_t in_unit = part + lane * 16;
            const bool live = seq * P::kUnit + in_unit < w.end_pos;
            if (live) {
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + in_unit), "l"(src + part) : "memory");
                if (slot * P::kUnit + in_unit < P::kMirror)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + in_unit + P::kRing), "l"(src + part) : "memory");
            }
        }
        return;
    }
    const uint32_t bar = w.ring + P::kBarsOff + slot * 8;
    uint32_t bytes = P::kUnit;
    if (seq * P::kUnit + P::kUnit > w.end_pos) bytes = ((w.end_pos - 1) & (P::kUnit - 1)) + 1;
    uint32_t mir = 0;                                                       // this unit's share of the mirror
    if (slot == 0) mir = P::kMirror < P::kUnit ? P::kMirror : P::kUnit;
    if (slot == 1 && P::kMirror > P::kUnit) mir = P::kMirror - P::kUnit;
    mir = mir < bytes ? mir : bytes;
    asm volatile(
        "{\n\t"
        ".reg .pred p, q;\n\t"
        ".reg .b32 t;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "setp.ne.and.u32 q, %4, 0, p;\n\t"
        "add.u32 t, %3, %4;\n\t"
        "@p mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], t;\n\t"
        "@p cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%1], [%2], %3, [%0];\n\t"
        "@q cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%5], [%2], %4, [%0];\n\t"
        "}"
        :
        : "r"(bar), "r"(dst), "l"(src), "r"(bytes), "r"(mir), "r"(dst + P::kRing)
        : "memory");
}

// wait for unit `seq`; false if the copy never lands (cannot happen for in-bounds copies)
template <class P>
__device__ __forceinline__ bool tma_wait(const TmaWindow& w, uint32_t seq)
{
    const uint32_t bar = w.ring + P::kBarsOff + (seq & (kTmaUnits - 1)) * 8;
    const uint32_t parity = (seq / kTmaUnits) & 1;
    if (mbar_try_wait(bar, parity)) return true;
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity))
        if (++spins > kTmaSpinLimit) return false;
    return true;
}

// One unit further (the slow path of a fill check, about once per kUnit consumed bytes): issue unit seq_ready + 1 --
// its slot held unit seq_ready - 3, which lies wholly behind the cursor whenever the check fires -- then wait for
// unit seq_ready.  Past the end of the stream nothing is issued or waited for; the counters move on all the same, so
// a corrupt stream that overruns reads stale ring bytes (never out of bounds) and is caught by the end-of-chunk check.
template <class P>
__device__ __forceinline__ void tma_advance(TmaWindow& w, uint32_t lane, uint32_t* __restrict__ status)
{
    const uint32_t seq_end = (w.end_pos + P::kUnit - 1) / P::kUnit;
    if (w.seq_ready + 1 < seq_end) tma_issue<P>(w, w.seq_ready + 1, lane);
    if (P::kRefill == kRefillCpAsync) {
        asm volatile("cp.async.commit_group;" ::: "memory");       // an empty group past the end keeps the count uniform
        asm volatile("cp.async.wait_group 1;" ::: "memory");       // everything but the unit just issued has landed
        __syncwarp();
    } else if (w.seq_ready < seq_end && !tma_wait<P>(w, w.seq_ready)) {
        if (lane == 0) atomicOr(status, kStatStall);
        w.end_pos = 0;                                                      // sticky: no more issues or waits
    }
    w.seq_ready++;
    w.limit += P::kUnit;
}

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

// One decode step for the whole warp: RansWordDecSym + RansWordDecRenorm (rans_word_sse41.h:123-141).
//   tab = shared address of the packed table freq << 20 | bias << 8 | symbol.
//   kWideMul: x * 2^20 as a 64-bit product gives q = x >> 12 in the high word and slot << 20 in the low one, from which
//   ptxas forms the table address with ONE LEA.HI; e * 2^12 likewise gives freq in the high word and bias << 20 in the
//   low one.  Two IMAD.WIDE + one shift replace five shift/mask instructions (16 instead of 18 per step) -- but they run
//   on the FMA-heavy pipe, which the four IMADs of the step already load, and measured slower than the shift form
//   (tools/decode_lab.cu); the shipped configuration uses shifts.
template <class P, bool WIDE>
__device__ __forceinline__ void tma_dec_step(uint32_t& x, uint32_t& cur, uint32_t tab, uint8_t* o, uint32_t lt, uint32_t lane,
                                             cudaTextureObject_t tex, bool via_tex, bool active)
{
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

    TmaWindow win;
    win.ring = tab + P::kWarpsOff + warp * P::kWarpStride;
    win.seq_ready = kTmaSeqBase;

    if (threadIdx.x == 0) mbar_init(bar_tab, 1);
    if (lane == 0 && P::kRefill == kRefillTma)
        for (uint32_t j = 0; j < kTmaUnits; j++) mbar_init(win.ring + P::kBarsOff + 8 * j, 1);
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

    const uint32_t lt = lanemask_lt();
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(&work->next_chunk, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= n_chunks) break;

        const uint64_t first = static_cast<uint64_t>(chunk) * chunk_syms;
        const uint64_t left = n - first;
        const uint32_t m = left < chunk_syms ? static_cast<uint32_t>(left) : chunk_syms;
        const uint64_t off = offsets[chunk];
        const uint64_t end = offsets[chunk + 1] & ~static_cast<uint64_t>(15);
        const bool dir_bad = (off & 1) || off + kHeaderBytes > end || end > blob_size || end - off > (1u << 30);   // not trusted
        if (__shfl_sync(0xffffffffu, dir_bad ? 1u : 0u, 0)) {
            if (lane == 0) atomicOr(status, kStatStream);
            continue;
        }
        // warp-uniform geometry of this chunk's stream; nothing is in flight and every slot is free here
        const uint32_t off_in = __shfl_sync(0xffffffffu, static_cast<uint32_t>(off % P::kUnit), 0);
        const uint32_t len = __shfl_sync(0xffffffffu, static_cast<uint32_t>(end - off), 0);
        const uint32_t seq0 = win.seq_ready;
        const uint32_t pos0 = seq0 * P::kUnit + off_in;                         // ring-linear position of the stream start
        win.end_pos = pos0 + len;
        win.src = reinterpret_cast<uint64_t>(blob) + (off - off_in) - static_cast<uint64_t>(seq0) * P::kUnit;
        if (P::kRefill == kRefillCpAsync) win.src += lane * 16;
        win.cur = win.ring + (pos0 & (P::kRing - 1));
        win.limit = win.cur - off_in - P::kNeed;                                // pos0 + kNeed > seq0 * kUnit as cur > limit
        if (!(P::kAblate & kAblNoRefill)) {
            tma_issue<P>(win, seq0, lane);
            if (P::kRefill == kRefillCpAsync) asm volatile("cp.async.commit_group;" ::: "memory");
            while (win.cur > win.limit) tma_advance<P>(win, lane, status);      // header + first group: two or three units
        }
        __syncwarp();

        // RansWordDecInit x 32 (rans_word_sse41.h:109-120): lane k's state is the k-th u32; the mirror covers a wrap
        uint32_t x = lds_u16(win.cur + 4 * lane) | (lds_u16(win.cur + 4 * lane + 2) << 16);
        win.cur += kHeaderBytes;

        uint8_t* o = out + first + lane;
        const uint32_t ring_end = win.ring + P::kRing;
        // kGroup steps: wrap (the mirror absorbed the previous group's overrun), fill check, steps
        auto group = [&](uint8_t* og) {
            if (win.cur >= ring_end) {
                win.cur -= P::kRing;
                win.limit -= P::kRing;
            }
            if (!(P::kAblate & kAblNoRefill) && __any_sync(0xffffffffu, win.cur > win.limit)) tma_advance<P>(win, lane, status);
#pragma unroll
            for (int j = 0; j < P::kGroup; j++)
                tma_dec_step<P, WIDE>(x, win.cur, tab, og + 32 * j, lt, lane, tex,
                                      P::kTexEvery > 0 && (j % (P::kTexEvery > 0 ? P::kTexEvery : 1)) == 0, true);
        };
        uint32_t todo = m >> 5;                                                 // full steps left
        for (; todo >= 2 * P::kGroup; todo -= 2 * P::kGroup) {
            group(o);
            group(o + 32 * P::kGroup);
            o += 64 * P::kGroup;
        }
        if (todo >= P::kGroup) {
            group(o);
            o += 32 * P::kGroup;
            todo -= P::kGroup;
        }
        // tail: fewer than kGroup steps and the ragged last one; together they touch less than kNeed bytes
        if (win.cur >= ring_end) {
            win.cur -= P::kRing;
            win.limit -= P::kRing;
        }
        if (!(P::kAblate & kAblNoRefill) && __any_sync(0xffffffffu, win.cur > win.limit)) tma_advance<P>(win, lane, status);
        for (; todo; todo--) {
            tma_dec_step<P, WIDE>(x, win.cur, tab, o, lt, lane, tex, false, true);
            o += 32;
        }
        if (m & 31) tma_dec_step<P, WIDE>(x, win.cur, tab, o, lt, lane, tex, false, lane < (m & 31));   // main_simd.cpp:328-332

        // A valid stream is consumed exactly to its (aligned) end and leaves every lane in the encoder's initial state.
        const uint32_t pos = win.cur + (win.seq_ready * P::kUnit - P::kNeed - win.limit);
        const bool bad = (pos != pos0 + len) || (x != kWordL);
        if (!P::kAblate && __any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, kStatStream);
        // drain: at most unit seq_ready is still in flight (a stream that stopped short); the next chunk starts
        // behind the last unit that was issued, so sequence numbers stay gap-free
        if (!(P::kAblate & kAblNoRefill)) {
            const uint32_t seq_end = (win.end_pos + P::kUnit - 1) / P::kUnit;
            if (P::kRefill == kRefillCpAsync) asm volatile("cp.async.wait_group 0;" ::: "memory");
            if (win.seq_ready < seq_end) {
                if (P::kRefill == kRefillTma) tma_wait<P>(win, win.seq_ready);
                win.seq_ready++;
            } else {
                win.seq_ready = seq_end;
            }
        }
        __syncwarp();
    }

    // last warp out re-arms the work state for the next launch
    if (lane == 0) {
        const uint32_t total = gridDim.x * P::kWarps;
        if (atomicAdd(&work->warps_done, 1u) == total - 1) {
            work->next_chunk = 0;
            work->warps_done = 0;
        }
    }
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

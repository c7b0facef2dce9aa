// decode_stream.cuh -- the per-warp chunk decoder shared by every coder: one warp turns one 32-way interleaved stream
// back into one chunk of symbols.
//
// Two stream windows, each with its own driver:
//   StreamWindow + decode_window_chunk     a 1 KiB shared-memory ring per warp, refilled by LDG -> STS one unit ahead;
//                                          one chunk per warp of the grid (per-block, byte and rans64 decoders)
//   TmaWindow + decode_persistent<P>       a ring of 512-byte units filled by cp.async or cp.async.bulk, with a mirror
//                                          behind its end so that reads need no wrap mask; persistent warps pull chunk ids
//                                          from a DecodeWork counter (word and alias decoders)
// Both drivers own the directory check, the window set-up, the header read, the stepping with its refills, the ragged
// last step and the end-of-stream check: a valid stream is consumed exactly to its (16-byte aligned) end and leaves
// every lane in the encoder's initial state.
//
// A coder is a small value type that holds its table addresses and provides:
//   X                      state type (uint32_t or uint64_t)
//   kHeaderBytes           bytes of the 32 lanes' final states at the stream start
//   kUnit                  renormalisation unit in bytes: a stream starts at a multiple of it
//   kL                     the state every lane ends in (the encoder's initial state)
//   kMaxBytes              most bytes one lane reads in one step
//   read_header(at, lane)  lane's initial state; at(b) = shared address of header byte b
//   step<FULL>(x, cursor, ring, o, lt, active)
//                          window step: one decode step for the warp, reads the ring at (cursor & (kRingBytes - 1));
//                          FULL: all 32 lanes take part (active == true), only the ragged last step is not FULL
//   step_p<P>(x, cur, o, lt, lane, j, active)
//                          persistent step: reads the ring at the shared address cur; j = index within the group
//                          (-1 for the tail steps, which never use the texture pipe)
#pragma once
#include "device_utils.cuh"
#include "tables.h"

namespace rb200 {

__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// The directory is not trusted: a stream must start on a unit, hold its header, end inside the blob and be shorter
// than 2^30 bytes (no encoder writes one of more than 512 + 2 * 2^24), so that 32-bit stream positions cannot wrap.
template <class C>
__device__ __forceinline__ bool dir_entry_bad(uint64_t off, uint64_t end, uint64_t blob_size)
{
    return (off & (C::kUnit - 1)) || off + C::kHeaderBytes > end || end > blob_size || end - off > (1u << 30);
}

// ---------------------------------------------------------------------------
// Per-warp stream window: a 1 KiB shared-memory ring over the compressed stream,
// refilled 512 B at a time with one coalesced 128-bit load per lane.  The load for
// the next unit is issued one refill ahead and parked in registers, so its HBM
// latency is hidden behind >= 8 decode steps.  The cursor never leaves the ring,
// which also bounds every read a corrupt stream could cause.
// ---------------------------------------------------------------------------
constexpr uint32_t kRingBytes = 1024;
constexpr uint32_t kUnitBytes = 512;

struct StreamWindow {
    uint32_t ring;          // shared-space address of this warp's ring, 1 KiB aligned
    uint32_t fill_end;      // low 32 bits of the absolute blob byte offset filled so far
    uint32_t next_vec;      // this lane's 16-byte vector of the next unit to fetch (index into the blob)
    uint32_t limit_vec;     // blob_size / 16 (the C-ABI rejects blobs of 64 GiB and more)
    const uint4* base;      // blob, warp-uniform
    uint4 parked;           // unit in flight

    // Past the end of the blob the last vector is fetched again instead: what lies beyond a stream's
    // own end is never consumed by a valid stream, and a corrupt one may read any in-bounds bytes.
    __device__ __forceinline__ uint4 fetch()
    {
        const uint4 v = ldg_stream_u128(base + min(next_vec, limit_vec - 1));
        next_vec += 32;
        return v;
    }

    // off = absolute byte offset of the stream start inside the blob
    __device__ __forceinline__ void open(const uint8_t* blob, uint64_t blob_size, uint64_t off, uint32_t ring_addr, uint32_t lane)
    {
        ring = ring_addr;
        base = reinterpret_cast<const uint4*>(blob);
        const uint32_t unit0 = static_cast<uint32_t>(off / kUnitBytes);
        next_vec = unit0 * 32 + lane;
        limit_vec = static_cast<uint32_t>(blob_size / 16);
        uint4 a = fetch();
        uint4 b = fetch();
        parked = fetch();
        sts_u128(ring + ((unit0 & 1) * kUnitBytes) + lane * 16, a);
        sts_u128(ring + (((unit0 + 1) & 1) * kUnitBytes) + lane * 16, b);
        fill_end = (unit0 + 2) * kUnitBytes;
        __syncwarp();
    }

    // Call before every run of steps that consumes at most 256 bytes.
    __device__ __forceinline__ void top_up(uint32_t cursor, uint32_t lane)
    {
        if (fill_end - cursor <= kUnitBytes) {          // warp-uniform
            __syncwarp();
            sts_u128(ring + (fill_end & kUnitBytes) + lane * 16, parked);
            fill_end += kUnitBytes;
            parked = fetch();
            __syncwarp();
        }
    }
};

// Decode chunk `chunk` (one warp) into chunk_out[0, m); ring = shared address of this warp's 1 KiB window.
template <class C>
__device__ __forceinline__ void decode_window_chunk(const C& coder, const uint8_t* __restrict__ blob, uint64_t blob_size,
                                                    const uint64_t* __restrict__ offsets, uint32_t chunk, uint32_t ring,
                                                    uint8_t* __restrict__ chunk_out, uint32_t m, uint32_t* __restrict__ status)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t off = offsets[chunk];
    const uint64_t end = offsets[chunk + 1] & ~static_cast<uint64_t>(15);
    if (dir_entry_bad<C>(off, end, blob_size)) {
        if (lane == 0) atomicOr(status, kStatStream);
        return;
    }

    StreamWindow win;
    win.open(blob, blob_size, off, ring, lane);
    uint32_t cursor = static_cast<uint32_t>(off);
    typename C::X x = coder.read_header([&](uint32_t b) { return win.ring | ((cursor + b) & (kRingBytes - 1)); }, lane);
    cursor += C::kHeaderBytes;

    constexpr uint32_t kRun = 256 / (32 * C::kMaxBytes);       // steps per top_up
    static_assert(kRun >= 1, "a step must read at most 256 bytes for the warp");
    const uint32_t lt = lanemask_lt();
    uint8_t* o = chunk_out + lane;
    const uint32_t steps = m >> 5, rem = m & 31;
    uint32_t g = 0;
    for (; g + 2 * kRun <= steps; g += 2 * kRun) {
        win.top_up(cursor, lane);
#pragma unroll
        for (uint32_t j = 0; j < kRun; j++) coder.template step<true>(x, cursor, win.ring, o + 32 * j, lt, true);
        win.top_up(cursor, lane);
#pragma unroll
        for (uint32_t j = kRun; j < 2 * kRun; j++) coder.template step<true>(x, cursor, win.ring, o + 32 * j, lt, true);
        o += 64 * kRun;
    }
    if (g + kRun <= steps) {
        win.top_up(cursor, lane);
#pragma unroll
        for (uint32_t j = 0; j < kRun; j++) coder.template step<true>(x, cursor, win.ring, o + 32 * j, lt, true);
        o += 32 * kRun;
        g += kRun;
    }
    win.top_up(cursor, lane);                                    // the last < kRun steps and the ragged one
    for (; g < steps; g++) {
        coder.template step<true>(x, cursor, win.ring, o, lt, true);
        o += 32;
    }
    if (rem) coder.template step<false>(x, cursor, win.ring, o, lt, lane < rem);

    const bool bad = (cursor != static_cast<uint32_t>(end)) || (x != C::kL);
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, kStatStream);
}

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
          int kAblate_ = 0, bool kIadd3_ = false, uint32_t kTableBytes_ = 4096 * 4>   // default: the word coder's 16 KiB table
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

// One stored chunk, one warp (block_decode_planned_kernel's stored blocks, the version 6 decoders' stored chunks):
// chunk_syms symbols from src (16-byte aligned: a stored stream starts a vector) to dst, with 16-byte loads; whole
// 16-byte stores where dst and the length allow them, bytes otherwise.
__device__ __forceinline__ void block_copy_stored(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t chunk_syms, uint32_t lane)
{
    const bool vec = ((reinterpret_cast<uintptr_t>(dst) | chunk_syms) & 15) == 0;
    for (uint32_t v = lane; v < (chunk_syms + 15) / 16; v += 32) {
        const uint4 q = ldg_stream_u128(reinterpret_cast<const uint4*>(src) + v);
        if (vec) {
            stg_stream_u128(reinterpret_cast<uint4*>(dst) + v, q);
        } else {
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (uint32_t j = 0; j < 16; j++)
                if (16 * v + j < chunk_syms) dst[16 * v + j] = static_cast<uint8_t>(w[j >> 2] >> (8 * (j & 3)));
        }
    }
}

// The persistent chunk loop of one warp: pull chunk ids from work->next_chunk until none is left, decode each into
// out[chunk * chunk_syms, ...) through the warp's TmaWindow at shared address `ring`; the last warp out re-arms `work`
// for the next launch.  With kRefillTma the caller has initialised the ring's mbarriers behind a CTA barrier.
// STORED (the version 6 decoders): a chunk whose bit is set in stored_bits is copied from blob + offsets[chunk]
// (block_copy_stored; the container's checks saw its step and padding), with no window set-up.
template <class P, bool STORED = false, class C>
__device__ __forceinline__ void decode_persistent(const C& coder, uint32_t ring, const uint8_t* __restrict__ blob, uint64_t blob_size,
                                                  const uint64_t* __restrict__ offsets, uint8_t* __restrict__ out, uint64_t n,
                                                  uint32_t chunk_syms, uint32_t n_chunks, DecodeWork* __restrict__ work,
                                                  uint32_t lane, uint32_t* __restrict__ status, const uint32_t* __restrict__ stored_bits = nullptr)
{
    static_assert(C::kMaxBytes <= 2, "DecPolicy::kNeed and the mirror are sized for at most 2 bytes per lane per step");
    TmaWindow win;
    win.ring = ring;
    win.seq_ready = kTmaSeqBase;
    const uint32_t lt = lanemask_lt();
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(&work->next_chunk, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= n_chunks) break;

        const uint64_t first = static_cast<uint64_t>(chunk) * chunk_syms;
        const uint64_t left = n - first;
        const uint32_t m = left < chunk_syms ? static_cast<uint32_t>(left) : chunk_syms;
        if (STORED && ((stored_bits[chunk >> 5] >> (chunk & 31)) & 1u)) {
            block_copy_stored(blob + offsets[chunk], out + first, m, lane);
            continue;
        }
        const uint64_t off = offsets[chunk];
        const uint64_t end = offsets[chunk + 1] & ~static_cast<uint64_t>(15);
        if (__shfl_sync(0xffffffffu, dir_entry_bad<C>(off, end, blob_size) ? 1u : 0u, 0)) {
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

        // lane k's state is the k-th state of the header; the mirror covers a wrap
        typename C::X x = coder.read_header([&](uint32_t b) { return win.cur + b; }, lane);
        win.cur += C::kHeaderBytes;

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
            for (int j = 0; j < P::kGroup; j++) coder.template step_p<P>(x, win.cur, og + 32 * j, lt, lane, j, true);
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
            coder.template step_p<P>(x, win.cur, o, lt, lane, -1, true);
            o += 32;
        }
        if (m & 31) coder.template step_p<P>(x, win.cur, o, lt, lane, -1, lane < (m & 31));

        const uint32_t pos = win.cur + (win.seq_ready * P::kUnit - P::kNeed - win.limit);
        const bool bad = (pos != pos0 + len) || (x != C::kL);
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

}  // namespace rb200

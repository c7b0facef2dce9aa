// placement.cuh -- how the fused encoders (word K2f, the fused mode of the alias / byte encoder, per-block K5f) turn
// finished chunk streams into the container, the chunk loop K2f and the alias / byte encoder run it from, and the stream
// copy the split path's compaction (K6) shares with them.
//
// Every worker warp fetches chunk ids in order, encodes a chunk into one of its own scratch slots and publishes the
// padded size in look[chunk].  One scanner warp of the grid turns the published sizes into end offsets in chunk order.
// A worker places chunk k (moves its stream to blob[E_k - size .. E_k) and writes the directory entry) only after it
// has encoded the chunks that fill its other slots, so its E_k is normally ready and no warp polls.  One launch, no CTA
// barrier in the loop.  (Two earlier variants -- per-CTA and per-warp decoupled look-back -- were correct but slower
// than the split path because of polling; see DESIGN.md section 6.)
#pragma once
#include "device_utils.cuh"
#include "encode_stream.cuh"

namespace rb200 {

constexpr uint64_t kLookAgg = 1ull << 62, kLookPrefix = 2ull << 62, kLookValue = (1ull << 62) - 1;
constexpr uint64_t kLookStallNs = 8ull * 1000 * 1000 * 1000;   // a bug must not hang the GPU: after 8 s without progress give up and
                                                               // flag kStatStall (time, not iterations: the waits are legitimate and
                                                               // stretch by orders of magnitude under compute-sanitizer)

__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p)
{
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint4 ldg_l2_u128(const uint4* p)      // L2-coherent: data this kernel wrote itself
{
    uint4 v;
    asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

// Move one finished stream (it ends at src_end, 16-byte aligned) to blob[end - size .. end): the container keeps every
// stream end-aligned with zero gap bytes in front, so the first 16-byte vector is gap zeros + the stream head and the
// rest moves as whole 128-bit vectors.
// SAME_LAUNCH: this kernel wrote the stream, so it is read L2-coherently (ld.global.cg, a volatile head byte);
// otherwise an earlier launch wrote it and the read-only path (ld.global.nc) is safe.
template <bool SAME_LAUNCH>
__device__ __forceinline__ void place_stream(const uint8_t* src_end, uint32_t size, uint8_t* __restrict__ blob, uint64_t end, uint32_t lane)
{
    const uint32_t padded = (size + 15u) & ~15u;
    const uint32_t gap = padded - size;
    const uint8_t* src = src_end - size;
    uint8_t* dst_vec0 = blob + (end - padded);
    if (lane < 16) {
        uint8_t v = 0;
        if (lane >= gap) {
            if (SAME_LAUNCH) v = *reinterpret_cast<const volatile uint8_t*>(src + (lane - gap));
            else v = src[lane - gap];
        }
        dst_vec0[lane] = v;
    }
    const uint4* s4 = reinterpret_cast<const uint4*>(src + (16 - gap));
    uint4* d4 = reinterpret_cast<uint4*>(dst_vec0 + 16);
    const uint32_t nvec = padded / 16 - 1;
    auto ld = [](const uint4* p) { return SAME_LAUNCH ? ldg_l2_u128(p) : ldg_stream_u128(p); };
    uint32_t v = lane;
    for (; v + 96 < nvec; v += 128) {                      // four loads in flight per lane
        const uint4 a = ld(s4 + v), b = ld(s4 + v + 32), c = ld(s4 + v + 64), d = ld(s4 + v + 96);
        stg_stream_u128(d4 + v, a);
        stg_stream_u128(d4 + v + 32, b);
        stg_stream_u128(d4 + v + 64, c);
        stg_stream_u128(d4 + v + 96, d);
    }
    for (; v < nvec; v += 32) stg_stream_u128(d4 + v, ld(s4 + v));
}

// A stored chunk (rb200_container_blocks_stored_encode_async): its m symbols at src, then zero bytes up to a multiple of
// 16, to dst (16-byte aligned), one warp.  Whole 16-byte loads where src and m allow them, bytes otherwise.
__device__ __forceinline__ void place_stored(const uint8_t* __restrict__ src, uint32_t m, uint8_t* __restrict__ dst, uint32_t lane)
{
    const bool vec = ((reinterpret_cast<uintptr_t>(src) | m) & 15) == 0;
    for (uint32_t v = lane; v < (m + 15) / 16; v += 32) {
        uint4 q;
        if (vec) {
            q = ldg_stream_u128(reinterpret_cast<const uint4*>(src) + v);
        } else {
            uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
            for (uint32_t j = 0; j < 16; j++)
                if (16 * v + j < m) w[j >> 2] |= static_cast<uint32_t>(src[16 * v + j]) << (8 * (j & 3));
            q = make_uint4(w[0], w[1], w[2], w[3]);
        }
        stg_stream_u128(reinterpret_cast<uint4*>(dst) + v, q);
    }
}

// The scanner: ONE warp of the grid walks the status array in chunk order and rewrites every published
// size (kLookAgg | padded size) into the inclusive end offset E_c (kLookPrefix | E_c).  Chunks are handed
// out in order, so the entry it waits for always belongs to a chunk some resident warp is encoding.
__device__ __forceinline__ void fused_scanner(uint64_t* look, uint32_t n_chunks, uint32_t lane, uint32_t* status)
{
    constexpr int kPer = 8;                 // consecutive entries per lane: 256 entries per trip, one warp scan per trip
    uint64_t run = 0, idle_since = 0;
    uint32_t pos = 0;
    while (pos < n_chunks) {
        const uint32_t base = pos + kPer * lane;
        uint64_t v[kPer];
#pragma unroll
        for (int j = 0; j < kPer; j++) v[j] = (base + j < n_chunks) ? ld_relaxed_u64(look + base + j) : 0;   // independent loads
        // r = length of this lane's leading run of published entries; local inclusive sums over that run
        uint32_t r = 0;
        uint64_t sum[kPer];
        uint64_t acc = 0;
        bool open = true;
#pragma unroll
        for (int j = 0; j < kPer; j++) {
            open = open && ((v[j] >> 62) == 1);
            if (open) { acc += v[j] & kLookValue; r = j + 1; }
            sum[j] = acc;
        }
        // the contiguous ready prefix of the whole window: all of lanes < f, the first r_f entries of lane f
        const uint32_t full = __ballot_sync(0xffffffffu, r == kPer);
        const uint32_t f = full == 0xffffffffu ? 32u : static_cast<uint32_t>(__ffs(~full)) - 1u;
        const uint32_t cnt = lane < f ? kPer : (lane == f ? r : 0u);
        const uint64_t mine = cnt ? sum[cnt - 1] : 0;
        uint64_t incl = mine;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= static_cast<uint32_t>(d)) incl += t;
        }
        const uint64_t before = run + incl - mine;
#pragma unroll
        for (int j = 0; j < kPer; j++)
            if (static_cast<uint32_t>(j) < cnt) st_relaxed_u64(look + base + j, kLookPrefix | (before + sum[j]));
        run += __shfl_sync(0xffffffffu, incl, 31);
        const uint32_t r_f = __shfl_sync(0xffffffffu, r, f & 31);
        const uint32_t done = f == 32 ? 32u * kPer : f * kPer + r_f;
        pos += done;
        if (done == 0) {
            const uint64_t now = global_timer_ns();
            if (!idle_since) idle_since = now;
            if (now - idle_since > kLookStallNs) {   // never hang the GPU: give up and flag
                if (lane == 0) atomicOr(status, kStatStall);
                return;
            }
            __nanosleep(100);
        } else {
            idle_since = 0;
        }
    }
}

// What placement writes, and the status array it reads E_c from.
struct PlaceOut {
    uint64_t* look;          // n_chunks entries, zeroed by the host: kLookAgg | padded size, then kLookPrefix | E_c
    uint32_t n_chunks;
    uint8_t* blob;
    uint64_t blob_cap;
    uint64_t* offsets;       // n_chunks + 1 directory entries
    uint32_t* status;
};

// one warp: wait for the scanner to publish E_c of `chunk`, then move the stream and write the directory entry
__device__ __forceinline__ void fused_place(const PlaceOut& out, uint32_t chunk, const uint8_t* slot_end, uint32_t produced, uint32_t lane)
{
    // Warps do not progress evenly, so the scan front (the oldest unfinished chunk) can trail this warp by a chunk time
    // and more: the wait is real, and every poll costs ~12 issue slots that the encoding warps of the SM want.  Back off
    // exponentially (128 ns .. 4 us): round 1 polled every 100 ns and spent a fifth of the kernel's instructions here
    // (seen in the ncu source view as millions of poll iterations per GiB).
    uint64_t v = 0, since = 0;
    uint32_t ns = 128;
    for (;;) {
        if (lane == 0) v = ld_relaxed_u64(out.look + chunk);
        v = __shfl_sync(0xffffffffu, v, 0);
        if ((v >> 62) == 2) break;
        if (ns >= 4096) {                                  // only once the back-off has topped out: keep the common path short
            const uint64_t now = global_timer_ns();
            if (!since) since = now;
            if (now - since > kLookStallNs) {
                if (lane == 0) atomicOr(out.status, kStatStall);
                return;
            }
        }
        __nanosleep(ns);
        if (ns < 4096) ns <<= 1;
    }
    const uint64_t end = v & kLookValue;                   // E_c
    if (lane == 0) {
        out.offsets[chunk] = end - produced;
        if (chunk == out.n_chunks - 1) out.offsets[out.n_chunks] = end;
    }
    if (end <= out.blob_cap) {
        place_stream<true>(slot_end, produced, out.blob, end, lane);
    } else if (lane == 0) {
        atomicOr(out.status, kStatSpace);
    }
}

// one warp: wait for the scanner to publish E_c of `chunk`, with fused_place's back-off; returns kLookPrefix | E_c, or 0
// once the wait has expired (kStatStall is then set).  fused_place keeps its own copy of the loop: calling this from
// it changes the code ptxas makes for every fused encoder.
__device__ __forceinline__ uint64_t wait_end_offset(const PlaceOut& out, uint32_t chunk, uint32_t lane)
{
    uint64_t v = 0, since = 0;
    uint32_t ns = 128;
    for (;;) {
        if (lane == 0) v = ld_relaxed_u64(out.look + chunk);
        v = __shfl_sync(0xffffffffu, v, 0);
        if ((v >> 62) == 2) return v;
        if (ns >= 4096) {
            const uint64_t now = global_timer_ns();
            if (!since) since = now;
            if (now - since > kLookStallNs) {
                if (lane == 0) atomicOr(out.status, kStatStall);
                return 0;
            }
        }
        __nanosleep(ns);
        if (ns < 4096) ns <<= 1;
    }
}

// One worker warp's SLOTS scratch slots, at scratch + worker * SLOTS * slot_bytes (the host sizes the scratch as
// workers x SLOTS slots).  A chunk is encoded into the slot that ends at next_end(), published by finish() and placed
// SLOTS - 1 chunks later; drain() places what is left once the warp runs out of chunks.
// The chunks are placed late on purpose.  Warps do not progress evenly (the issue arbiter favours high warp ids), so
// the scan front -- the oldest unfinished chunk -- trails the fastest warps by about one chunk time: placing 32 steps
// into the next chunk instead was measured to be about twice as slow: the workers spent their issue slots polling.
template <uint32_t SLOTS>
struct SlotQueue {
    static_assert(SLOTS >= 2, "a chunk is placed while the next one is encoded into another slot");
    uint8_t* slots;
    uint32_t slot_bytes;
    uint8_t* cur_end;                                      // end of the slot the next chunk is encoded into
    uint32_t pend_chunk[SLOTS - 1], pend_size[SLOTS - 1];  // oldest first, in the slots before cur_end; registers (static indexing only)
    uint32_t n_pending = 0;

    __device__ __forceinline__ SlotQueue(uint8_t* scratch, uint64_t worker, uint32_t slot_bytes_)
        : slots(scratch + worker * SLOTS * slot_bytes_), slot_bytes(slot_bytes_), cur_end(slots + slot_bytes_) {}

    __device__ __forceinline__ uint8_t* next_end() const { return cur_end; }

    // the slots form a ring
    __device__ __forceinline__ uint8_t* after(uint8_t* end) const
    {
        return end == slots + SLOTS * static_cast<uint64_t>(slot_bytes) ? slots + slot_bytes : end + slot_bytes;
    }
    __device__ __forceinline__ uint8_t* before(uint8_t* end) const
    {
        return end == slots + slot_bytes ? slots + SLOTS * static_cast<uint64_t>(slot_bytes) : end - slot_bytes;
    }

    // the chunk encoded at next_end() is `produced` bytes long: publish it, and place the oldest pending chunk once
    // every slot is taken
    __device__ __forceinline__ void finish(const PlaceOut& out, uint32_t chunk, uint32_t produced, uint32_t lane)
    {
        if (lane == 0) st_relaxed_u64(out.look + chunk, kLookAgg | ((produced + 15u) & ~15u));
        __syncwarp();
        if (n_pending == SLOTS - 1) {                      // the oldest sits in the slot after this one
            fused_place(out, pend_chunk[0], after(cur_end), pend_size[0], lane);
#pragma unroll
            for (int j = 0; j + 1 < static_cast<int>(SLOTS) - 1; j++) {
                pend_chunk[j] = pend_chunk[j + 1];
                pend_size[j] = pend_size[j + 1];
            }
            n_pending--;
        }
#pragma unroll
        for (int j = 0; j < static_cast<int>(SLOTS) - 1; j++)
            if (static_cast<uint32_t>(j) == n_pending) {
                pend_chunk[j] = chunk;
                pend_size[j] = produced;
            }
        n_pending++;
        cur_end = after(cur_end);
        __syncwarp();
    }

    // place the pending chunks, oldest first: the oldest sits n_pending slots before cur_end
    __device__ __forceinline__ void drain(const PlaceOut& out, uint32_t lane)
    {
        uint8_t* end = cur_end;
#pragma unroll
        for (int j = 0; j < static_cast<int>(SLOTS) - 1; j++)
            if (static_cast<uint32_t>(j) < n_pending) end = before(end);
#pragma unroll
        for (int j = 0; j < static_cast<int>(SLOTS) - 1; j++)
            if (static_cast<uint32_t>(j) < n_pending) {
                fused_place(out, pend_chunk[j], end, pend_size[j], lane);
                end = after(end);
            }
    }
};

// The chunk loop of a fused encoder of WARPS warps per CTA (K2f, the fused alias / byte mode).  Warp 0 of CTA 0 is the
// scanner; every other warp takes chunk ids from `counter` (zeroed by the host, so chunks start in order), encodes each
// into its SlotQueue<SLOTS> and places it SLOTS - 1 chunks later.  No CTA barrier: warps are independent from here on.
// wsm = this warp's 1 KiB of shared memory, KEEP as in encode_stream.
template <uint32_t SLOTS, uint32_t WARPS, bool KEEP, class Coder>
__device__ __forceinline__ void encode_chunks_fused(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, const Coder coder,
                                                    uint32_t wsm, uint8_t* __restrict__ scratch, uint32_t slot_bytes, const PlaceOut& out,
                                                    uint32_t* __restrict__ counter)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.x == 0 && warp == 0) {
        fused_scanner(out.look, out.n_chunks, lane, out.status);
        return;
    }
    SlotQueue<SLOTS> q(scratch, blockIdx.x * WARPS + warp, slot_bytes);
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(counter, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= out.n_chunks) break;
        const ChunkRange r = chunk_range(chunk, chunk_syms, n);
        const uint32_t produced = encode_stream<KEEP>(in + r.first, r.m, coder, wsm, q.next_end(), out.status);
        q.finish(out, chunk, produced, lane);
    }
    q.drain(out, lane);
}

}  // namespace rb200

// encode_ring.cuh -- the chunk loop of the fused word encoder whose streams stay in shared memory (K2r,
// word_kernels.cuh): each warp's stream ring, its spill slots, and the placement of a finished stream with TMA bulk
// copies.
//
// The protocol is placement.cuh's: a worker publishes kLookAgg | padded size in look[chunk], the scanner (warp 0 of
// CTA 0, fused_scanner) rewrites it to kLookPrefix | E_chunk, and the worker then writes the directory entry and stores
// the stream to blob[E - padded .. E).  The stream's bytes are stored from the warp's ring by one lane with
// cp.async.bulk (shared -> global), and the ring space is reused once the copy has read it
// (cp.async.bulk.wait_group.read).
//
// Streams are laid out downwards in the ring, each directly below the previous one, so a byte at distance d below the
// end (`top`) of its stream goes to blob[E - d - 1].  At most one finished stream waits for its offset (`pending`); the
// next chunk is encoded below it meanwhile.  The ring is smaller than a worst-case stream plus the one pending before
// it (that buys warps: DESIGN.md section 4), so when the next 16 steps could write into space still held, room is made
// oldest bytes first:
//   1. the pending stream: placed if its offset is published, otherwise its oldest ring bytes (up to PEND_PIECE, see
//      RB200_RING_PEND_PIECE) are copied to its spill slot;
//   2. then the current stream's oldest bytes, kSpillPiece at a time, to its spill slot.
// Each warp has two spill slots in global memory (the pending stream's and the current one's), a stream's byte at
// distance d below its end at slot_end - d - 1.  A stream with k bytes spilled (k % 16 == 0) is placed as a bulk store
// of its ring part to blob[E - padded, E - k) and a warp copy of slot_end - k .. slot_end to blob[E - k, E).  The spill
// stores carry an L2 evict_last hint, so the round trip normally stays in L2.
//
// Memory ordering of the spill slots, which racecheck does not model (async proxy):
//   - shared -> slot: every lane fences its ring writes to the async proxy (fence.proxy.async.shared::cta) and the warp
//     synchronises before lane 0 issues the copy, as for the blob stores.
//   - slot -> blob: lane 0 waits for every bulk copy to COMPLETE (cp.async.bulk.wait_group 0, not .read), which makes
//     their global writes visible to it, then fences the async proxy against the generic one (fence.proxy.async.global)
//     and the warp synchronises (__syncwarp orders memory among its threads) before the lanes read the slot with
//     L2-coherent loads (ld.global.cg, never .nc: the slot was written in this launch).
//   - slot reuse: the next spill into a slot is issued after the lanes' loads of it have returned (their values have
//     been stored), a fence.proxy.async.global by every lane and a __syncwarp.
#pragma once
#include "device_utils.cuh"
#include "encode_stream.cuh"
#include "placement.cuh"

namespace rb200 {

__device__ __forceinline__ void bulk_store_s2g(uint8_t* dst, uint32_t src, uint32_t bytes)   // both 16-byte aligned, bytes % 16 == 0
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_store_s2g_keep(uint8_t* dst, uint32_t src, uint32_t bytes)   // bulk_store_s2g, L2 evict_last
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst), "r"(src), "r"(bytes),
                 "l"(l2_policy_keep())
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// this thread's generic-proxy shared-memory writes become visible to the async proxy (the bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// orders this thread's global-memory accesses of the async proxy against those of the generic proxy, both ways
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// What one warp's ring did, for the timing lab: placements that waited for an offset, spills of a pending stream,
// and the bytes spilled (both kinds).
struct RingStats {
    uint32_t waits, pend_spills, spilled_bytes;
};

// One warp's stream ring of RING bytes at shared address `ring`, and its two spill slots of SLOT bytes (the longest
// stream a chunk can make) at `slots`.  All members are warp-uniform; lane 0 issues the bulk copies and owns their bulk group.
// PEND_PIECE: at most this many bytes of a pending stream whose offset is not yet published go to its slot per step
// of making room, oldest first (SLOT: the whole stream at once); 0: the offset is waited for instead (lab only).
template <uint32_t RING, uint32_t SLOT, uint32_t PEND_PIECE>
struct StreamRing {
    static_assert(RING % 16 == 0 && SLOT % 16 == 0 && RING > 2048 && SLOT <= 2 * RING, "ring positions wrap at most twice");
    static constexpr uint32_t kSpillPiece = 1024;

    PlaceOut out;
    uint8_t* slots;
    uint32_t ring, lane;
    uint32_t top = 0;          // ring position where the current stream ends (16-byte aligned)
    int32_t held = 0;          // ring bytes above `top` that may not be written (the pending stream's ring part, space
                               // still being read); negative once the current stream's oldest bytes are spilled and freed
    uint32_t inflight = 0;     // of those, the topmost ones, whose bulk copies may still be reading
    uint32_t cur_k = 0, cur_slot = 0;                          // the current stream's spilled bytes and slot
    uint32_t pend_chunk = 0, pend_size = 0, pend_top = 0, pend_k = 0;   // the pending stream (pend_size 0: none), in slot cur_slot ^ 1
    RingStats stats = {};

    __device__ __forceinline__ StreamRing(const PlaceOut& o, uint8_t* slots_, uint32_t ring_, uint32_t lane_)
        : out(o), slots(slots_), ring(ring_), lane(lane_) {}

    static __device__ __forceinline__ uint32_t pad(uint32_t b) { return (b + 15u) & ~15u; }
    // ring position d bytes below position p (p < RING, d <= SLOT <= 2 RING): p + 2 RING - d in [0, 3 RING), reduced
    static __device__ __forceinline__ uint32_t below(uint32_t p, uint32_t d)
    {
        uint32_t t = p + 2 * RING - d;
        t = min(t, t - RING);
        return min(t, t - RING);
    }
    __device__ __forceinline__ uint8_t* slot_end(uint32_t s) const { return slots + (s + 1) * SLOT; }

    // lane 0: bulk-store ring bytes [hi - bytes, hi) (modulo RING, hi in [0, RING)) to dst[0, bytes), one bulk group
    template <bool KEEP>
    __device__ __forceinline__ void store_ring(uint8_t* dst, uint32_t hi, uint32_t bytes)
    {
        auto copy = [](uint8_t* d, uint32_t s, uint32_t b) {
            if (KEEP) bulk_store_s2g_keep(d, s, b);
            else bulk_store_s2g(d, s, b);
        };
        const uint32_t lo = hi - bytes;
        if (static_cast<int32_t>(lo) >= 0) {
            copy(dst, ring + lo, bytes);
        } else {                                   // wraps: [lo + RING, RING) then [0, hi)
            copy(dst, ring + lo + RING, 0u - lo);
            if (hi) copy(dst + (0u - lo), ring, hi);
        }
        bulk_commit();
    }

    // the ring space of every issued bulk copy can be written again
    __device__ __forceinline__ void release()
    {
        if (lane == 0) bulk_wait_read();
        __syncwarp();
        held -= static_cast<int32_t>(inflight);
        inflight = 0;
    }

    // the current stream's emitted bytes, from their count modulo RING (its ring part is shorter than RING)
    __device__ __forceinline__ uint32_t emitted(uint32_t emitted_mod) const
    {
        const uint32_t t = emitted_mod - (cur_k >= RING ? cur_k - RING : cur_k);
        return cur_k + min(t, t + RING);
    }

    // store the pending stream, which ends at E = end, and write its directory entry
    __device__ __forceinline__ void place(uint64_t end)
    {
        const uint32_t padded = pad(pend_size), rp = padded - pend_k;
        if (lane == 0) {
            out.offsets[pend_chunk] = end - pend_size;
            if (pend_chunk == out.n_chunks - 1) out.offsets[out.n_chunks] = end;
        }
        if (end <= out.blob_cap) {
            if (pend_k) {                              // the spilled part, from the slot (ordering: file comment)
                if (lane == 0) {
                    bulk_wait_all();
                    fence_proxy_async_global();
                }
                __syncwarp();
                held -= static_cast<int32_t>(inflight);    // every copy has completed, so it has also read the ring
                inflight = 0;
                place_stream<true>(slot_end(cur_slot ^ 1), pend_k, out.blob, end, lane);
                fence_proxy_async_global();
                __syncwarp();
            }
            if (rp && lane == 0) store_ring<false>(out.blob + (end - padded), below(pend_top, pend_k), rp);
        } else if (lane == 0) {
            atomicOr(out.status, kStatSpace);
        }
        if (rp) inflight = held;                       // its ring part sits at the top of the held space
        pend_size = 0;
    }

    // wait for the pending stream's offset and place it (after an expired wait it is dropped: kStatStall is set)
    __device__ __forceinline__ void place_blocking()
    {
        uint64_t v = 0;
        if (lane == 0) v = ld_relaxed_u64(out.look + pend_chunk);
        v = __shfl_sync(0xffffffffu, v, 0);
        if ((v >> 62) != 2) {
            stats.waits++;
            v = wait_end_offset(out, pend_chunk, lane);
        }
        if (v) {
            place(v & kLookValue);
        } else {
            if (pad(pend_size) != pend_k) inflight = held;
            pend_size = 0;
        }
    }

    // returns once `need` bytes below the emitted ones (`emitted_mod`, modulo RING) of the current stream are free
    __device__ __forceinline__ void reserve(uint32_t emitted_mod, uint32_t need)
    {
        const uint32_t e = emitted(emitted_mod);
        // strict: the ring part of the current stream stays shorter than RING, so emitted() can unwrap its count
        while (static_cast<int32_t>(e + need) + held >= static_cast<int32_t>(RING)) {
            if (inflight) {
                release();
            } else if (pend_size && pad(pend_size) != pend_k) {      // the pending stream still has bytes in the ring
                uint64_t v = 0;
                if (lane == 0) v = ld_relaxed_u64(out.look + pend_chunk);
                v = __shfl_sync(0xffffffffu, v, 0);
                if ((v >> 62) == 2) {
                    place(v & kLookValue);
                } else if (PEND_PIECE) {                            // its oldest ring bytes to its slot
                    const uint32_t padded = pad(pend_size), p = min(PEND_PIECE, padded - pend_k);
                    if (lane == 0) store_ring<true>(slot_end(cur_slot ^ 1) - pend_k - p, below(pend_top, pend_k), p);
                    stats.pend_spills++;
                    stats.spilled_bytes += p;
                    pend_k += p;
                    inflight = static_cast<uint32_t>(held) - (padded - pend_k);   // all above its remaining ring part
                } else {
                    place_blocking();
                }
            } else {                                                // held == -cur_k: the current stream's oldest bytes
                const uint32_t p = min(kSpillPiece, (e & ~15u) - cur_k);
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) store_ring<true>(slot_end(cur_slot) - cur_k - p, below(top, cur_k), p);
                cur_k += p;
                inflight = p;
                stats.spilled_bytes += p;
            }
        }
    }

    // the stream of `chunk`, `produced` bytes ending at top, is complete: publish its size; it becomes the pending
    // stream (an older one still pending is placed first, which also frees the slot the next stream spills to)
    __device__ __forceinline__ void finish(uint32_t chunk, uint32_t produced)
    {
        const uint32_t padded = pad(produced);
        if (lane == 0) st_relaxed_u64(out.look + chunk, kLookAgg | padded);
        fence_proxy_async_smem();
        __syncwarp();
        if (pend_size) place_blocking();
        pend_chunk = chunk;
        pend_size = produced;
        pend_top = top;
        pend_k = cur_k;
        cur_k = 0;
        cur_slot ^= 1;
        held += static_cast<int32_t>(padded);
        top = below(top, padded);
    }

    // place what is left and let every bulk copy complete
    __device__ __forceinline__ void drain()
    {
        if (pend_size) place_blocking();
        if (lane == 0) bulk_wait_all();
        __syncwarp();
    }
};

// The chunk loop of K2r: warp 0 of CTA 0 is the scanner; every other warp takes chunk ids from `counter` (zeroed by the
// host) and encodes each with encode(chunk_in, m, ring) into its StreamRing.  `slots`: this warp's two spill slots.
// Returns what the warp's ring did.
template <uint32_t RING, uint32_t SLOT, uint32_t PEND_PIECE, class Encode>
__device__ __forceinline__ RingStats encode_chunks_ring(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t ring,
                                                        uint8_t* slots, const PlaceOut& out, uint32_t* __restrict__ counter, Encode&& encode)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.x == 0 && warp == 0) {
        fused_scanner(out.look, out.n_chunks, lane, out.status);
        return RingStats{};
    }
    StreamRing<RING, SLOT, PEND_PIECE> q(out, slots, ring, lane);
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(counter, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);
        if (chunk >= out.n_chunks) break;
        const ChunkRange r = chunk_range(chunk, chunk_syms, n);
        const uint32_t produced = encode(in + r.first, r.m, q);
        q.finish(chunk, produced);
    }
    q.drain();
    return q.stats;
}

}  // namespace rb200

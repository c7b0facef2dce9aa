// encode_ring.cuh -- the chunk loop of the fused word encoder whose streams stay in shared memory (K2r,
// word_kernels.cuh): each warp's stream ring, and the placement of a finished stream with TMA bulk copies.
//
// The protocol is placement.cuh's: a worker publishes kLookAgg | padded size in look[chunk], the scanner (warp 0 of
// CTA 0, fused_scanner) rewrites it to kLookPrefix | E_chunk, and the worker then writes the directory entry and stores
// the stream to blob[E - padded .. E).  Here the stream never leaves the warp's ring before that store: one lane issues
// cp.async.bulk (shared -> global) for it, and the ring space is reused once the copy has read it
// (cp.async.bulk.wait_group.read).
//
// Streams are laid out downwards in the ring, each directly below the previous one.  At most one finished stream waits
// for its offset (`pending`); the next chunk is encoded below it meanwhile.  The pending stream is placed only when the
// next 16 steps could write into its space, by then its offset is normally published, so placing it rarely waits
// (placement.cuh's bounded back-off, then kStatStall).  Looking for the offset once per 16 steps instead, to place the
// stream earlier, was slower (1.60 against 1.38 ms per GiB, DESIGN.md section 4).
#pragma once
#include "device_utils.cuh"
#include "encode_stream.cuh"
#include "placement.cuh"

namespace rb200 {

__device__ __forceinline__ void bulk_store_s2g(uint8_t* dst, uint32_t src, uint32_t bytes)   // both 16-byte aligned, bytes % 16 == 0
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// this thread's generic-proxy shared-memory writes become visible to the async proxy (the bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One warp's stream ring of RING bytes at shared address `ring`.  All members are warp-uniform; lane 0 issues the
// bulk copies and owns their bulk group.
template <uint32_t RING>
struct StreamRing {
    PlaceOut out;
    uint32_t ring, lane;
    uint32_t top = 0;          // ring position where the next stream ends (16-byte aligned)
    uint32_t held = 0;         // bytes above `top` that may not be written: the pending stream and placed ones still being read
    uint32_t inflight = 0;     // of those, placed streams whose bulk copies may still be reading
    uint32_t pend_chunk = 0, pend_size = 0, pend_top = 0;    // the pending stream (pend_size 0: none)
    uint32_t waits = 0;        // placements whose offset was not yet published (counted for the timing lab)

    __device__ __forceinline__ StreamRing(const PlaceOut& o, uint32_t ring_, uint32_t lane_) : out(o), ring(ring_), lane(lane_) {}

    // store the pending stream, which ends at E = end, and write its directory entry
    __device__ __forceinline__ void place(uint64_t end)
    {
        const uint32_t padded = (pend_size + 15u) & ~15u;
        if (lane == 0) {
            out.offsets[pend_chunk] = end - pend_size;
            if (pend_chunk == out.n_chunks - 1) out.offsets[out.n_chunks] = end;
            if (end <= out.blob_cap) {
                uint8_t* dst = out.blob + (end - padded);
                const uint32_t lo = pend_top - padded;
                if (static_cast<int32_t>(lo) >= 0) {
                    bulk_store_s2g(dst, ring + lo, padded);
                } else {                                   // the stream wraps: [lo + RING, RING) then [0, pend_top)
                    bulk_store_s2g(dst, ring + lo + RING, 0u - lo);
                    if (pend_top) bulk_store_s2g(dst + (0u - lo), ring, pend_top);
                }
                bulk_commit();
            } else {
                atomicOr(out.status, kStatSpace);
            }
        }
        inflight += padded;
        pend_size = 0;
    }

    // wait for the pending stream's offset and place it (after an expired wait it is dropped: kStatStall is set)
    __device__ __forceinline__ void place_blocking()
    {
        uint64_t v = 0;
        if (lane == 0) v = ld_relaxed_u64(out.look + pend_chunk);
        v = __shfl_sync(0xffffffffu, v, 0);
        if ((v >> 62) != 2) {
            waits++;
            v = wait_end_offset(out, pend_chunk, lane);
        }
        if (v) {
            place(v & kLookValue);
        } else {
            held -= (pend_size + 15u) & ~15u;
            pend_size = 0;
        }
    }

    // returns once `need` bytes below the `emitted` bytes of the stream being encoded are not held
    __device__ __forceinline__ void reserve(uint32_t emitted, uint32_t need)
    {
        while (held && emitted + need > RING - held) {
            if (inflight) {
                if (lane == 0) bulk_wait_read();
                __syncwarp();
                held -= inflight;
                inflight = 0;
            } else {
                place_blocking();
            }
        }
    }

    // the stream of `chunk`, `produced` bytes ending at top(), is complete: publish its size; it becomes the pending
    // stream (an older one still pending is placed first)
    __device__ __forceinline__ void finish(uint32_t chunk, uint32_t produced)
    {
        const uint32_t padded = (produced + 15u) & ~15u;
        if (lane == 0) st_relaxed_u64(out.look + chunk, kLookAgg | padded);
        fence_proxy_async_smem();
        __syncwarp();
        if (pend_size) place_blocking();
        pend_chunk = chunk;
        pend_size = produced;
        pend_top = top;
        held += padded;
        const uint32_t t = top - padded;
        top = min(t, t + RING);
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
// host) and encodes each with encode(chunk_in, m, top, ring) into its StreamRing.  Returns the warp's ring waits.
template <uint32_t RING, class Encode>
__device__ __forceinline__ uint32_t encode_chunks_ring(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t ring,
                                                       const PlaceOut& out, uint32_t* __restrict__ counter, Encode&& encode)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.x == 0 && warp == 0) {
        fused_scanner(out.look, out.n_chunks, lane, out.status);
        return 0;
    }
    StreamRing<RING> q(out, ring, lane);
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
    return q.waits;
}

}  // namespace rb200

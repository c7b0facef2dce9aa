// container_decode.cuh -- rb200_container_blocks_decode_async: a per-block (version 2) container in device memory,
// checked and decoded by kernels alone, so that the call only enqueues work (and can be captured in a CUDA graph).
//
// The stages run in stream order; each reads what the one before it left in the context's BlocksAsyncWork:
//   container_plan_kernel          one warp: container_header_ok on buf[0, 64) against size -> the plan; clears the
//                                  verdict words
//   crc32_kernel x 2               meta CRC of buf + 64, length from the plan; blob CRC at buf + blob_off (both lengths
//                                  are zero when the header is rejected, the blob's also when the flag is clear)
//   container_prefix_check_kernel  container_block_model_ok for every block, container_dir_step_ok for every
//                                  directory entry, container_dir_ends_ok once
//   container_verdict_kernel       one warp: header CRC (crc fields zero) joined with the meta CRC, both CRCs compared;
//                                  writes n_symbols, then sets go or ORs kStatStream / kStatSpace into the status word
//   block_decode_planned_kernel    a fixed grid that exits at once unless go; CTAs take block ids from a counter, build
//                                  the block's slot table in shared memory and decode its chunks
// The rules are the host parser's (container_format.h); they run in its order: content errors before kStatSpace.
#pragma once
#include "block_kernels.cuh"
#include "container_format.h"
#include "crc_kernels.cuh"

namespace rb200 {

// What the plan kernel read from the header.  ok == 0 when the header is rejected; every length is then zero, so the
// CRC launches read nothing.
struct BlocksPlan {
    uint64_t n_symbols, n_chunks, dir_off, blob_off, blob_bytes;
    uint64_t meta_len;          // bytes meta_crc covers after the header: model section and directory
    uint64_t blob_len;          // blob_bytes with RB200_CONTAINER_CRC_BLOB, else 0
    uint32_t ok, n_blocks, block_size, chunk_syms;
};

// The call's workspace: fixed-size, allocated with the context, so the call never allocates.
struct BlocksAsyncWork {
    BlocksPlan plan;
    CrcSlot crc[2];             // meta, blob
    CrcWork crc_work;           // crc32_kernel's accumulator, zero between launches
    uint32_t bad;               // a block model or a directory entry broke a rule
    uint32_t go;                // the verdict: decode.  Private to the call, so that status bits left by earlier calls
                                // that were not synchronised do not change this call's outcome
    uint32_t next_block;        // the decoder's work counter; zero between launches (the last CTA out re-arms it)
    uint32_t ctas_done;
};

__global__ void __launch_bounds__(32) container_plan_kernel(const uint8_t* __restrict__ buf, uint64_t size, BlocksAsyncWork* w)
{
    if (threadIdx.x) return;
    BlocksPlan p = {};
    if (size >= sizeof(ContainerHeader)) {                           // a shorter buffer is not read at all
        const ContainerHeader h = *reinterpret_cast<const ContainerHeader*>(buf);
        if (container_header_ok(h, size, kContainerVersionBlocks)) {
            p.ok = 1;
            p.n_symbols = h.n_symbols;
            p.n_chunks = h.n_chunks;
            p.dir_off = container_dir_offset(h);
            p.blob_off = container_blob_offset(h);
            p.blob_bytes = h.blob_bytes;
            p.meta_len = container_dir_end(h) - sizeof(ContainerHeader);
            p.blob_len = (h.flags & RB200_CONTAINER_CRC_BLOB) ? h.blob_bytes : 0;
            p.n_blocks = h.n_blocks;
            p.block_size = h.block_size;
            p.chunk_syms = h.chunk_syms;
        }
    }
    w->plan = p;
    w->bad = 0;
    w->go = 0;
}

// The per-element rules of the prefix.  Each warp stages 32 block models (16 KiB, coalesced) in shared memory with
// rows padded to 129 words, so that lane r checking row r reads a different bank from every other lane.
constexpr int kPrefixWarps = 2;
constexpr uint32_t kPrefixRowWords = 129;

__global__ void __launch_bounds__(kPrefixWarps * 32)
    container_prefix_check_kernel(const uint8_t* __restrict__ buf, BlocksAsyncWork* w)
{
    __shared__ uint32_t s_rows[kPrefixWarps][32 * kPrefixRowWords];
    const BlocksPlan p = w->plan;
    if (!p.ok) return;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint4* models = reinterpret_cast<const uint4*>(buf + sizeof(ContainerHeader));        // 32 vectors per block
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + p.dir_off);
    bool ok = true;
    uint32_t* rows = s_rows[warp];
    const uint64_t warps = static_cast<uint64_t>(gridDim.x) * kPrefixWarps;
    for (uint64_t b0 = (static_cast<uint64_t>(blockIdx.x) * kPrefixWarps + warp) * 32; b0 < p.n_blocks; b0 += warps * 32) {
        const uint32_t n = p.n_blocks - b0 < 32 ? static_cast<uint32_t>(p.n_blocks - b0) : 32u;
        for (uint32_t i = lane; i < n * 32; i += 32) {
            const uint4 v = models[b0 * 32 + i];
            uint32_t* d = rows + (i >> 5) * kPrefixRowWords + (i & 31) * 4;
            d[0] = v.x;
            d[1] = v.y;
            d[2] = v.z;
            d[3] = v.w;
        }
        __syncwarp();
        if (lane < n) ok &= container_block_model_ok(reinterpret_cast<const uint16_t*>(rows + lane * kPrefixRowWords));
        __syncwarp();
    }
    const uint64_t threads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (uint64_t c = t; c < p.n_chunks; c += threads) ok &= container_dir_step_ok(offsets, c);
    if (t == 0) ok &= container_dir_ends_ok(offsets, p.n_chunks, p.blob_bytes);
    if (!ok) w->bad = 1;
}

// One warp.  meta_crc covers the header with its crc fields zeroed, then meta_len bytes whose CRC is in crc[0];
// the header's CRC is taken here with container_finish_kernel's warp helpers and joined (crc32_combine).
__global__ void __launch_bounds__(32)
    container_verdict_kernel(const uint8_t* __restrict__ buf, uint64_t out_cap, uint64_t* __restrict__ n_symbols, BlocksAsyncWork* w,
                             uint32_t* status)
{
    using namespace crc_detail;
    __shared__ uint4 s_head_v[sizeof(ContainerHeader) / 16];
    uint32_t* s_head = reinterpret_cast<uint32_t*>(s_head_v);
    const uint32_t lane = threadIdx.x;
    const BlocksPlan& p = w->plan;
    if (!p.ok) {
        if (lane == 0) atomicOr(status, kStatStream);
        return;
    }
    if (lane < sizeof(ContainerHeader) / 16) s_head_v[lane] = reinterpret_cast<const uint4*>(buf)[lane];
    __syncwarp();
    const uint32_t meta_crc = s_head[offsetof(ContainerHeader, meta_crc) / 4];
    const uint32_t blob_crc = s_head[offsetof(ContainerHeader, blob_crc) / 4];
    const uint32_t flags = s_head[offsetof(ContainerHeader, flags) / 4];
    __syncwarp();
    if (lane == 0) {
        s_head[offsetof(ContainerHeader, meta_crc) / 4] = 0;
        s_head[offsetof(ContainerHeader, blob_crc) / 4] = 0;
    }
    __syncwarp();
    // 2 bytes per lane, each shifted past the bytes after it
    uint32_t c = raw_bytes_bitwise(reinterpret_cast<const uint8_t*>(s_head) + lane * 2, 2);
    c = __reduce_xor_sync(0xffffffffu, crc32_shift(c, sizeof(ContainerHeader) - 2 * (lane + 1)));
    const uint32_t head_crc = finish_warp(0, sizeof(ContainerHeader), c);
    const uint32_t meta = crc32_mulmod(head_crc, x8pow_warp(p.meta_len)) ^ w->crc[0].crc;
    if (lane) return;
    const bool prefix_ok = meta == meta_crc && !w->bad;
    if (prefix_ok && n_symbols) *n_symbols = p.n_symbols;
    if (!prefix_ok || ((flags & RB200_CONTAINER_CRC_BLOB) && w->crc[1].crc != blob_crc))
        atomicOr(status, kStatStream);
    else if (p.n_symbols > out_cap)
        atomicOr(status, kStatSpace);
    else
        w->go = 1;
}

// The per-block decoder for a geometry only the device knows: a fixed grid of kPlannedWarps-warp CTAs (resident all at
// once) takes block ids from w->next_block; per block, the slot table as block_decode_kernel builds it (the WIDE
// variant chosen per block), then the warps take the block's 1..32 chunks in turn.
constexpr int kPlannedWarps = 8;

__global__ void __launch_bounds__(kPlannedWarps * 32, 8)
    block_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, BlocksAsyncWork* w, uint32_t* __restrict__ status)
{
    __shared__ __align__(1024) uint8_t s_ring[kPlannedWarps * kRingBytes];
    __shared__ __align__(16) uint32_t s_tab[kWordSlots];
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[2];                               // [0] bad model, [1] wide (a freq of 4096)
    __shared__ uint32_t s_block;
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    if (w->go) {                                                 // the same for the whole grid
        const BlocksPlan& p = w->plan;
        const uint32_t n_blocks = p.n_blocks, block_size = p.block_size, chunk_syms = p.chunk_syms;
        const uint32_t per_block = block_size / chunk_syms;
        const uint64_t blob_bytes = p.blob_bytes;
        const uint16_t* models = reinterpret_cast<const uint16_t*>(buf + sizeof(ContainerHeader));
        const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + p.dir_off);
        const uint8_t* blob = buf + p.blob_off;
        const uint32_t ring = smem_addr(s_ring) + warp * kRingBytes;
        for (;;) {
            __syncthreads();                                     // the previous block's table is no longer in use
            if (tid == 0) {
                s_block = atomicAdd(&w->next_block, 1u);
                s_flag[1] = 0;
            }
            __syncthreads();
            const uint32_t block = s_block;
            if (block >= n_blocks) break;
            if (!block_prefix(models + static_cast<uint64_t>(block) * 256, s_cum, &s_flag[0])) {   // checked before: not reached
                if (tid == 0) atomicOr(status, kStatStream);
                continue;
            }
            block_fill_slots(s_cum, s_tab, &s_flag[1]);
            __syncthreads();
            const bool wide = s_flag[1] != 0;
            for (uint32_t k = warp; k < per_block; k += kPlannedWarps) {
                const uint32_t chunk = block * per_block + k;
                uint8_t* dst = out + static_cast<uint64_t>(block) * block_size + static_cast<uint64_t>(k) * chunk_syms;
                if (wide)
                    decode_window_chunk(WordDecoder<true>{smem_addr_pinned(s_tab), 0}, blob, blob_bytes, offsets, chunk, ring, dst, chunk_syms, status);
                else
                    decode_window_chunk(WordDecoder<false>{smem_addr_pinned(s_tab), 0}, blob, blob_bytes, offsets, chunk, ring, dst, chunk_syms, status);
            }
        }
    }
    // every CTA has taken its last block id before it counts itself out: the last one re-arms the counter
    if (tid == 0 && atomicAdd(&w->ctas_done, 1u) == gridDim.x - 1) {
        w->next_block = 0;
        w->ctas_done = 0;
    }
}

// The launch shapes, fixed per device: the decoder's grid is every CTA that is resident at once.
struct BlocksAsyncShape {
    uint32_t decode_grid, check_grid;
};

inline BlocksAsyncShape configure_container_decode(uint32_t sms)
{
    cudaFuncSetAttribute(block_decode_planned_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, block_decode_planned_kernel, kPlannedWarps * 32, 0);
    return BlocksAsyncShape{sms * static_cast<uint32_t>(per_sm < 1 ? 1 : per_sm), sms * 8};
}

}  // namespace rb200

// container_decode.cuh -- rb200_container_decode_async (version 1, one model, any coder),
// rb200_container_blocks_decode_async (version 2, per-block models), rb200_container_blocks_coder_decode_async
// (version 3, per-block models of the byte or rans64 coder) and rb200_container_blocks_alias_decode_async (version 4,
// per-block models of the alias coder): a container in device memory, checked and decoded by kernels alone, so that the
// call only enqueues work (and can be captured in a CUDA graph).
//
// The stages run in stream order; each reads what the one before it left in the call's ContainerAsyncWork (one per
// version, allocated with the context):
//   container_plan_kernel          one warp: container_header_ok on buf[0, 64) against size for the call's version ->
//                                  the plan, coder and scale_bits; clears the verdict words and the decoders' work
//                                  counters, so that a call never depends on how the previous one ended
//   crc32_kernel x 2               meta CRC of buf + 64, length from the plan; blob CRC at buf + blob_off (both lengths
//                                  are zero when the header is rejected, the blob's also when the flag is clear)
//   container_prefix_check_kernel  container_block_model_sums_to(1 << scale_bits) for every block (none in version 1),
//                                  container_dir_step_ok for every directory entry, container_dir_ends_ok once
//   container_table_kernel         version 1, one CTA: container_model_ok and container_model_decodable on the model,
//                                  then the header coder's decode table, byte for byte what rb200_model_create uploads
//   container_verdict_kernel       one warp: header CRC (crc fields zero) joined with the meta CRC, both CRCs compared,
//                                  what the decoders refuse; writes n_symbols, then sets go to the id of the decoder to
//                                  run (container_decoder) or ORs kStatStream / kStatSpace into the status word
//   the version's decoders         one launch per decoder the version can need, each on a fixed grid of every CTA that
//                                  is resident at once; only the one whose id is in go runs, every other exits before
//                                  it touches shared memory, TMA or its counter.  Version 1: one per variant rb200_decode
//                                  can pick (kDec*); versions 2, 3 and 4: block_decode_planned_kernel<CODER, SB>, one per
//                                  instance of RB200_BLOCK_DISPATCH of the version's coders.  The per-block ones take
//                                  block ids from a counter, build the block's table in shared memory (block_decode_table;
//                                  version 4: the block's alias pairing first) and decode its chunks.
// The rules are the host parser's (container_format.h); they run in its order: content errors before kStatSpace.
//
// rb200_container_blocks_any_decode_async runs the same stages on its own workspace for whichever per-block version the
// header names (kContainerVersionAnyBlocks), then the decoders of versions 2, 3 and 4: their ids are unique across
// those versions.
#pragma once
#include "alias_kernels.cuh"
#include "block_coder_kernels.cuh"
#include "block_kernels.cuh"
#include "container_format.h"
#include "crc_kernels.cuh"
#include "rans64_kernels.cuh"
#include "word_decode_tma.cuh"

namespace rb200 {

// What the plan kernel read from the header.  ok == 0 when the header is rejected; every length is then zero, so the
// CRC launches read nothing.
struct BlocksPlan {
    uint64_t n_symbols, n_chunks, dir_off, blob_off, blob_bytes;
    uint64_t meta_len;          // bytes meta_crc covers after the header: model section and directory
    uint64_t blob_len;          // blob_bytes with RB200_CONTAINER_CRC_BLOB, else 0
    uint32_t ok, n_blocks, block_size, chunk_syms;   // n_blocks, block_size: per-block versions only (else zero)
};

// the largest decode table: rans64's cum2sym at scale_bits 16 and its 256 x {start, freq}
constexpr uint32_t kSingleTableBytes = (1u << 16) + 2048;

// The call's workspace: fixed-size, allocated with the context, so the call never allocates.
struct ContainerAsyncWork {
    BlocksPlan plan;
    CrcSlot crc[2];             // meta, blob
    CrcWork crc_work;           // crc32_kernel's accumulator, zero between launches
    uint32_t bad;               // the model, a block model or a directory entry broke a rule
    uint32_t go;                // the verdict: the id of the decoder to run, 0 for none.  Private to the call, so that
                                // status bits left by earlier calls that were not synchronised do not change its outcome
    uint32_t next_block;        // the per-block decoders' work counter; zero between launches (the last CTA out re-arms it)
    uint32_t ctas_done;
    uint32_t coder, scale_bits; // from the header, when plan.ok
    uint32_t wide;              // version 1: the word table has a slot of frequency 4096
    uint32_t refused;           // version 1: the decoders refuse the model (container_model_decodable)
    DecodeWork work;            // version 1: the decoder's chunk counter; zero between launches (the last warp out re-arms it)
    alignas(16) uint8_t table[kSingleTableBytes];   // version 1: the decode table of the header's coder, as rb200_model_create's
};

// The decoders, with ids from 1 in the order of the launch table (configure_container_decode); the verdict stores the id
// of the one to run in go, kDecNone decodes nothing.  Version 1: one per variant rb200_decode picks, the word coder
// narrow or WIDE (a frequency of 4096), the alias and byte coders specialised for scale_bits 16, 14, 12 or generic
// (RB200_ALIAS_SB_DISPATCH), rans64.  Versions 2, 3 and 4, numbered once across them: one per instance of
// RB200_BLOCK_DISPATCH, the word coder (1), the byte coder at scale_bits 14, 12 or generic (2, 3, 4), rans64 (5), the
// alias coder at scale_bits 14, 12 or generic (6, 7, 8).
constexpr uint32_t kDecNone = 0, kDecWord = 1, kDecWordWide = 2, kDecAlias = 3, kDecByte = 7, kDecRans64 = 11;
// the version argument of rb200_container_blocks_any_decode_async's plan and verdict: whichever of versions 2, 3 and 4
// the header names
constexpr uint16_t kContainerVersionAnyBlocks = 0;
// offset of a specialisation from kDecAlias / kDecByte
__host__ __device__ constexpr uint32_t sb_variant(uint32_t sb) { return sb == 16 ? 0 : sb == 14 ? 1 : sb == 12 ? 2 : 3; }

// the id of the decoder a container of `version` needs for the header's coder and scale_bits (version 1: rb200_decode's
// choice of kernel, decode_device; wide: the word table has a slot of frequency 4096)
__host__ __device__ constexpr uint32_t container_decoder(uint32_t version, uint32_t coder, uint32_t sb, uint32_t wide)
{
    if (version != kContainerVersion) {                              // the per-block versions
        if (coder == RB200_CODER_WORD) return 1;
        if (coder == RB200_CODER_RANS64) return 5;
        return (coder == RB200_CODER_ALIAS ? 6 : 2) + (sb == 14 ? 0 : sb == 12 ? 1 : 2);
    }
    if (coder == RB200_CODER_WORD) return wide ? kDecWordWide : kDecWord;
    if (coder == RB200_CODER_ALIAS) return kDecAlias + sb_variant(sb);
    if (coder == RB200_CODER_BYTE) return kDecByte + sb_variant(sb);
    return kDecRans64;
}

// One warp: the plan of a header that passes the rules of the call's version (a zero plan otherwise), with the verdict
// words and the decoders' counters cleared.  kContainerVersionAnyBlocks: the version the header names when that is 2, 3
// or 4; any other version, or fewer than 64 bytes, gets the zero plan.
__global__ void __launch_bounds__(32)
    container_plan_kernel(const uint8_t* __restrict__ buf, uint64_t size, uint32_t version, ContainerAsyncWork* w)
{
    if (threadIdx.x) return;
    if (version == kContainerVersionAnyBlocks) {
        version = size >= sizeof(ContainerHeader) ? reinterpret_cast<const ContainerHeader*>(buf)->version : 0u;
        if (version < kContainerVersionBlocks || version > kContainerVersionBlocksAlias) size = 0;
    }
    BlocksPlan p = {};
    uint32_t coder = 0, scale_bits = 0;
    if (size >= sizeof(ContainerHeader)) {                           // a shorter buffer is not read at all
        const ContainerHeader h = *reinterpret_cast<const ContainerHeader*>(buf);
        if (container_header_ok(h, size, static_cast<uint16_t>(version))) {
            p.ok = 1;
            p.n_symbols = h.n_symbols;
            p.n_chunks = h.n_chunks;
            p.dir_off = container_dir_offset(h);
            p.blob_off = container_blob_offset(h);
            p.blob_bytes = h.blob_bytes;
            p.meta_len = container_dir_end(h) - sizeof(ContainerHeader);
            p.blob_len = (h.flags & RB200_CONTAINER_CRC_BLOB) ? h.blob_bytes : 0;
            if (container_per_block(h)) {                            // version 1 does not check n_blocks and block_size
                p.n_blocks = h.n_blocks;
                p.block_size = h.block_size;
            }
            p.chunk_syms = h.chunk_syms;
            coder = h.coder;
            scale_bits = h.scale_bits;
        }
    }
    w->plan = p;
    w->bad = 0;
    w->go = 0;
    w->next_block = 0;
    w->ctas_done = 0;
    w->coder = coder;
    w->scale_bits = scale_bits;
    w->wide = 0;
    w->refused = 0;
    w->work = DecodeWork{0, 0};
}

// The per-element rules of the prefix.  Each warp stages 32 block models (16 KiB, coalesced) in shared memory with
// rows padded to 129 words, so that lane r checking row r reads a different bank from every other lane.  Every block
// sums to 1 << scale_bits; version 1 has no blocks (n_blocks 0), so only the directory rules run.
constexpr int kPrefixWarps = 2;
constexpr uint32_t kPrefixRowWords = 129;

__global__ void __launch_bounds__(kPrefixWarps * 32)
    container_prefix_check_kernel(const uint8_t* __restrict__ buf, ContainerAsyncWork* w)
{
    __shared__ uint32_t s_rows[kPrefixWarps][32 * kPrefixRowWords];
    const BlocksPlan p = w->plan;
    if (!p.ok) return;
    const uint32_t total = 1u << w->scale_bits;
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
        if (lane < n) ok &= container_block_model_sums_to(reinterpret_cast<const uint16_t*>(rows + lane * kPrefixRowWords), total);
        __syncwarp();
    }
    const uint64_t threads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t t = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (uint64_t c = t; c < p.n_chunks; c += threads) ok &= container_dir_step_ok(offsets, c);
    if (t == 0) ok &= container_dir_ends_ok(offsets, p.n_chunks, p.blob_bytes);
    if (!ok) w->bad = 1;
}

// The version 1 model (256 x u32 at buf + 64) checked and turned into the decode table of the header's coder in
// s->table, byte for byte what rb200_model_create builds on the host (tables.h has the formats and the per-entry
// formulas both sides call).  Slot-to-symbol is a binary search over cum, per slot (word) or per 4 slots (the cum2sym
// bytes of the byte and rans64 coders, stored as one u32); the alias pairing runs on one thread.
constexpr int kTableThreads = 512;

__global__ void __launch_bounds__(kTableThreads) container_table_kernel(const uint8_t* __restrict__ buf, ContainerAsyncWork* s)
{
    __shared__ uint32_t s_freq[256], s_cum[257];
    __shared__ uint32_t s_divider[256], s_adjust[512], s_slot_freqs[512], s_rest[256], s_given[256];
    __shared__ uint8_t s_sym_id[512];
    __shared__ uint32_t s_build;
    const uint32_t tid = threadIdx.x;
    if (!s->plan.ok) return;
    const uint32_t coder = s->coder, sb = s->scale_bits;
    if (tid < 256) s_freq[tid] = reinterpret_cast<const uint32_t*>(buf + sizeof(ContainerHeader))[tid];
    __syncthreads();
    if (tid == 0) {
        bool build = false;
        if (!container_model_ok(coder, sb, s_freq)) {
            s->bad = 1;                                              // what rb200_container_open rejects
        } else if (!container_model_decodable(coder, s_freq)) {
            s->refused = 1;                                          // what rb200_container_decode refuses
        } else if (coder == RB200_CODER_ALIAS) {
            build = alias_tables_core(s_freq, (1u << sb) / 256, s_divider, s_adjust, s_slot_freqs, s_sym_id, s_rest, s_given);
            if (!build) s->refused = 1;                              // rb200_model_create: RB200_E_MODEL
        } else {
            build = true;
        }
        s_cum[0] = 0;
        for (int i = 0; i < 256; i++) s_cum[i + 1] = s_cum[i] + s_freq[i];    // < 2^17 once the model is ok
        s_build = build;
    }
    __syncthreads();
    if (!s_build) return;
    const uint32_t M = 1u << sb;
    // the symbol whose range holds slot: the largest s with cum[s] <= slot (zero-width symbols hold none)
    auto symbol_of = [&](uint32_t slot) {
        uint32_t lo = 0, hi = 256;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s_cum[mid] <= slot) lo = mid; else hi = mid;
        }
        return lo;
    };
    if (coder == RB200_CODER_WORD) {
        uint32_t* tab = reinterpret_cast<uint32_t*>(s->table);
        bool wide = false;
        for (uint32_t slot = tid; slot < M; slot += kTableThreads) {
            const uint32_t sym = symbol_of(slot), f = s_cum[sym + 1] - s_cum[sym];
            wide |= f == M;
            tab[slot] = word_dec_entry(sym, f, slot - s_cum[sym]);
        }
        if (wide) s->wide = 1;
    } else if (coder == RB200_CODER_ALIAS) {
        if (tid < 256) reinterpret_cast<AliasDecEntry*>(s->table)[tid] = alias_dec_entry(tid, s_divider, s_adjust, s_slot_freqs, s_sym_id);
    } else {                                                         // byte, rans64: cum2sym[M], then 256 symbol entries
        uint32_t* c2s = reinterpret_cast<uint32_t*>(s->table);
        for (uint32_t q = tid; q < M / 4; q += kTableThreads) {
            uint32_t sym = symbol_of(4 * q), packed = 0;
            for (uint32_t k = 0; k < 4; k++) {
                while (4 * q + k >= s_cum[sym + 1]) sym++;           // steps over zero-width symbols
                packed |= sym << (8 * k);
            }
            c2s[q] = packed;
        }
        uint32_t* syms = reinterpret_cast<uint32_t*>(s->table + M);
        if (tid < 256) {
            const uint32_t f = s_cum[tid + 1] - s_cum[tid];
            if (coder == RB200_CODER_BYTE) {
                syms[tid] = byte_dec_symbol(s_cum[tid], f);
            } else {                                                 // Rans64DecSymbol {start, freq}
                syms[2 * tid] = s_cum[tid];
                syms[2 * tid + 1] = f;
            }
        }
    }
}

// One warp.  meta_crc covers the header with its crc fields zeroed, then meta_len bytes whose CRC is in crc[0];
// the header's CRC is taken here with container_finish_kernel's warp helpers and joined (crc32_combine).  What open
// accepts but the decoders do not take is refused as content (kStatStream): a blob of 2^36 bytes or more and version 1's
// chunk sizes outside 32 .. 2^24 (container_geometry_decodable), version 1's models that the table kernel refused.
__global__ void __launch_bounds__(32)
    container_verdict_kernel(const uint8_t* __restrict__ buf, uint64_t out_cap, uint64_t* __restrict__ n_symbols, ContainerAsyncWork* w,
                             uint32_t* status, uint32_t version)
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
    const bool refused = w->refused || !container_geometry_decodable(p.chunk_syms, p.blob_bytes);
    if (!prefix_ok || refused || ((flags & RB200_CONTAINER_CRC_BLOB) && w->crc[1].crc != blob_crc))
        atomicOr(status, kStatStream);
    else if (p.n_symbols > out_cap)
        atomicOr(status, kStatSpace);
    else
        w->go = container_decoder(version, w->coder, w->scale_bits, w->wide);
}

// The per-block decoders for a geometry only the device knows, one per instance of RB200_BLOCK_DISPATCH, each on a fixed
// grid of kPlannedWarps-warp CTAs (resident all at once).  Only the one whose id is in go runs; every other exits before
// it touches shared memory or the counter.  CTAs take block ids from w->next_block; per block, block_decode_kernel's two
// steps: the table in shared memory (block_decode_table), then the warps take the block's 1..32 chunks in turn
// (block_decode_chunk).  The alias coder's pairing overlays the table the previous block's warps read: the barrier at
// the loop's top keeps it behind their last chunk.  The word instance keeps 8 CTAs per SM (32 registers).
constexpr int kPlannedWarps = 8;

template <uint32_t CODER, uint32_t SB>
__global__ void __launch_bounds__(kPlannedWarps * 32, CODER == RB200_CODER_WORD ? 8 : 0)
    block_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, ContainerAsyncWork* __restrict__ w,
                                uint32_t* __restrict__ status)
{
    if (w->go != container_decoder(kContainerVersionBlocks, CODER, SB, 0)) return;   // the same for the whole grid
    // [kPlannedWarps x 1 KiB rings][the block's decode table]: dynamic, but static for the word coder, whose decode
    // step ptxas schedules better with the table at a fixed address
    extern __shared__ __align__(1024) uint8_t s_dyn[];
    __shared__ __align__(1024) uint8_t s_word[CODER == RB200_CODER_WORD ? kPlannedWarps * kRingBytes + kWordSlots * 4 : 1];
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[2];                              // [0] bad model, [1] wide (word coder)
    __shared__ uint32_t s_block;
    uint8_t* s_bdec = CODER == RB200_CODER_WORD ? s_word : s_dyn;
    const BlocksPlan& p = w->plan;
    const uint32_t sb = SB ? SB : w->scale_bits;
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const uint32_t n_blocks = p.n_blocks, block_size = p.block_size, chunk_syms = p.chunk_syms;
    const uint32_t per_block = block_size / chunk_syms;
    const uint64_t blob_bytes = p.blob_bytes;
    const uint16_t* models = reinterpret_cast<const uint16_t*>(buf + sizeof(ContainerHeader));
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + p.dir_off);
    const uint8_t* blob = buf + p.blob_off;
    // the word coder takes its table's address per chunk: hoisted, it goes to a uniform register and the step changes
    const uint32_t ring = smem_addr(s_bdec) + warp * kRingBytes;
    const uint32_t tab = CODER == RB200_CODER_WORD ? 0 : smem_addr_pinned(s_bdec + kPlannedWarps * kRingBytes);
    for (;;) {
        __syncthreads();                                             // the previous block's table is no longer in use
        if (tid == 0) s_block = atomicAdd(&w->next_block, 1u);
        __syncthreads();
        const uint32_t block = s_block;
        if (block >= n_blocks) break;
        // a model that does not sum was refused by the prefix check: not reached
        if (!block_decode_table<CODER, SB>(models + static_cast<uint64_t>(block) * 256, 1u << sb, s_cum, s_flag, s_bdec, kPlannedWarps)) {
            if (tid == 0) atomicOr(status, kStatStream);
            continue;
        }
        const bool wide = CODER == RB200_CODER_WORD && s_flag[1];
        for (uint32_t k = warp; k < per_block; k += kPlannedWarps) {
            uint8_t* dst = out + static_cast<uint64_t>(block) * block_size + static_cast<uint64_t>(k) * chunk_syms;
            block_decode_chunk<CODER, SB>(blob, blob_bytes, offsets, block * per_block + k, ring,
                                          CODER == RB200_CODER_WORD ? smem_addr_pinned(s_bdec + kPlannedWarps * kRingBytes) : tab, sb, wide, dst,
                                          chunk_syms, status);
        }
    }
    // every CTA has taken its last block id before it counts itself out: the last one re-arms the counter
    if (tid == 0 && atomicAdd(&w->ctas_done, 1u) == gridDim.x - 1) {
        w->next_block = 0;
        w->ctas_done = 0;
    }
}

// The version 1 decoders.  Each takes the geometry, the table and its counter from the call's ContainerAsyncWork and runs
// only when go is its id.  Word and alias: the shipped persistent kernels' CTA set-up around decode_persistent with the
// shipped policies; byte and rans64: the shipped kernels' table staging around a counter-driven loop over
// decode_window_chunk (their own kernels launch one warp per chunk, a grid only the host can size).

template <bool WIDE>
__global__ void __launch_bounds__(DecShip::kWarps * 32, DecShip::kMinBlocks)
    word_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, ContainerAsyncWork* __restrict__ w,
                               uint32_t* __restrict__ status)
{
    using P = DecShip;
    static_assert(P::kRefill == kRefillCpAsync, "the ring's mbarriers are not initialised here: cp.async refill only");
    if (w->go != (WIDE ? kDecWordWide : kDecWord)) return;        // the same for the whole grid
    const BlocksPlan p = w->plan;
    extern __shared__ __align__(1024) uint8_t s_dec[];     // [16 KiB table][table mbarrier][kWarps x (ring, mirror, mbarriers)]
    const uint32_t tab = smem_addr_pinned(s_dec);
    const uint32_t bar_tab = tab + kWordSlots * 4;
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);       // warp-uniform for ptxas
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t ring = tab + P::kWarpsOff + warp * P::kWarpStride;

    if (threadIdx.x == 0) mbar_init(bar_tab, 1);
    mbar_fence_init();
    __syncthreads();
    if (threadIdx.x == 0) {                                // the table for the whole CTA: one 16 KiB bulk copy
        mbar_arrive_expect_tx(bar_tab, kWordSlots * 4);
        bulk_g2s(tab, w->table, kWordSlots * 4, bar_tab);
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
    decode_persistent<P>(WordDecoder<WIDE>{tab, 0}, ring, buf + p.blob_off, p.blob_bytes, reinterpret_cast<const uint64_t*>(buf + p.dir_off),
                         out, p.n_symbols, p.chunk_syms, static_cast<uint32_t>(p.n_chunks), &w->work, lane, status);
}

template <uint32_t SB>
__global__ void __launch_bounds__(AliasDecShip::kWarps * 32, AliasDecShip::kMinBlocks)
    alias_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, ContainerAsyncWork* __restrict__ w,
                                uint32_t* __restrict__ status)
{
    using P = AliasDecShip;
    if (w->go != kDecAlias + sb_variant(SB)) return;
    const BlocksPlan p = w->plan;
    const uint32_t sb_rt = w->scale_bits;
    const AliasDecEntry* g_dec = reinterpret_cast<const AliasDecEntry*>(w->table);
    extern __shared__ __align__(1024) uint8_t s_adec[];       // [32 KiB table][16 B][kWarps x (ring, mirror)]
    uint4* s_tab = reinterpret_cast<uint4*>(s_adec);
    for (uint32_t i = threadIdx.x; i < 256 * kAliasDecReplicas; i += blockDim.x) {
        const AliasDecEntry e = g_dec[i / kAliasDecReplicas];
        if (kAliasLean && SB > 8) s_tab[i] = alias_lean_entry<(SB > 8 ? SB : 9)>(e, i / kAliasDecReplicas);
        else s_tab[i] = make_uint4(e.divider, e.alt0, e.alt1, e.adjust);
    }
    __syncthreads();

    const uint32_t base = smem_addr_pinned(s_adec);
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const uint32_t lane = threadIdx.x & 31;
    const AliasDecoder<SB, kAliasLean> coder = {base + (lane & (kAliasDecReplicas - 1)) * 16, sb_rt};
    decode_persistent<P>(coder, base + P::kWarpsOff + warp * P::kWarpStride, buf + p.blob_off, p.blob_bytes,
                         reinterpret_cast<const uint64_t*>(buf + p.dir_off), out, p.n_symbols, p.chunk_syms, static_cast<uint32_t>(p.n_chunks),
                         &w->work, lane, status);
}

// Every warp of the grid takes chunk ids from w->work until none is left and decodes each through its 1 KiB stream
// window at shared address `ring`; the last warp out re-arms the counter.
template <class C>
__device__ __forceinline__ void decode_window_planned(const C& coder, const uint8_t* __restrict__ buf, uint8_t* __restrict__ out,
                                                      ContainerAsyncWork* __restrict__ w, uint32_t ring, uint32_t* __restrict__ status)
{
    const BlocksPlan p = w->plan;
    const uint8_t* blob = buf + p.blob_off;
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + p.dir_off);
    const uint32_t lane = threadIdx.x & 31, n_chunks = static_cast<uint32_t>(p.n_chunks);
    for (;;) {
        uint32_t chunk = 0;
        if (lane == 0) chunk = atomicAdd(&w->work.next_chunk, 1u);
        chunk = __shfl_sync(0xffffffffu, chunk, 0);       // also orders the previous chunk's ring reads before the next fill
        if (chunk >= n_chunks) break;
        const uint64_t first = static_cast<uint64_t>(chunk) * p.chunk_syms;
        const uint32_t m = static_cast<uint32_t>(min(static_cast<uint64_t>(p.chunk_syms), p.n_symbols - first));
        decode_window_chunk(coder, blob, p.blob_bytes, offsets, chunk, ring, out + first, m, status);
    }
    if (lane == 0 && atomicAdd(&w->work.warps_done, 1u) == gridDim.x * (blockDim.x / 32) - 1) {
        w->work.next_chunk = 0;
        w->work.warps_done = 0;
    }
}

// dynamic shared memory of the byte decoder: 16 rings, 256 symbol entries and cum2sym at the largest scale_bits the
// variant decodes (the generic one: 15)
__host__ __device__ constexpr uint32_t byte_planned_smem(uint32_t SB) { return kAliasDecWarps * kRingBytes + 1024 + (1u << (SB ? SB : 15)); }

template <uint32_t SB>
__global__ void __launch_bounds__(kAliasDecWarps * 32, 4)
    byte_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, ContainerAsyncWork* __restrict__ w,
                               uint32_t* __restrict__ status)
{
    if (w->go != kDecByte + sb_variant(SB)) return;
    const uint32_t sb = SB ? SB : w->scale_bits;
    extern __shared__ __align__(1024) uint8_t s_adec[];       // [16 x 1 KiB rings][table]
    uint4* s_tab = reinterpret_cast<uint4*>(s_adec + kAliasDecWarps * kRingBytes);
    const uint32_t vecs = ((1u << sb) + 1024) / 16;
    for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) s_tab[i] = reinterpret_cast<const uint4*>(w->table)[i];
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5;
    decode_window_planned(ByteDecoder<SB>{smem_addr_pinned(s_tab), sb}, buf, out, w, smem_addr(s_adec) + warp * kRingBytes, status);
}

constexpr uint32_t kRans64PlannedSmem = kRans64Warps * kRingBytes + kRans64DecSymBytes + (1u << 16);

__global__ void __launch_bounds__(kRans64Warps * 32, 2)
    rans64_decode_planned_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ out, ContainerAsyncWork* __restrict__ w,
                                 uint32_t* __restrict__ status)
{
    if (w->go != kDecRans64) return;
    const uint32_t sb = w->scale_bits;
    extern __shared__ __align__(1024) uint8_t s_r64[];        // [16 x 1 KiB rings][cum2sym][256 x 16 replicas x {start, freq}]
    uint4* s_tab = reinterpret_cast<uint4*>(s_r64 + kRans64Warps * kRingBytes);
    const uint32_t vecs = (1u << sb) / 16;
    for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) s_tab[i] = reinterpret_cast<const uint4*>(w->table)[i];
    {
        const uint2* g_syms = reinterpret_cast<const uint2*>(w->table + (1u << sb));
        uint2* s_syms = reinterpret_cast<uint2*>(s_r64 + kRans64Warps * kRingBytes + (1u << sb));
        for (uint32_t i = threadIdx.x; i < 256 * kRans64DecReplicas; i += blockDim.x) s_syms[i] = g_syms[i / kRans64DecReplicas];
    }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tab = smem_addr(s_tab);
    const Rans64Decoder coder = {tab, tab + (1u << sb) + (lane & (kRans64DecReplicas - 1)) * 8, sb};
    decode_window_planned(coder, buf, out, w, smem_addr(s_r64) + warp * kRingBytes, status);
}

// One launch of a decoder: kernel, grid, threads, dynamic shared memory.
struct DecoderLaunch {
    void (*kernel)(const uint8_t*, uint8_t*, ContainerAsyncWork*, uint32_t*);
    uint32_t grid, threads, smem;
    const char* name;
};

// The decoders of every version in one launch table, each version's in id order: version v's are the entries
// kDecoderFirst[v - 1] .. kDecoderFirst[v] - 1.
constexpr int kDecoderFirst[] = {0, 11, 12, 16, 19};
constexpr int kContainerDecoders = kDecoderFirst[4];
// the prefix check's grid: kPrefixCtasPerSm CTAs of kPrefixWarps warps per SM
constexpr uint32_t kPrefixCtasPerSm = 8;

// The launch table, fixed per device: each decoder's grid is every CTA that is resident at once (the version 1 word and
// alias grids are the shipped kernels' full grids); the generic byte and rans64 decoders get shared memory for the
// largest scale_bits they decode, the version 4 ones the alias bucket table, whose size does not depend on scale_bits.
inline void configure_container_decode(uint32_t sms, DecoderLaunch* out)
{
    constexpr uint32_t planned = kPlannedWarps * 32;
    const DecoderLaunch l[kContainerDecoders] = {
        {word_decode_planned_kernel<false>, sms * DecShip::kMinBlocks, DecShip::kWarps * 32, DecShip::kSmemBytes, "word_decode_planned_kernel"},
        {word_decode_planned_kernel<true>, sms * DecShip::kMinBlocks, DecShip::kWarps * 32, DecShip::kSmemBytes, "word_decode_planned_kernel(wide)"},
        {alias_decode_planned_kernel<16>, sms * AliasDecShip::kMinBlocks, AliasDecShip::kWarps * 32, AliasDecShip::kSmemBytes, "alias_decode_planned_kernel<16>"},
        {alias_decode_planned_kernel<14>, sms * AliasDecShip::kMinBlocks, AliasDecShip::kWarps * 32, AliasDecShip::kSmemBytes, "alias_decode_planned_kernel<14>"},
        {alias_decode_planned_kernel<12>, sms * AliasDecShip::kMinBlocks, AliasDecShip::kWarps * 32, AliasDecShip::kSmemBytes, "alias_decode_planned_kernel<12>"},
        {alias_decode_planned_kernel<0>, sms * AliasDecShip::kMinBlocks, AliasDecShip::kWarps * 32, AliasDecShip::kSmemBytes, "alias_decode_planned_kernel<0>"},
        {byte_decode_planned_kernel<16>, 0, kAliasDecWarps * 32, byte_planned_smem(16), "byte_decode_planned_kernel<16>"},
        {byte_decode_planned_kernel<14>, 0, kAliasDecWarps * 32, byte_planned_smem(14), "byte_decode_planned_kernel<14>"},
        {byte_decode_planned_kernel<12>, 0, kAliasDecWarps * 32, byte_planned_smem(12), "byte_decode_planned_kernel<12>"},
        {byte_decode_planned_kernel<0>, 0, kAliasDecWarps * 32, byte_planned_smem(0), "byte_decode_planned_kernel<0>"},
        {rans64_decode_planned_kernel, 0, kRans64Warps * 32, kRans64PlannedSmem, "rans64_decode_planned_kernel"},
        {block_decode_planned_kernel<RB200_CODER_WORD, kWordScaleBits>, 0, planned, 0, "block_decode_planned_kernel<word, 12>"},
        {block_decode_planned_kernel<RB200_CODER_BYTE, 14>, 0, planned, block_coder_decode_smem(RB200_CODER_BYTE, 14, planned),
         "block_decode_planned_kernel<byte, 14>"},
        {block_decode_planned_kernel<RB200_CODER_BYTE, 12>, 0, planned, block_coder_decode_smem(RB200_CODER_BYTE, 12, planned),
         "block_decode_planned_kernel<byte, 12>"},
        {block_decode_planned_kernel<RB200_CODER_BYTE, 0>, 0, planned,
         block_coder_decode_smem(RB200_CODER_BYTE, kBlockCoderMaxScaleBits, planned), "block_decode_planned_kernel<byte, 0>"},
        {block_decode_planned_kernel<RB200_CODER_RANS64, 0>, 0, planned,
         block_coder_decode_smem(RB200_CODER_RANS64, kBlockCoderMaxScaleBits, planned), "block_decode_planned_kernel<rans64, 0>"},
        {block_decode_planned_kernel<RB200_CODER_ALIAS, 14>, 0, planned, block_coder_decode_smem(RB200_CODER_ALIAS, 14, planned),
         "block_decode_planned_kernel<alias, 14>"},
        {block_decode_planned_kernel<RB200_CODER_ALIAS, 12>, 0, planned, block_coder_decode_smem(RB200_CODER_ALIAS, 12, planned),
         "block_decode_planned_kernel<alias, 12>"},
        {block_decode_planned_kernel<RB200_CODER_ALIAS, 0>, 0, planned,
         block_coder_decode_smem(RB200_CODER_ALIAS, kBlockCoderMaxScaleBits, planned), "block_decode_planned_kernel<alias, 0>"},
    };
    for (int i = 0; i < kContainerDecoders; i++) {
        out[i] = l[i];
        cudaFuncSetAttribute(l[i].kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(l[i].kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(l[i].smem));
        if (!out[i].grid) {
            int per_sm = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, l[i].kernel, static_cast<int>(l[i].threads), l[i].smem);
            out[i].grid = sms * static_cast<uint32_t>(per_sm < 1 ? 1 : per_sm);
        }
    }
}

}  // namespace rb200

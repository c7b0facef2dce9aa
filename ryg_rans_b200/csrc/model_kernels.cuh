// model_kernels.cuh -- rb200_container_model_encode_async: a single-model (version 1) container whose model is built
// from the data on the GPU, so that the whole encode only enqueues work (and can be captured in a CUDA graph).
//
// The stages run in stream order on the context's stream (rans_b200.cu); each reads what the one before it left in the
// context's ModelAsyncWork:
//   memset + histogram_kernel   the data's 256 counts into counts[]
//   container_model_kernel      one CTA: calc_cum_freqs + normalize_freqs(1 << scale_bits) on the counts, bit-exact
//                               (block_normalize); the checks of rb200_model_create (kStatModel on refusal); the coder's
//                               encode tables, byte for byte what rb200_model_create uploads (tables.h formulas)
//   the coder's encoder         the shipped kernel with its table pointers into the workspace.  The word coder runs
//                               both GATED instances of K2 or K2f (word_kernels.cuh); r32 names the one that encodes,
//                               the other exits before it touches the counter, look[] or scratch
//   crc32_kernel x 1-2, container_finish_kernel
//                               as rb200_container_encode in device memory, with the model section from freqs[]
//
// rb200_container_model_encode_varlen_async runs the same stages on launch shapes the host sizes for a bound n_max,
// and reads the length from device memory: varlen_plan_kernel checks *d_n and writes the geometry record (VarlenGeom,
// device_utils.cuh) into geom; every later kernel is the GEOM instance of the same kernel, which takes n, the chunk
// count and the directory's and blob's places from there and exits at entry when the checks failed.
//
// rb200_container_model_encode_auto_async runs coder_choice_kernel after the histogram: it applies the rule of
// rb200_choose_coder to the counts and writes the choice record (CoderChoice).  The CHOSEN instance of the model kernel
// builds the chosen coder's tables from it; the host launches one gated group per distinct encoder instance the list
// needs (word: both GATED instances, whose gate r32 the model kernel closes for other coders; alias/byte per SB
// instance; rans64), each with its own directory and compaction when split, and only the recorded group runs; the
// CHOSEN instance of container_finish_kernel writes the chosen coder and scale_bits into the header.
//
// rb200_container_blocks_model_encode_auto_async does the same for the per-block containers (versions 2-4):
// blocks_choice_kernel applies the rule of rb200_choose_blocks_coder block by block and writes BlocksChoice
// (device_utils.cuh); one gated group per distinct per-block encoder instance follows (the GATED instances of
// block_encode_fused_kernel and block_coder_encode_kernel, with C7's GATED scan, prefix and compaction), then the CRCs
// and container_blocks_finish_kernel, which writes version, coder and scale_bits from the record.
//
// rb200_container_blocks_model_encode_varlen_async runs those stages on launch shapes sized for n_blocks_max:
// blocks_varlen_plan_kernel reads *d_n_blocks into BlocksVarlenGeom (device_utils.cuh), and the choice kernel, the
// encoders, the scan and compaction, the blob length and the header kernel are the GEOM instances of the same kernels,
// which take the count, the directory's place (after the count's models) and the blob's from it.
//
// rb200_container_blocks_stored_encode_async (version 5) runs the choice kernel (blocks_one_pair_kernel for one
// candidate) and one GATED split encoder per group into one workspace, then blocks_store_kernel, which stores every
// block whose coded chunks take more blob than its symbols, and one ungated scan and compact_stored_kernel.
//
// rb200_container_stored_encode_async (version 6) runs the histogram, the choice and the CHOSEN model kernel of the auto
// encode, then one GATED split encoder per group into one workspace, chunks_store_kernel, which stores every chunk whose
// stream is longer than its symbols and writes the bitmap, one ungated scan and chunks_stored_compaction_kernel.
//
// rb200_container_stored_encode_varlen_async and rb200_container_blocks_stored_encode_varlen_async run those two on
// launch shapes sized for the bound: stored_varlen_plan_kernel (StoredVarlenGeom, device_utils.cuh) or
// blocks_varlen_plan_kernel reads the size, and every later kernel is the GEOM instance of the same stage
// (chunks_store_varlen_kernel, blocks_store_varlen_kernel and the *_varlen_kernel compactions and header kernels).
#pragma once
#include "block_kernels.cuh"
#include "container_format.h"
#include "tables.h"
#include "word_kernels.cuh"

namespace rb200 {

// The call's workspace: fixed-size (about 170 KiB), allocated with the context, so the call never allocates for the
// model.  Every table has the layout of its rb200_model counterpart.
struct ModelAsyncWork {
    unsigned long long counts[256];               // the histogram; zeroed in stream order before each call
    uint32_t freqs[256];                          // the normalised model: the container's model section
    uint32_t r32;                                 // the word encoder to run: 1 the 32-bit reciprocal instance, 0 the 33-bit
    alignas(16) WordEncEntry word_enc[256];       // word: 33-bit reciprocals (WordDeviceTables::enc)
    alignas(16) WordEncEntry word_enc32[256];     // word: 32-bit reciprocals (WordDeviceTables::enc32)
    alignas(16) AliasEncEntry alias_enc[256];
    alignas(16) AliasEncEntry byte_enc[256];      // RansEncSymbol images
    alignas(16) uint4 r64_enc[256 * 2];           // Rans64EncSymbol images, 32 bytes each
    alignas(16) uint16_t alias_remap[1u << 16];   // the first 1 << scale_bits entries are the model's
    VarlenGeom geom;                              // rb200_container_model_encode_varlen_async: the length and layout of this run
    alignas(16) CoderChoice choice;               // rb200_container_model_encode_auto_async: the choice of this run
    uint32_t cand_freqs[kMaxCandidates][256];     // its candidates' models; the chosen row is the container's
};

constexpr uint32_t kWordGateClosed = 2;          // r32 when the auto encode chose another coder: neither word instance runs

constexpr int kModelThreads = 256;                // one thread per symbol

// coder and scale_bits are valid (the host checks them); r32_allowed is word_r32_allowed().  A model
// rb200_model_create refuses sets kStatModel, and the tables are written all the same (the encoders then run on
// well-formed entries, and container_finish_kernel writes no header).  Normalisation itself cannot fail for targets
// >= 256: a squashed symbol needs a donor of width > 1, and while any symbol is squashed the widths, which sum to the
// target, cannot all be <= 1.  block_normalize keeps its check all the same, with kStatModel as the verdict.
// GEOM (the device-length call): with *d_n == 0 the counts are all zero and normalisation has no total to scale, so it
// runs only when the plan passed.
// CHOSEN (the auto encode): coder, scale_bits and the normalised model come from the choice record (coder_choice_kernel
// normalised every candidate); the arguments coder and sb are unused.  Another coder than word closes both word gates.
template <bool GEOM = false, bool CHOSEN = false>
__global__ void __launch_bounds__(kModelThreads)
    container_model_kernel(uint32_t coder, uint32_t sb, uint32_t r32_allowed, ModelAsyncWork* __restrict__ w, uint32_t* __restrict__ status)
{
    if (GEOM && !w->geom.go) return;
    if (CHOSEN) {
        coder = w->choice.coder;
        sb = w->choice.scale_bits;
    }
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];
    __shared__ uint32_t s_divider[256], s_adjust[512], s_slot_freqs[512], s_rest[256], s_given[256];
    __shared__ uint8_t s_sym_id[512];
    __shared__ uint32_t s_paired;
    const uint32_t tid = threadIdx.x, M = 1u << sb;
    if (CHOSEN) {
        s_w[tid] = w->freqs[tid] = w->cand_freqs[w->choice.index][tid];
    } else {
        s_cnt[tid] = static_cast<uint32_t>(w->counts[tid]);    // n < 2^32, so every count and their sum fit
        __syncthreads();
        if (tid < 32) block_normalize(s_cnt, s_cum, s_w, w->freqs, M, kStatModel, status);
    }
    __syncthreads();
    if (tid == 0) {
        bool ok = container_model_ok(coder, sb, s_w) && container_model_decodable(coder, s_w);
        uint32_t c = 0;
        for (int s = 0; s < 256; s++) {
            s_cum[s] = c;
            c += s_w[s];
        }
        s_cum[256] = c;
        bool paired = false;
        if (ok && coder == RB200_CODER_ALIAS) {
            paired = alias_tables_core(s_w, M / 256, s_divider, s_adjust, s_slot_freqs, s_sym_id, s_rest, s_given);
            ok = paired;
        }
        s_paired = paired;
        if (!ok) atomicOr(status, kStatModel);
    }
    __syncthreads();
    const uint32_t f = s_w[tid], cum = s_cum[tid];
    if (CHOSEN && coder != RB200_CODER_WORD && tid == 0) w->r32 = kWordGateClosed;
    if (coder == RB200_CODER_WORD) {
        int exact = 1;
        w->word_enc[tid] = word_enc_entry(f, cum);
        w->word_enc32[tid] = word_enc32_entry(f, cum, &exact);
        const bool r32 = __syncthreads_and(exact) != 0;
        if (tid == 0) w->r32 = r32 && r32_allowed;
    } else if (coder == RB200_CODER_ALIAS) {
        w->alias_enc[tid] = alias_enc_entry(f, cum);
        if (s_paired) {
            // alias_remap as rb200_alias_tables_build fills it: bucket b gives its own part to symbol b and the rest to
            // its partner, each after what earlier buckets gave that symbol; one thread per code slot
            const uint32_t bucket = M / 256;
            for (uint32_t i = tid; i < M; i += kModelThreads) {
                const uint32_t b = i / bucket, k = i - b * bucket, lo = b * bucket, own = s_divider[b] - lo;
                const uint32_t dst = k < own ? s_cum[b] + (lo - s_adjust[2 * b + 1]) + k
                                             : s_cum[s_sym_id[2 * b]] + (lo + own - s_adjust[2 * b]) + (k - own);
                w->alias_remap[dst] = static_cast<uint16_t>(lo + k);
            }
        }
    } else if (coder == RB200_CODER_BYTE) {
        w->byte_enc[tid] = byte_enc_entry(f, cum, sb);
    } else {
        uint32_t e[8];
        rans64_enc_entry(f, cum, sb, e);
        w->r64_enc[2 * tid] = make_uint4(e[0], e[1], e[2], e[3]);
        w->r64_enc[2 * tid + 1] = make_uint4(e[4], e[5], e[6], e[7]);
    }
}

// The candidate list of rb200_container_model_encode_auto_async, by value: the pairs (RB200_CANDIDATE) and the launch
// group of each (the host's numbering: one group per distinct encoder instance).
struct CandidateList {
    uint32_t pair[kMaxCandidates];
    uint32_t group[kMaxCandidates];
    uint32_t n, tolerance_ppm;
};

// The rule of rb200_choose_coder (container_format.h) on the histogram, one CTA with one warp per candidate: warp i
// normalises the counts to 1 << sb_i into cand_freqs[i] (block_normalize, bit-exact), checks the model as the fixed
// call would, and sums its bits_q; thread 0 then applies the rule and writes the choice record.  No feasible candidate
// sets kStatModel and records the first one, whose tables the model kernel then builds as the fixed call would (the
// header is never written).  n_chunks is the fixed call's; geom set: the device-length call, which takes it from the
// record and runs only when the plan passed.
__global__ void __launch_bounds__(kMaxCandidates * 32)
    coder_choice_kernel(CandidateList list, uint64_t n_chunks, ModelAsyncWork* __restrict__ w, const VarlenGeom* __restrict__ geom,
                        uint32_t* __restrict__ status)
{
    if (geom) {
        if (!geom->go) return;
        n_chunks = geom->n_chunks;
    }
    __shared__ uint32_t s_cnt[256], s_cum[kMaxCandidates][257], s_fail[kMaxCandidates];
    __shared__ __align__(16) uint32_t s_w[kMaxCandidates][256];
    __shared__ uint64_t s_cost[kMaxCandidates];
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (uint32_t s = tid; s < 256; s += blockDim.x) s_cnt[s] = static_cast<uint32_t>(w->counts[s]);   // n < 2^32
    if (lane == 0) s_fail[warp] = 0;
    __syncthreads();
    const uint32_t coder = list.pair[warp] >> 8, sb = list.pair[warp] & 0xffu;
    uint32_t* f = s_w[warp];
    block_normalize(s_cnt, s_cum[warp], f, w->cand_freqs[warp], 1u << sb, 1u, &s_fail[warp]);
    __syncwarp();
    // container_model_ok and container_model_decodable, spread over the warp (the pair itself is valid): the model sums
    // to 1 << sb, and the byte coder's frequencies stay below 65536
    uint64_t bits_q = 0;
    uint32_t sum = 0, top = 0;
    for (uint32_t s = lane; s < 256; s += 32) {
        bits_q += candidate_bits_q(s_cnt[s], f[s], sb);
        sum += f[s];
        top = max(top, f[s]);
    }
    for (int d = 16; d; d >>= 1) bits_q += __shfl_xor_sync(0xffffffffu, bits_q, d);
    sum = __reduce_add_sync(0xffffffffu, sum);
    top = __reduce_max_sync(0xffffffffu, top);
    if (lane == 0) {
        const bool ok = !s_fail[warp] && sum == (1u << sb) && (coder != RB200_CODER_BYTE || top < 65536u);
        s_cost[warp] = ok ? candidate_cost(bits_q, n_chunks, coder) : ~0ull;
    }
    __syncthreads();
    if (tid < list.n) w->choice.costs[tid] = s_cost[tid];
    if (tid == 0) {
        const int k = choose_candidate(s_cost, list.n, list.tolerance_ppm);
        if (k < 0) atomicOr(status, kStatModel);
        const uint32_t i = k < 0 ? 0u : static_cast<uint32_t>(k);
        w->choice.coder = list.pair[i] >> 8;
        w->choice.scale_bits = list.pair[i] & 0xffu;
        w->choice.index = i;
        w->choice.group = list.group[i];
    }
}

constexpr int kBlocksChoiceWarps = 8;
constexpr uint32_t kBlocksChoiceRowWords = 784;  // a warp's rows over the free histogram: widths, model, cumulative (16-byte aligned)

// The rule of rb200_choose_blocks_coder, one CTA per block: count_freqs with the bank-private histogram
// (block_histogram_wide, as K5f's model build), then warp w takes candidates w, w + 8: block_normalize to 1 << sb_i
// (the device normaliser every per-block encoder uses, bit-exact), bits_q by warp reduction, and the block's cost
// (blocks_candidate_cost) added into sums[i].  Every candidate is feasible on every block (byte at <= 15 stays below
// 65536, a model that sums always pairs, word takes 4096 through WIDE), so there is no infeasible cost.  The last CTA
// out applies choose_candidate and writes the record.
// GEOM (rb200_container_blocks_model_encode_varlen_async): the block count from the record (BlocksVarlenGeom), on the
// grid of n_blocks_max; the CTAs at or past it exit at entry, before they count, so the last of the device count's CTAs
// is the last out (none runs when the plan failed: n_blocks is then 0).
template <bool GEOM = false>
__global__ void __launch_bounds__(kBlocksChoiceWarps * 32)
    blocks_choice_kernel(CandidateList list, const uint8_t* __restrict__ in, uint32_t block_size, uint32_t chunk_syms, BlocksChoice* r,
                         uint32_t* __restrict__ status, const BlocksVarlenGeom* __restrict__ geom)
{
    if (GEOM && blockIdx.x >= geom->n_blocks) return;            // the same for the whole CTA
    __shared__ __align__(16) uint32_t s_hist[256 * 32];          // the histogram copies, then the warps' rows
    __shared__ uint32_t s_cnt[256];
    __shared__ uint64_t s_cost[kMaxCandidates];
    __shared__ uint32_t s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    block_histogram_wide(in + static_cast<uint64_t>(blockIdx.x) * block_size, block_size, s_hist, s_cnt);
    static_assert(kBlocksChoiceWarps * kBlocksChoiceRowWords <= 256 * 32, "the rows fit the histogram's place");
    uint32_t* s_w = s_hist + warp * kBlocksChoiceRowWords;       // 256 widths, 256 frequencies, 257 cumulative
    uint32_t* s_f = s_w + 256;
    uint32_t* s_cum = s_w + 512;
    for (uint32_t i = warp; i < list.n; i += kBlocksChoiceWarps) {
        const uint32_t coder = list.pair[i] >> 8, sb = list.pair[i] & 0xffu;
        block_normalize(s_cnt, s_cum, s_w, s_f, 1u << sb, kStatStream, status);
        __syncwarp();
        uint64_t bits_q = 0;
        bool one_symbol = false;
        for (uint32_t s = lane; s < 256; s += 32) {
            bits_q += candidate_bits_q(s_cnt[s], s_f[s], sb);
            one_symbol |= s_f[s] == (1u << sb);
        }
        for (int d = 16; d; d >>= 1) bits_q += __shfl_xor_sync(0xffffffffu, bits_q, d);
        one_symbol = __any_sync(0xffffffffu, one_symbol);
        if (lane == 0) atomicAdd(&r->sums[i], static_cast<unsigned long long>(blocks_candidate_cost(bits_q, block_size, chunk_syms, coder, one_symbol)));
        __syncwarp();
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();                                         // this CTA's sums before its count
        s_last = atomicAdd(&r->done, 1u) == (GEOM ? geom->n_blocks : gridDim.x) - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid < list.n) s_cost[tid] = r->choice.costs[tid] = __ldcg(&r->sums[tid]);
    __syncthreads();
    if (tid == 0) {
        const int k = choose_candidate(s_cost, list.n, list.tolerance_ppm);   // every cost is finite: k >= 0
        const uint32_t i = k < 0 ? 0u : static_cast<uint32_t>(k);
        r->choice.coder = list.pair[i] >> 8;
        r->choice.scale_bits = list.pair[i] & 0xffu;
        r->choice.index = i;
        r->choice.group = list.group[i];
        r->version = container_blocks_version(r->choice.coder);
    }
}

// rb200_container_blocks_stored_encode_async with one candidate, one thread: the choice record of that pair as group 0,
// which the gated encoders and the header kernel read (no choice kernel runs; its costs are left as they are)
__global__ void __launch_bounds__(32) blocks_one_pair_kernel(uint32_t pair, BlocksChoice* __restrict__ r)
{
    if (threadIdx.x) return;
    r->choice.coder = pair >> 8;
    r->choice.scale_bits = pair & 0xffu;
    r->choice.index = 0;
    r->choice.group = 0;
    r->version = container_blocks_version(r->choice.coder);
}

// The store rule of rb200_container_blocks_stored_encode_async, one warp per block, after the encoder wrote every chunk's
// stream size to sizes[]: the blob bytes of the block's chunks (each stream rounded up to 16, as the compaction places
// it) against per_block x round16(chunk_syms), its size stored.  Above that the block is stored: its model row in the
// container is zeroed, every chunk's size becomes round16(chunk_syms), and stored[block] = 1 has the compaction copy
// the chunk's symbols in place of its stream; otherwise stored[block] = 0.  Stream sizes stay below 2^26 (a slot), so
// a block's sum fits 32 bits.
// GEOM (rb200_container_blocks_stored_encode_varlen_async): on the grid of n_blocks_max, the count from the record
// (BlocksVarlenGeom, 0 when the plan failed); the models stay at out + 64, so nothing else moves.
constexpr int kStoreWarps = 8;

template <bool GEOM>
__device__ __forceinline__ void blocks_store(uint32_t* __restrict__ sizes, uint32_t n_blocks, uint32_t per_block, uint32_t chunk_syms,
                                             uint16_t* __restrict__ models, uint32_t* __restrict__ stored,
                                             const BlocksVarlenGeom* __restrict__ geom)
{
    if (GEOM) n_blocks = geom->n_blocks;
    const uint32_t lane = threadIdx.x & 31, block = blockIdx.x * kStoreWarps + (threadIdx.x >> 5);
    if (block >= n_blocks) return;                               // the same for the whole warp
    const uint32_t raw = static_cast<uint32_t>(container_stored_bytes(chunk_syms));
    uint32_t* s = sizes + static_cast<uint64_t>(block) * per_block;
    const uint32_t coded = __reduce_add_sync(0xffffffffu, lane < per_block ? (s[lane] + 15u) & ~15u : 0u);
    const bool store = coded > per_block * raw;
    if (lane == 0) stored[block] = store;
    if (!store) return;
    if (lane < per_block) s[lane] = raw;
    reinterpret_cast<uint4*>(models + static_cast<uint64_t>(block) * 256)[lane] = make_uint4(0, 0, 0, 0);   // 32 x 16 bytes
}

__global__ void __launch_bounds__(kStoreWarps * 32)
    blocks_store_kernel(uint32_t* __restrict__ sizes, uint32_t n_blocks, uint32_t per_block, uint32_t chunk_syms, uint16_t* __restrict__ models,
                        uint32_t* __restrict__ stored)
{
    blocks_store<false>(sizes, n_blocks, per_block, chunk_syms, models, stored, nullptr);
}

__global__ void __launch_bounds__(kStoreWarps * 32)
    blocks_store_varlen_kernel(uint32_t* __restrict__ sizes, uint32_t per_block, uint32_t chunk_syms, uint16_t* __restrict__ models,
                               uint32_t* __restrict__ stored, const BlocksVarlenGeom* __restrict__ geom)
{
    blocks_store<true>(sizes, 0, per_block, chunk_syms, models, stored, geom);
}

// The store rule of rb200_container_stored_encode_async (version 6), one thread per chunk, after the encoder wrote every
// chunk's stream size to sizes[]: chunk c is stored when its stream, rounded up to 16 as the compaction places it, is
// longer than round16(m_c), its symbols' stored size; ties stay coded.  A stored chunk's size becomes round16(m_c) and
// stored[c] = 1 has the compaction copy its symbols in place of its stream; otherwise stored[c] = 0.  Each warp's ballot
// is one word of the container's bitmap: the grid covers the padding words too, which it writes zero, and thread 0
// zeroes the pad between the directory and the bitmap, both of which meta_crc covers.
// GEOM (rb200_container_stored_encode_varlen_async): on the grid of n_max's bitmap words, n and the chunk count from the
// record (VarlenGeom); the bitmap's place and its words follow that count, and the CTAs past its words exit at entry,
// so nothing is written for the bound's extra words.  Every CTA exits when the plan failed.
constexpr int kChunkStoreThreads = 256;

template <bool GEOM>
__device__ __forceinline__ void chunks_store(uint32_t* __restrict__ sizes, uint32_t n_chunks, uint64_t n, uint32_t chunk_syms,
                                             uint8_t* __restrict__ out, uint32_t* __restrict__ stored, const VarlenGeom* __restrict__ geom)
{
    if (GEOM) {
        if (!geom->go) return;
        n_chunks = geom->n_chunks;
        n = geom->n;
        if (static_cast<uint64_t>(blockIdx.x) * kChunkStoreThreads >= container_bitmap_words(n_chunks) * 32) return;
    }
    const uint64_t c = static_cast<uint64_t>(blockIdx.x) * kChunkStoreThreads + threadIdx.x;
    bool store = false;
    if (c < n_chunks) {
        const uint32_t raw = static_cast<uint32_t>(container_stored_bytes(container_chunk_symbols(c, chunk_syms, n)));
        store = ((sizes[c] + 15u) & ~15u) > raw;
        stored[c] = store;
        if (store) sizes[c] = raw;
    }
    const uint32_t word = __ballot_sync(0xffffffffu, store);
    const uint64_t bitmap = container_bitmap_offset(n_chunks), dir_end = kContainerDirOffset + (n_chunks + 1) * sizeof(uint64_t);
    if ((threadIdx.x & 31) == 0 && c / 32 < container_bitmap_words(n_chunks)) reinterpret_cast<uint32_t*>(out + bitmap)[c / 32] = word;
    if (c == 0 && bitmap > dir_end) *reinterpret_cast<uint64_t*>(out + dir_end) = 0;
}

__global__ void __launch_bounds__(kChunkStoreThreads)
    chunks_store_kernel(uint32_t* __restrict__ sizes, uint32_t n_chunks, uint64_t n, uint32_t chunk_syms, uint8_t* __restrict__ out,
                        uint32_t* __restrict__ stored)
{
    chunks_store<false>(sizes, n_chunks, n, chunk_syms, out, stored, nullptr);
}

__global__ void __launch_bounds__(kChunkStoreThreads)
    chunks_store_varlen_kernel(uint32_t* __restrict__ sizes, uint32_t chunk_syms, uint8_t* __restrict__ out, uint32_t* __restrict__ stored,
                               const VarlenGeom* __restrict__ geom)
{
    chunks_store<true>(sizes, 0, 0, chunk_syms, out, stored, geom);
}

// The first kernel of rb200_container_model_encode_varlen_async, one warp: reads n = *d_n, checks 1 <= n <= n_max
// (n == 0 is kStatModel, as the fixed call's RB200_E_MODEL; n > n_max is kStatArg) and writes the geometry of a
// version 1 container of n symbols into *g, with go = 1 when the checks pass.  On failure *g is zero: every later
// kernel exits at entry and the CRC kernels, which read their lengths from *g, cover nothing.  out_cap is at least the
// blob offset of n_max (the host checks it), so blob_cap does not wrap.
__global__ void __launch_bounds__(32)
    varlen_plan_kernel(const uint64_t* __restrict__ d_n, uint64_t n_max, uint32_t chunk_syms, uint64_t out_cap, VarlenGeom* __restrict__ g,
                       uint32_t* __restrict__ status)
{
    if (threadIdx.x) return;
    const uint64_t n = *d_n;
    VarlenGeom r = {};
    if (n == 0 || n > n_max) {
        atomicOr(status, n == 0 ? kStatModel : kStatArg);
    } else {
        const uint64_t chunks = n / chunk_syms + (n % chunk_syms != 0);
        r.n = n;
        r.n_chunks = static_cast<uint32_t>(chunks);
        r.dir_len = (chunks + 1) * sizeof(uint64_t);
        r.dir_off = kContainerDirOffset;
        r.blob_off = (kContainerDirOffset + r.dir_len + 15) & ~15ull;
        r.blob_cap = out_cap - r.blob_off;
        r.go = 1;
    }
    *g = r;
}

// The first kernel of rb200_container_stored_encode_varlen_async, one warp: varlen_plan_kernel's checks and verdicts,
// with the geometry of a version 6 container of n symbols (the blob after the stored-chunk bitmap, the meta CRC over
// directory, pad and bitmap) written into *g.  The same VarlenGeom goes to *model_geom, the record the GEOM model
// kernel reads its gate from (ModelAsyncWork::geom).  On failure both are zero.
__global__ void __launch_bounds__(32)
    stored_varlen_plan_kernel(const uint64_t* __restrict__ d_n, uint64_t n_max, uint32_t chunk_syms, uint64_t out_cap,
                              StoredVarlenGeom* __restrict__ g, VarlenGeom* __restrict__ model_geom, uint32_t* __restrict__ status)
{
    if (threadIdx.x) return;
    const uint64_t n = *d_n;
    StoredVarlenGeom r = {};
    if (n == 0 || n > n_max) {
        atomicOr(status, n == 0 ? kStatModel : kStatArg);
    } else {
        const uint64_t chunks = n / chunk_syms + (n % chunk_syms != 0);
        r.v.n = n;
        r.v.n_chunks = static_cast<uint32_t>(chunks);
        r.v.dir_len = (chunks + 1) * sizeof(uint64_t);
        r.v.dir_off = kContainerDirOffset;
        r.v.blob_off = container_bitmap_blob_offset(chunks);
        r.v.blob_cap = out_cap - r.v.blob_off;
        r.meta_len = r.v.blob_off - kContainerDirOffset;
        r.v.go = 1;
    }
    *g = r;
    *model_geom = r.v;
}

// After the encoder, one thread: blob_len = the directory's last entry, the length of the blob CRC (crc32_kernel's
// n_dev); the directory is at out + dir_off in the container `out`
__global__ void __launch_bounds__(32) varlen_blob_len_kernel(const uint8_t* __restrict__ out, VarlenGeom* __restrict__ g)
{
    if (threadIdx.x == 0 && g->go) g->blob_len = reinterpret_cast<const uint64_t*>(out + g->dir_off)[g->n_chunks];
}

// The first kernel of rb200_container_blocks_model_encode_varlen_async, one warp: reads n_blocks = *d_n_blocks, checks
// 1 <= n_blocks <= n_blocks_max (both failures are kStatArg: zero blocks is the fixed call's RB200_E_ARG) and writes the
// geometry of a per-block container of n_blocks blocks into *g, with v.go = 1 when the checks pass.  On failure *g is
// zero: every later kernel exits at entry and the CRC kernels, which read their lengths from *g, cover nothing.  out_cap
// is at least the blob offset of n_blocks_max (the host checks it), and the offset grows with the count, so blob_cap
// does not wrap.  one_pair set (a list of one candidate, for which the host launches no choice kernel): the choice
// record the gated groups and the header kernel read, that pair as group 0; its costs are left as they are.
__global__ void __launch_bounds__(32)
    blocks_varlen_plan_kernel(const uint32_t* __restrict__ d_n_blocks, uint32_t n_blocks_max, uint32_t block_size, uint32_t chunk_syms,
                              uint64_t out_cap, uint32_t one_pair, BlocksVarlenGeom* __restrict__ g, BlocksChoice* __restrict__ r,
                              uint32_t* __restrict__ status)
{
    if (threadIdx.x) return;
    const uint32_t n_blocks = *d_n_blocks;
    BlocksVarlenGeom q = {};
    if (n_blocks == 0 || n_blocks > n_blocks_max) {
        atomicOr(status, kStatArg);
    } else {
        const uint64_t chunks = static_cast<uint64_t>(n_blocks) * (block_size / chunk_syms);
        q.n_blocks = n_blocks;
        q.v.dir_off = sizeof(ContainerHeader) + kBlockModelBytes * n_blocks;
        q.v.n = static_cast<uint64_t>(n_blocks) * block_size;
        q.v.n_chunks = static_cast<uint32_t>(chunks);
        q.v.dir_len = (chunks + 1) * sizeof(uint64_t);
        q.v.blob_off = (q.v.dir_off + q.v.dir_len + 15) & ~15ull;
        q.v.blob_cap = out_cap - q.v.blob_off;
        q.meta_len = q.v.dir_off + q.v.dir_len - sizeof(ContainerHeader);
        q.v.go = 1;
    }
    *g = q;
    if (one_pair) {
        r->choice.coder = one_pair >> 8;
        r->choice.scale_bits = one_pair & 0xffu;
        r->choice.index = 0;
        r->choice.group = 0;
        r->version = container_blocks_version(r->choice.coder);
    }
}

}  // namespace rb200

// block_coder_kernels.cuh -- per-block models for the byte (main.cpp) and rans64 (main64.cpp) coders at scale_bits 8..15:
// the version 2 geometry (one CTA per block, one warp per chunk, at most 32 chunks per block) with each block's model
// normalised to 1 << scale_bits instead of 4096.
//
//   block_coder_encode_kernel<CODER, SB, BUILD>
//                          BUILD: count_freqs + normalize_freqs(1 << sb) of the block (block_model_build_wide, bit-exact,
//                          written to block_freqs); else the caller's row.  Then the block's encoder table in shared
//                          memory from the tables.h formulas (byte_enc_entry / rans64_enc_entry, 8x replicated as K8 / K9
//                          stage it), and encode_chunk_split per warp with AliasEncoder<false, SB> / Rans64Encoder: the
//                          split path's slots, followed by K6's tile scan and compaction
//   block_coder_decode_kernel<CODER, SB>
//                          the block's decode table in shared memory (cum2sym[1 << sb], then byte_dec_symbol x 256 or
//                          rans64's 16x replicated {start, freq}), then decode_window_chunk per warp with ByteDecoder<SB> /
//                          Rans64Decoder
//
// A block whose frequencies do not sum to 1 << sb: the encoder codes it with an empty model (every symbol flagged,
// RB200_E_SYMBOL), the decoder flags kStatStream and decodes nothing of it, as K5 does for the word coder.
#pragma once
#include "alias_kernels.cuh"
#include "block_kernels.cuh"
#include "rans64_kernels.cuh"
#include "tables.h"

namespace rb200 {

// the largest scale_bits of a per-block model: its frequencies are u16, and 1 << 15 holds a one-symbol block
constexpr uint32_t kBlockCoderMaxScaleBits = 15;

// dynamic shared memory of the per-block byte / rans64 encoder: the 32 KiB table, then 1 KiB per warp (as K5's)
inline uint32_t block_coder_encode_smem(uint32_t threads) { return block_encode_smem(threads); }

// dynamic shared memory of the per-block decoder: 1 KiB of stream window per warp, cum2sym, then the symbol entries
__host__ __device__ constexpr uint32_t block_coder_sym_bytes(uint32_t coder)
{
    return coder == RB200_CODER_BYTE ? 256 * 4 : kRans64DecSymBytes;
}
inline uint32_t block_coder_decode_smem(uint32_t coder, uint32_t sb, uint32_t threads)
{
    return (threads / 32) * kRingBytes + (1u << sb) + block_coder_sym_bytes(coder);
}

template <uint32_t CODER, uint32_t SB, bool BUILD>
__global__ void __launch_bounds__(kMaxBlockWarps * 32)
block_coder_encode_kernel(const uint8_t* __restrict__ in, uint32_t block_size, uint16_t* __restrict__ block_freqs, uint32_t sb_rt,
                          uint32_t chunk_syms, uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint32_t* __restrict__ sizes,
                          uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_benc[];         // [32 KiB: histogram copies (BUILD), then the table][warps x 1 KiB]
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];                 // block_normalize reads it 16 bytes at a time
    __shared__ uint32_t s_flag[1];
    const uint32_t sb = SB ? SB : sb_rt, M = 1u << sb;
    const uint32_t tid = threadIdx.x, warp = tid >> 5;
    const uint8_t* blk = in + static_cast<uint64_t>(blockIdx.x) * block_size;
    uint16_t* freqs = block_freqs + static_cast<uint64_t>(blockIdx.x) * 256;
    bool ok;
    if (BUILD) {
        block_model_build_wide(blk, block_size, reinterpret_cast<uint32_t*>(s_benc), s_cnt, s_cum, s_w, freqs, status, M);
        ok = block_prefix(s_w, s_cum, &s_flag[0], M);                // the widths are still in shared memory
    } else {
        ok = block_prefix(static_cast<const uint16_t*>(freqs), s_cum, &s_flag[0], M);
    }
    // the encoder table as K8 / K9 stage theirs: one 16-byte entry per symbol, kEncReplicas copies
    uint4* s_tab = reinterpret_cast<uint4*>(s_benc);
    for (uint32_t s = tid; s < 256; s += blockDim.x) {
        const uint32_t f = ok ? s_cum[s + 1] - s_cum[s] : 0, cum = ok ? s_cum[s] : 0;
        uint4 x;
        if (CODER == RB200_CODER_BYTE) {
            const AliasEncEntry e = byte_enc_entry(f, cum, sb);       // {x_max, rcp_freq, bias, cmpl_freq | rcp_shift << 16}
            x = make_uint4(e.magic, e.freq, e.cum, e.shift);
        } else {
            uint32_t e[8];
            rans64_enc_entry(f, cum, sb, e);                          // {rcp_lo, rcp_hi, freq, bias}, {cmpl_freq, shift | bad}
            x = make_uint4(e[0], e[1], e[3], (e[4] & 0xfffffu) | ((e[5] & 63u) << 20) | (e[5] & kEncBadSymbol));
        }
#pragma unroll
        for (uint32_t r = 0; r < kEncReplicas; r++) s_tab[s * kEncReplicas + r] = x;
    }
    __syncthreads();

    const uint32_t per_block = block_size / chunk_syms;
    if (warp >= per_block) return;
    const uint32_t chunk = blockIdx.x * per_block + warp;
    const uint8_t* src = blk + static_cast<uint64_t>(warp) * chunk_syms;
    const uint32_t tab = smem_addr(s_benc), wsm = tab + kEncTableBytes + warp * kEncWarpSmem;
    if (CODER == RB200_CODER_BYTE)
        encode_chunk_split(src, chunk_syms, chunk, AliasEncoder<false, SB>{tab, 0, sb}, wsm, scratch, slot_bytes, sizes, status);
    else
        encode_chunk_split(src, chunk_syms, chunk, Rans64Encoder{tab, sb}, wsm, scratch, slot_bytes, sizes, status);
}

// A block's decode table in shared memory at s_tab, from its cumulative frequencies (s_cum[257], M = 1 << sb): cum2sym[M],
// then the symbol entries.  Every thread of the CTA takes part; the caller synchronises before the table is read.
template <uint32_t CODER>
__device__ __forceinline__ void block_coder_decode_table(const uint32_t* s_cum, uint8_t* s_tab, uint32_t M)
{
    const uint32_t tid = threadIdx.x;
    // cum2sym, 4 slots (one u32) at a time: one binary search per 4 slots for the largest s with cum[s] <= slot, then a
    // walk that also steps over zero-width symbols; the cost per slot does not depend on how skewed the model is, and
    // consecutive threads store consecutive words
    uint32_t* c2s = reinterpret_cast<uint32_t*>(s_tab);
    for (uint32_t q = tid; q < M / 4; q += blockDim.x) {
        uint32_t lo = 0, hi = 256;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s_cum[mid] <= 4 * q) lo = mid; else hi = mid;
        }
        uint32_t packed = 0;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) {
            while (4 * q + k >= s_cum[lo + 1]) lo++;
            packed |= lo << (8 * k);
        }
        c2s[q] = packed;
    }
    if (CODER == RB200_CODER_BYTE) {
        uint32_t* syms = reinterpret_cast<uint32_t*>(s_tab + M);
        for (uint32_t s = tid; s < 256; s += blockDim.x) syms[s] = byte_dec_symbol(s_cum[s], s_cum[s + 1] - s_cum[s]);
    } else {
        uint2* syms = reinterpret_cast<uint2*>(s_tab + M);
        for (uint32_t i = tid; i < 256 * kRans64DecReplicas; i += blockDim.x) {
            const uint32_t s = i / kRans64DecReplicas;
            syms[i] = make_uint2(s_cum[s], s_cum[s + 1] - s_cum[s]);
        }
    }
}

template <uint32_t CODER, uint32_t SB>
__global__ void __launch_bounds__(kMaxBlockWarps * 32)
block_coder_decode_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets,
                          const uint16_t* __restrict__ block_freqs, uint32_t sb_rt, uint32_t block_size, uint32_t chunk_syms,
                          uint8_t* __restrict__ out, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_bdec[];         // [warps x 1 KiB rings][cum2sym[1 << sb]][symbol entries]
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[1];
    const uint32_t sb = SB ? SB : sb_rt, M = 1u << sb;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, warps = blockDim.x >> 5;
    if (!block_prefix(block_freqs + static_cast<uint64_t>(blockIdx.x) * 256, s_cum, &s_flag[0], M)) {
        if (tid == 0) atomicOr(status, kStatStream);
        return;
    }
    uint8_t* s_tab = s_bdec + warps * kRingBytes;
    block_coder_decode_table<CODER>(s_cum, s_tab, M);
    __syncthreads();

    const uint32_t per_block = block_size / chunk_syms;
    if (warp >= per_block) return;
    const uint32_t chunk = blockIdx.x * per_block + warp;
    uint8_t* dst = out + static_cast<uint64_t>(blockIdx.x) * block_size + static_cast<uint64_t>(warp) * chunk_syms;
    const uint32_t ring = smem_addr(s_bdec) + warp * kRingBytes, tab = smem_addr_pinned(s_tab);
    if (CODER == RB200_CODER_BYTE)
        decode_window_chunk(ByteDecoder<SB>{tab, sb}, blob, blob_size, offsets, chunk, ring, dst, chunk_syms, status);
    else
        decode_window_chunk(Rans64Decoder{tab, tab + M + (lane & (kRans64DecReplicas - 1)) * 8, sb}, blob, blob_size, offsets, chunk, ring,
                            dst, chunk_syms, status);
}

// The instances: the byte coder specialised for scale_bits 14 (main.cpp) and 12, generic otherwise, as K8; rans64 generic
#define RB200_BLOCK_CODER_DISPATCH(coder, sb, CALL)                                      \
    if (coder == RB200_CODER_RANS64) {                                                   \
        constexpr uint32_t CODER = RB200_CODER_RANS64, SB = 0; CALL;                     \
    } else if (sb == 14) {                                                               \
        constexpr uint32_t CODER = RB200_CODER_BYTE, SB = 14; CALL;                      \
    } else if (sb == 12) {                                                               \
        constexpr uint32_t CODER = RB200_CODER_BYTE, SB = 12; CALL;                      \
    } else {                                                                             \
        constexpr uint32_t CODER = RB200_CODER_BYTE, SB = 0; CALL;                       \
    }

template <uint32_t CODER, uint32_t SB>
inline void configure_block_coder()
{
    for (const void* k : {reinterpret_cast<const void*>(block_coder_encode_kernel<CODER, SB, true>),
                          reinterpret_cast<const void*>(block_coder_encode_kernel<CODER, SB, false>)}) {
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, block_coder_encode_smem(kMaxBlockWarps * 32));
    }
    cudaFuncSetAttribute(block_coder_decode_kernel<CODER, SB>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(block_coder_decode_kernel<CODER, SB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         block_coder_decode_smem(CODER, kBlockCoderMaxScaleBits, kMaxBlockWarps * 32));
}
inline void configure_block_coder_kernels()
{
    configure_block_coder<RB200_CODER_BYTE, 14>();
    configure_block_coder<RB200_CODER_BYTE, 12>();
    configure_block_coder<RB200_CODER_BYTE, 0>();
    configure_block_coder<RB200_CODER_RANS64, 0>();
}

// one CTA per block of block_threads() threads; smem = block_coder_encode_smem(threads)
inline void launch_block_coder_encode(cudaStream_t stream, uint32_t coder, uint32_t sb, bool build, uint32_t n_blocks, uint32_t threads,
                                      uint32_t smem, const uint8_t* d_in, uint32_t block_size, uint16_t* d_freqs, uint32_t chunk_syms,
                                      uint8_t* scratch, uint32_t slot_bytes, uint32_t* sizes, uint32_t* status)
{
    RB200_BLOCK_CODER_DISPATCH(coder, sb, ((build ? block_coder_encode_kernel<CODER, SB, true> : block_coder_encode_kernel<CODER, SB, false>)
                                           <<<n_blocks, threads, smem, stream>>>(d_in, block_size, d_freqs, sb, chunk_syms, scratch,
                                                                                 slot_bytes, sizes, status)))
}

inline void launch_block_coder_decode(cudaStream_t stream, uint32_t coder, uint32_t sb, const uint8_t* blob, uint64_t blob_size,
                                      const uint64_t* offsets, const uint16_t* d_freqs, uint32_t n_blocks, uint32_t block_size,
                                      uint32_t chunk_syms, uint8_t* out, uint32_t* status)
{
    const uint32_t threads = block_threads(block_size, chunk_syms);
    const uint32_t smem = block_coder_decode_smem(coder, sb, threads);
    RB200_BLOCK_CODER_DISPATCH(coder, sb, (block_coder_decode_kernel<CODER, SB><<<n_blocks, threads, smem, stream>>>(
                                              blob, blob_size, offsets, d_freqs, sb, block_size, chunk_syms, out, status)))
}

}  // namespace rb200

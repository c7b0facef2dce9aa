// builders.cu -- the library's model and table builders run on the GPU, next to their host twins, for
// tests/test_model_builders_on_gpu.py.
//
// Nothing here restates a builder.  The md_* entries launch the shipped __global__ kernels unchanged on workspaces the
// caller allocated and filled (container_model_kernel, coder_choice_kernel, container_table_kernel), or thin batch
// kernels, one CTA per model, that call the shipped __device__ builders the way their callers do: the same shared
// arrays, alignment and blockDim.  The hw_* entries are the host twins from model_host.cpp (linked into this .so) and
// the format rules of container_format.h.  Every md_* entry launches on the default stream and returns the CUDA error
// of the batch after a device synchronisation.
#include "rans_b200.h"

#include <cstddef>
#include <cstring>

#include "block_coder_kernels.cuh"
#include "container_decode.cuh"
#include "container_format.h"
#include "model_kernels.cuh"
#include "tables.h"

using namespace rb200;

namespace {

int finish()
{
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return static_cast<int>(e);
}

// block_model_build at kModelWarps warps, with its workspace in static shared memory (16-byte aligned: block_normalize
// reads the widths in h[0] as uint4)
__global__ void __launch_bounds__(kModelWarps * 32)
    batch_block_model_build(const uint8_t* in, const uint64_t* off, const uint32_t* size, uint32_t target, uint16_t* dst, uint32_t* status)
{
    __shared__ __align__(16) BlockModelSmem sm;
    block_model_build(in + off[blockIdx.x], size[blockIdx.x], sm, dst + blockIdx.x * 256, status + blockIdx.x, target);
}

// block_model_build_wide with block_model_kernel's shared arrays
__global__ void __launch_bounds__(kMaxBlockWarps * 32)
    batch_block_model_build_wide(const uint8_t* in, const uint64_t* off, const uint32_t* size, uint32_t target, uint16_t* dst,
                                 uint32_t* status)
{
    __shared__ uint32_t s_hist[256 * 32];
    __shared__ uint32_t s_cnt[256], s_cum[257];
    __shared__ __align__(16) uint32_t s_w[256];
    block_model_build_wide(in + off[blockIdx.x], size[blockIdx.x], s_hist, s_cnt, s_cum, s_w, dst + blockIdx.x * 256, status + blockIdx.x,
                           target);
}

// block_prefix + block_fill_slots with block_decode_kernel's shared memory layout (rings, then the table); the slot table
// is pre-filled with a sentinel so that a slot the fill misses shows.  flags[2i] = block_prefix's verdict,
// flags[2i + 1] = wide.
__global__ void __launch_bounds__(kMaxBlockWarps * 32) batch_fill_slots(const uint16_t* rows, uint32_t* tab, uint32_t* flags)
{
    extern __shared__ __align__(1024) uint8_t s_bdec[];
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[2];
    uint32_t* s_tab = reinterpret_cast<uint32_t*>(s_bdec + (blockDim.x >> 5) * kRingBytes);
    const uint32_t tid = threadIdx.x;
    for (uint32_t i = tid; i < kWordSlots; i += blockDim.x) s_tab[i] = 0xdeadbeefu;
    if (tid == 0) s_flag[1] = 0;
    const bool ok = block_prefix(rows + blockIdx.x * 256, s_cum, &s_flag[0], kWordSlots);
    if (ok) block_fill_slots(s_cum, s_tab, &s_flag[1]);
    __syncthreads();
    for (uint32_t i = tid; i < kWordSlots; i += blockDim.x) tab[blockIdx.x * kWordSlots + i] = s_tab[i];
    if (tid == 0) {
        flags[2 * blockIdx.x] = ok;
        flags[2 * blockIdx.x + 1] = s_flag[1];
    }
}

// block_prefix + block_build_enc_table with block_coder_encode_kernel<word>'s shared arrays (the table at the start of the
// 1024-aligned dynamic shared memory).  flags[2i] = block_prefix's verdict, flags[2i + 1] = r32.
__global__ void __launch_bounds__(kMaxBlockWarps * 32) batch_enc_table(const uint16_t* rows, uint4* out, uint32_t* flags)
{
    extern __shared__ __align__(1024) uint8_t s_enc[];
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[1];
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc);
    const bool ok = block_prefix(rows + blockIdx.x * 256, s_cum, &s_flag[0], kWordSlots);
    const bool r32 = block_build_enc_table(s_cum, ok, s_tab);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) out[blockIdx.x * 256 * kEncReplicas + i] = s_tab[i];
    if (threadIdx.x == 0) {
        flags[2 * blockIdx.x] = ok;
        flags[2 * blockIdx.x + 1] = r32;
    }
}

// word_enc_expand<r32[i]> of 256 host-built entries per model: what the word encoders stage in shared memory
__global__ void __launch_bounds__(256) batch_enc_expand(const WordEncEntry* e, const uint32_t* r32, uint4* out)
{
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    out[i] = r32[blockIdx.x] ? word_enc_expand<true>(e[i]) : word_enc_expand<false>(e[i]);
}

// block_prefix + block_coder_decode_table<CODER> with block_decode_kernel's dynamic shared memory layout (rings,
// then the table); the table is pre-filled with a sentinel.  A row block_prefix rejects gets no table (ok[i] = 0), as
// in the shipped callers.
template <uint32_t CODER>
__global__ void __launch_bounds__(kMaxBlockWarps * 32) batch_coder_decode_table(const uint16_t* rows, uint32_t sb, uint8_t* out, uint32_t* ok)
{
    extern __shared__ __align__(1024) uint8_t s_bdec[];
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[1];
    const uint32_t M = 1u << sb, words = (M + block_coder_sym_bytes(CODER)) / 4;
    uint8_t* s_tab = s_bdec + (blockDim.x >> 5) * kRingBytes;
    uint32_t* s_words = reinterpret_cast<uint32_t*>(s_tab);
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) s_words[i] = 0xa5a5a5a5u;
    const bool good = block_prefix(rows + blockIdx.x * 256, s_cum, &s_flag[0], M);
    if (threadIdx.x == 0) ok[blockIdx.x] = good;
    if (!good) return;
    block_coder_decode_table<CODER>(s_cum, s_tab, M);
    __syncthreads();
    uint32_t* dst = reinterpret_cast<uint32_t*>(out) + static_cast<uint64_t>(blockIdx.x) * words;
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) dst[i] = s_words[i];
}

template <class T>
T* at(uint8_t* base, uint64_t stride, uint32_t i)
{
    return reinterpret_cast<T*>(base + stride * i);
}

}  // namespace

extern "C" {

// sizes and offsets of the workspaces, so the caller can fill and read them
uint64_t md_layout(int k)
{
    switch (k) {
    case 0: return sizeof(ModelAsyncWork);
    case 1: return offsetof(ModelAsyncWork, counts);
    case 2: return offsetof(ModelAsyncWork, freqs);
    case 3: return offsetof(ModelAsyncWork, r32);
    case 4: return offsetof(ModelAsyncWork, word_enc);
    case 5: return offsetof(ModelAsyncWork, word_enc32);
    case 6: return offsetof(ModelAsyncWork, alias_enc);
    case 7: return offsetof(ModelAsyncWork, byte_enc);
    case 8: return offsetof(ModelAsyncWork, r64_enc);
    case 9: return offsetof(ModelAsyncWork, alias_remap);
    case 10: return offsetof(ModelAsyncWork, choice);
    case 11: return offsetof(ModelAsyncWork, cand_freqs);
    case 12: return sizeof(ContainerAsyncWork);
    case 13: return offsetof(ContainerAsyncWork, plan) + offsetof(BlocksPlan, ok);
    case 14: return offsetof(ContainerAsyncWork, bad);
    case 15: return offsetof(ContainerAsyncWork, coder);
    case 16: return offsetof(ContainerAsyncWork, scale_bits);
    case 17: return offsetof(ContainerAsyncWork, wide);
    case 18: return offsetof(ContainerAsyncWork, refused);
    case 19: return offsetof(ContainerAsyncWork, table);
    case 20: return offsetof(CoderChoice, costs);
    case 21: return kEncReplicas;
    case 22: return kRans64DecReplicas;
    case 23: return kStatModel;
    case 24: return kMaxCandidates;
    default: return ~0ull;
    }
}

// container_model_kernel<false, CHOSEN> on works[i] (counts filled; CHOSEN: choice and cand_freqs filled), as
// rans_b200.cu launches it
int md_model(uint32_t n, const uint32_t* coder, const uint32_t* sb, uint32_t r32_allowed, uint8_t* works, uint32_t* status, int chosen)
{
    for (uint32_t i = 0; i < n; i++) {
        ModelAsyncWork* w = at<ModelAsyncWork>(works, sizeof(ModelAsyncWork), i);
        if (chosen)
            container_model_kernel<false, true><<<1, kModelThreads>>>(0, 0, r32_allowed, w, status + i);
        else
            container_model_kernel<false, false><<<1, kModelThreads>>>(coder[i], sb[i], r32_allowed, w, status + i);
    }
    return finish();
}

// coder_choice_kernel on works[i] (counts filled).  lists: per model kMaxCandidates pairs, kMaxCandidates groups, n,
// tolerance_ppm (34 words); list.n * 32 threads, as rans_b200.cu launches it
int md_choice(uint32_t n, const uint32_t* lists, const uint64_t* n_chunks, uint8_t* works, uint32_t* status)
{
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t* l = lists + i * (2 * kMaxCandidates + 2);
        CandidateList list;
        std::memcpy(list.pair, l, sizeof list.pair);
        std::memcpy(list.group, l + kMaxCandidates, sizeof list.group);
        list.n = l[2 * kMaxCandidates];
        list.tolerance_ppm = l[2 * kMaxCandidates + 1];
        coder_choice_kernel<<<1, list.n * 32>>>(list, n_chunks[i], at<ModelAsyncWork>(works, sizeof(ModelAsyncWork), i), nullptr, status + i);
    }
    return finish();
}

// container_table_kernel on works[i] (plan.ok, coder, scale_bits set; the rest zero) and the model at bufs[i] + 64
int md_table(uint32_t n, const uint8_t* bufs, uint64_t buf_stride, uint8_t* works)
{
    for (uint32_t i = 0; i < n; i++)
        container_table_kernel<<<1, kTableThreads>>>(bufs + buf_stride * i, at<ContainerAsyncWork>(works, sizeof(ContainerAsyncWork), i));
    return finish();
}

// block_model_build (wide == 0, 8 warps) or block_model_build_wide (wide != 0, `threads` threads), one block per CTA
int md_block_build(int wide, uint32_t threads, uint32_t n, const uint8_t* in, const uint64_t* off, const uint32_t* size, uint32_t target,
                   uint16_t* dst, uint32_t* status)
{
    if (wide)
        batch_block_model_build_wide<<<n, threads>>>(in, off, size, target, dst, status);
    else
        batch_block_model_build<<<n, kModelWarps * 32>>>(in, off, size, target, dst, status);
    return finish();
}

int md_fill_slots(uint32_t threads, uint32_t n, const uint16_t* rows, uint32_t* tab, uint32_t* flags)
{
    const uint32_t smem = block_coder_decode_smem(RB200_CODER_WORD, kWordScaleBits, threads);
    cudaFuncSetAttribute(batch_fill_slots, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    batch_fill_slots<<<n, threads, smem>>>(rows, tab, flags);
    return finish();
}

int md_enc_table(uint32_t threads, uint32_t n, const uint16_t* rows, uint4* out, uint32_t* flags)
{
    batch_enc_table<<<n, threads, kEncTableBytes>>>(rows, out, flags);
    return finish();
}

int md_enc_expand(uint32_t n, const WordEncEntry* e, const uint32_t* r32, uint4* out)
{
    batch_enc_expand<<<n, 256>>>(e, r32, out);
    return finish();
}

// out: per model (1 << sb) + block_coder_sym_bytes(coder) bytes
int md_coder_decode_table(uint32_t coder, uint32_t sb, uint32_t threads, uint32_t n, const uint16_t* rows, uint8_t* out, uint32_t* ok)
{
    const uint32_t smem = block_coder_decode_smem(coder, sb, threads);
    if (coder == RB200_CODER_BYTE) {
        cudaFuncSetAttribute(batch_coder_decode_table<RB200_CODER_BYTE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        batch_coder_decode_table<RB200_CODER_BYTE><<<n, threads, smem>>>(rows, sb, out, ok);
    } else {
        cudaFuncSetAttribute(batch_coder_decode_table<RB200_CODER_RANS64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        batch_coder_decode_table<RB200_CODER_RANS64><<<n, threads, smem>>>(rows, sb, out, ok);
    }
    return finish();
}

// ---- host twins: the tables rb200_model_create uploads (model_host.cpp) and the format rules

int hw_word(const uint32_t* freqs, uint32_t* dec, WordEncEntry* enc, WordEncEntry* enc32, int32_t* flags)
{
    static WordDeviceTables t;
    const int rc = build_word_device_tables(freqs, t);
    if (rc != RB200_OK) return rc;
    std::memcpy(dec, t.dec, sizeof t.dec);
    std::memcpy(enc, t.enc, sizeof t.enc);
    std::memcpy(enc32, t.enc32, sizeof t.enc32);
    flags[0] = t.wide;
    flags[1] = t.enc32_ok;
    return rc;
}

int hw_alias(const uint32_t* freqs, uint32_t sb, AliasDecEntry* dec, AliasEncEntry* enc, uint16_t* remap)
{
    static AliasDeviceTables t;
    const int rc = build_alias_device_tables(freqs, sb, t);
    if (rc != RB200_OK) return rc;
    std::memcpy(dec, t.dec, sizeof t.dec);
    std::memcpy(enc, t.enc, sizeof t.enc);
    std::memcpy(remap, t.remap.data(), t.remap.size() * sizeof(uint16_t));
    return rc;
}

int hw_byte(const uint32_t* freqs, uint32_t sb, uint8_t* dec, AliasEncEntry* enc)
{
    static ByteDeviceTables t;
    const int rc = build_byte_device_tables(freqs, sb, t);
    if (rc != RB200_OK) return rc;
    std::memcpy(dec, t.dec.data(), t.dec.size());
    std::memcpy(enc, t.enc, sizeof t.enc);
    return rc;
}

int hw_rans64(const uint32_t* freqs, uint32_t sb, uint8_t* dec, uint32_t* enc)
{
    static Rans64DeviceTables t;
    const int rc = build_rans64_device_tables(freqs, sb, t);
    if (rc != RB200_OK) return rc;
    std::memcpy(dec, t.dec.data(), t.dec.size());
    std::memcpy(enc, t.enc, sizeof t.enc);
    return rc;
}

int hw_model_ok(uint32_t coder, uint32_t sb, const uint32_t* freqs) { return container_model_ok(coder, sb, freqs); }
int hw_model_decodable(uint32_t coder, const uint32_t* freqs) { return container_model_decodable(coder, freqs); }

}  // extern "C"

// rans_b200.cu -- C-ABI (include/rans_b200.h) over the sm_90a rANS kernels.
//
// Host code is C++ like the reference's drivers; it owns no global state: everything
// lives in rb200_ctx (device, stream, grow-only workspaces) and rb200_model (device
// tables).  Data pointers are either host memory (the call stages them through the
// context's device buffers and is synchronous, like the reference's loops) or device
// memory (the call only enqueues kernels on the context's stream).
#include "rans_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "alias_kernels.cuh"
#include "block_coder_kernels.cuh"
#include "block_kernels.cuh"
#include "container_decode.cuh"
#include "container_format.h"
#include "crc_kernels.cuh"
#include "model_kernels.cuh"
#include "planes_kernels.cuh"
#include "rans64_kernels.cuh"
#include "tables.h"
#include "word_kernels.cuh"
#include "word_decode_tma.cuh"

using namespace rb200;

// ---------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
};

struct rb200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint32_t* d_status = nullptr;     // kStat* bits, OR-ed by kernels
    uint32_t* h_status = nullptr;     // pinned mirror
    DecodeWork* d_work = nullptr;     // persistent decoder's chunk counter; zero between launches (self-resetting)
    int sms = 0;                      // multiprocessors of `device`
    uint64_t launches = 0;
    std::string last_error;
    // encode workspaces
    DevBuf scratch, sizes;
    // staging for RB200_MEM_HOST calls
    DevBuf st_in, st_blob, st_offsets, st_out, st_aux;
    // host-mode slice pipeline: H2D on s_in, kernels on `stream`, D2H on s_out
    cudaStream_t s_in = nullptr, s_out = nullptr;
    static constexpr int kMaxSlices = 256;
    cudaEvent_t ev_in[kMaxSlices] = {}, ev_done[kMaxSlices] = {};
    cudaEvent_t ev_start = nullptr, ev_out = nullptr;
    uint64_t* h_slice_total = nullptr;   // pinned, kMaxSlices entries
    uint64_t* h_dir = nullptr;           // pinned staging for directories (caller's `offsets` may be pageable)
    size_t h_dir_cap = 0;                // entries
    // CRC-32 (crc_kernels.cuh): the kernel's self-resetting accumulator, one result per pipeline slice, pinned mirror
    CrcWork* d_crc_work = nullptr;
    CrcSlot* d_crc = nullptr;            // kMaxSlices entries
    CrcSlot* h_crc = nullptr;
    // the async container decodes (container_decode.cuh): one fixed workspace per version, so that calls of different
    // versions never share state, and every version's decoder launches
    ContainerAsyncWork* d_async[6] = {};
    DecoderLaunch async_decoders[kContainerDecoders] = {};
    // rb200_container_blocks_any_decode_async: its own workspace, for its checks and the decoders of versions 2-4
    ContainerAsyncWork* d_async_any = nullptr;
    // rb200_container_model_encode_async (model_kernels.cuh): the counts, the model and its encode tables
    ModelAsyncWork* d_model_async = nullptr;
    // rb200_container_blocks_model_encode_auto_async (model_kernels.cuh): the choice record and its running sums
    BlocksChoice* d_blocks_choice = nullptr;
    // rb200_container_blocks_model_encode_varlen_async: the geometry of the count its plan kernel read
    BlocksVarlenGeom* d_blocks_geom = nullptr;
    // rb200_container_stored_encode_varlen_async: the geometry of the length its plan kernel read
    StoredVarlenGeom* d_stored_geom = nullptr;
    // the byte-plane calls (planes_kernels.cuh): each call's record, the encode's split planes and staging area, the
    // decode's decoded planes and staging area
    PlanesWork* d_planes_enc = nullptr;
    PlanesWork* d_planes_dec = nullptr;
    DevBuf planes_in, planes_enc_stage, planes_out, planes_dec_stage;
    // rb200_container_planes_encode_varlen_async: the length its plan kernel read
    PlanesVarlenGeom* d_planes_geom = nullptr;
    // the delta calls (version 8): the base's CRC, one record for the encode, one for the decode
    DeltaWork* d_delta_enc = nullptr;
    DeltaWork* d_delta_dec = nullptr;
    // the tensor-list calls (version 9): the directory's CRC and the list's prefix, one of each for the encode and the
    // decode
    TensorsWork* d_tensors_enc = nullptr;
    TensorsWork* d_tensors_dec = nullptr;
    DevBuf tensors_enc_prefix, tensors_dec_prefix;
};

struct rb200_model {
    rb200_ctx* ctx = nullptr;
    int coder = 0;
    uint32_t scale_bits = 0;
    int wide = 0;
    uint32_t* d_word_dec = nullptr;          // 4096 x u32
    WordEncEntry* d_word_enc = nullptr;      // 256; the 32-bit-reciprocal table when enc_r32 (tables.h)
    int enc_r32 = 0;
    AliasDecEntry* d_alias_dec = nullptr;    // 256 x 16 B
    AliasEncEntry* d_alias_enc = nullptr;    // 256
    uint16_t* d_alias_remap = nullptr;       // 1 << scale_bits
    uint8_t* d_byte_dec = nullptr;           // cum2sym[1 << scale_bits] + 256 x u32
    AliasEncEntry* d_byte_enc = nullptr;     // 256 RansEncSymbol images
    uint8_t* d_r64_dec = nullptr;            // cum2sym[1 << scale_bits] + 256 x {start, freq}
    uint4* d_r64_enc = nullptr;              // 256 x 32 B Rans64EncSymbol images
    uint32_t freqs[256] = {};                // the model's frequencies: the model section of a container
    uint32_t* d_freqs = nullptr;             // device copy, for rb200_container_encode in device memory
};

namespace {

int cuda_fail(rb200_ctx* ctx, cudaError_t e, const char* what)
{
    if (ctx) ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
    return RB200_E_CUDA;
}

#define RB_CUDA(ctx, call)                                              \
    do {                                                                \
        cudaError_t e_ = (call);                                        \
        if (e_ != cudaSuccess) return cuda_fail((ctx), e_, #call);      \
    } while (0)

int reserve(rb200_ctx* ctx, DevBuf& b, size_t bytes)
{
    if (bytes <= b.cap) return RB200_OK;
    if (b.p) {
        RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        RB_CUDA(ctx, cudaFree(b.p));
        b.p = nullptr;
        b.cap = 0;
    }
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) {
        b.p = nullptr;
        cuda_fail(ctx, e, "cudaMalloc(workspace)");
        return RB200_E_NOMEM;
    }
    b.cap = want;
    return RB200_OK;
}

void release(DevBuf& b)
{
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
}

inline size_t round16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }
constexpr size_t kBoundFixed = 512;   // headers (128 B; 256 B for rans64) + one extra unit per lane
inline uint32_t slot_bytes_for(uint32_t chunk_syms) { return static_cast<uint32_t>(round16(kBoundFixed + 2ull * chunk_syms)); }

int status_to_code(uint32_t bits)
{
    if (bits & kStatArg) return RB200_E_ARG;
    if (bits & kStatModel) return RB200_E_MODEL;
    if (bits & kStatSymbol) return RB200_E_SYMBOL;
    if (bits & kStatSpace) return RB200_E_SPACE;
    if (bits & kStatStream) return RB200_E_STREAM;
    if (bits & kStatBase) return RB200_E_BASE;
    if (bits & kStatStall) return RB200_E_STALL;
    return RB200_OK;
}

int check_launch(rb200_ctx* ctx, const char* what)
{
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(ctx, e, what);
    ctx->launches++;
    return RB200_OK;
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev)
    {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

bool chunk_ok(uint32_t chunk_syms) { return container_chunk_ok(chunk_syms); }     // 32 .. 2^24 symbols

}  // namespace

extern "C" int rb200_version(void) { return RB200_VERSION; }

extern "C" const char* rb200_strerror(int code)
{
    switch (code) {
    case RB200_OK: return "ok";
    case RB200_E_ARG: return "bad argument";
    case RB200_E_MODEL: return "invalid model";
    case RB200_E_SPACE: return "output buffer too small";
    case RB200_E_STREAM: return "corrupt or truncated stream";
    case RB200_E_CUDA: return "CUDA error";
    case RB200_E_NOMEM: return "out of device memory";
    case RB200_E_SYMBOL: return "symbol with zero model frequency";
    case RB200_E_NCCL: return "NCCL error";
    case RB200_E_STALL: return "a bounded wait inside a kernel expired";
    case RB200_E_BASE: return "the base is not the tensor the delta was encoded against";
    }
    return "unknown";
}

extern "C" int rb200_ctx_create(rb200_ctx** out, int device, void* stream)
{
    if (!out) return RB200_E_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return RB200_E_CUDA;
    rb200_ctx* ctx = new (std::nothrow) rb200_ctx;
    if (!ctx) return RB200_E_NOMEM;
    ctx->device = device;
    ctx->stream = static_cast<cudaStream_t>(stream);
    DeviceGuard g(device);
    cudaError_t e = cudaMalloc(&ctx->d_status, sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_status, 0, sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_work, sizeof(DecodeWork));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_work, 0, sizeof(DecodeWork));
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->sms, cudaDevAttrMultiProcessorCount, device);
    if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_status, sizeof(uint32_t));
    if (e != cudaSuccess || ctx->sms <= 0) {
        if (ctx->d_status) cudaFree(ctx->d_status);
        if (ctx->d_work) cudaFree(ctx->d_work);
        delete ctx;
        return RB200_E_CUDA;
    }
    *ctx->h_status = 0;
    e = cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_start, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_out, cudaEventDisableTiming);
    for (int i = 0; i < rb200_ctx::kMaxSlices && e == cudaSuccess; i++) {
        e = cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_slice_total, rb200_ctx::kMaxSlices * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_crc_work, sizeof(CrcWork));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_crc_work, 0, sizeof(CrcWork));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_crc, rb200_ctx::kMaxSlices * sizeof(CrcSlot));
    if (e == cudaSuccess) e = cudaMallocHost(&ctx->h_crc, rb200_ctx::kMaxSlices * sizeof(CrcSlot));
    for (ContainerAsyncWork*& w : ctx->d_async) {
        if (e == cudaSuccess) e = cudaMalloc(&w, sizeof(ContainerAsyncWork));
        if (e == cudaSuccess) e = cudaMemset(w, 0, sizeof(ContainerAsyncWork));
    }
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_model_async, sizeof(ModelAsyncWork));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_model_async, 0, sizeof(ModelAsyncWork));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_async_any, sizeof(ContainerAsyncWork));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_async_any, 0, sizeof(ContainerAsyncWork));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_blocks_choice, sizeof(BlocksChoice));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_blocks_choice, 0, sizeof(BlocksChoice));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_blocks_geom, sizeof(BlocksVarlenGeom));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_blocks_geom, 0, sizeof(BlocksVarlenGeom));
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_stored_geom, sizeof(StoredVarlenGeom));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_stored_geom, 0, sizeof(StoredVarlenGeom));
    for (PlanesWork** r : {&ctx->d_planes_enc, &ctx->d_planes_dec}) {
        if (e == cudaSuccess) e = cudaMalloc(r, sizeof(PlanesWork));
        if (e == cudaSuccess) e = cudaMemset(*r, 0, sizeof(PlanesWork));
    }
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_planes_geom, sizeof(PlanesVarlenGeom));
    if (e == cudaSuccess) e = cudaMemset(ctx->d_planes_geom, 0, sizeof(PlanesVarlenGeom));
    for (DeltaWork** d : {&ctx->d_delta_enc, &ctx->d_delta_dec}) {
        if (e == cudaSuccess) e = cudaMalloc(d, sizeof(DeltaWork));
        if (e == cudaSuccess) e = cudaMemset(*d, 0, sizeof(DeltaWork));
    }
    for (TensorsWork** t : {&ctx->d_tensors_enc, &ctx->d_tensors_dec}) {
        if (e == cudaSuccess) e = cudaMalloc(t, sizeof(TensorsWork));
        if (e == cudaSuccess) e = cudaMemset(*t, 0, sizeof(TensorsWork));
    }
    if (e != cudaSuccess) {
        rb200_ctx_destroy(ctx);
        return RB200_E_CUDA;
    }
    // the decoders want the large shared-memory carve-out (tables + per-warp rings)
    configure_word_decode_tma();
    configure_word_kernels();
    configure_alias_kernels();
    configure_block_kernels();
    configure_rans64_kernels();
    configure_crc_kernels();
    configure_container_decode(static_cast<uint32_t>(ctx->sms), ctx->async_decoders);
    cudaGetLastError();
    *out = ctx;
    return RB200_OK;
}

extern "C" void rb200_ctx_destroy(rb200_ctx* ctx)
{
    if (!ctx) return;
    DeviceGuard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    release(ctx->scratch); release(ctx->sizes);
    release(ctx->st_in); release(ctx->st_blob); release(ctx->st_offsets); release(ctx->st_out); release(ctx->st_aux);
    release(ctx->planes_in); release(ctx->planes_enc_stage); release(ctx->planes_out); release(ctx->planes_dec_stage);
    release(ctx->tensors_enc_prefix); release(ctx->tensors_dec_prefix);
    if (ctx->d_status) cudaFree(ctx->d_status);
    if (ctx->d_work) cudaFree(ctx->d_work);
    if (ctx->h_status) cudaFreeHost(ctx->h_status);
    if (ctx->h_slice_total) cudaFreeHost(ctx->h_slice_total);
    if (ctx->h_dir) cudaFreeHost(ctx->h_dir);
    if (ctx->d_crc_work) cudaFree(ctx->d_crc_work);
    if (ctx->d_crc) cudaFree(ctx->d_crc);
    if (ctx->h_crc) cudaFreeHost(ctx->h_crc);
    for (ContainerAsyncWork* w : ctx->d_async)
        if (w) cudaFree(w);
    if (ctx->d_model_async) cudaFree(ctx->d_model_async);
    if (ctx->d_async_any) cudaFree(ctx->d_async_any);
    if (ctx->d_blocks_choice) cudaFree(ctx->d_blocks_choice);
    if (ctx->d_blocks_geom) cudaFree(ctx->d_blocks_geom);
    if (ctx->d_stored_geom) cudaFree(ctx->d_stored_geom);
    if (ctx->d_planes_enc) cudaFree(ctx->d_planes_enc);
    if (ctx->d_planes_dec) cudaFree(ctx->d_planes_dec);
    if (ctx->d_planes_geom) cudaFree(ctx->d_planes_geom);
    if (ctx->d_delta_enc) cudaFree(ctx->d_delta_enc);
    if (ctx->d_delta_dec) cudaFree(ctx->d_delta_dec);
    if (ctx->d_tensors_enc) cudaFree(ctx->d_tensors_enc);
    if (ctx->d_tensors_dec) cudaFree(ctx->d_tensors_dec);
    for (int i = 0; i < rb200_ctx::kMaxSlices; i++) {
        if (ctx->ev_in[i]) cudaEventDestroy(ctx->ev_in[i]);
        if (ctx->ev_done[i]) cudaEventDestroy(ctx->ev_done[i]);
    }
    if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
    if (ctx->ev_out) cudaEventDestroy(ctx->ev_out);
    if (ctx->s_in) cudaStreamDestroy(ctx->s_in);
    if (ctx->s_out) cudaStreamDestroy(ctx->s_out);
    delete ctx;
}

extern "C" int rb200_ctx_set_stream(rb200_ctx* ctx, void* stream)
{
    if (!ctx) return RB200_E_ARG;
    ctx->stream = static_cast<cudaStream_t>(stream);
    return RB200_OK;
}

extern "C" const char* rb200_last_cuda_error(const rb200_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }
extern "C" uint64_t rb200_launch_count(const rb200_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int rb200_sync(rb200_ctx* ctx)
{
    if (!ctx) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    RB_CUDA(ctx, cudaMemcpyAsync(ctx->h_status, ctx->d_status, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, sizeof(uint32_t), ctx->stream));
    RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*ctx->h_status) RB_CUDA(ctx, cudaMemsetAsync(ctx->d_work, 0, sizeof(DecodeWork), ctx->stream));   // a kernel may have bailed out
    return status_to_code(*ctx->h_status);
}

// ---------------------------------------------------------------------------
// models
// ---------------------------------------------------------------------------

extern "C" void rb200_model_destroy(rb200_model* m)
{
    if (!m) return;
    DeviceGuard g(m->ctx->device);
    cudaStreamSynchronize(m->ctx->stream);
    cudaFree(m->d_word_dec); cudaFree(m->d_word_enc);
    cudaFree(m->d_alias_dec); cudaFree(m->d_alias_enc); cudaFree(m->d_alias_remap);
    cudaFree(m->d_byte_dec); cudaFree(m->d_byte_enc);
    cudaFree(m->d_r64_dec); cudaFree(m->d_r64_enc);
    cudaFree(m->d_freqs);
    delete m;
}

namespace {
// RB200_WORD_RECIPROCAL=33 forces the any-x (33-bit) reciprocal even where the 32-bit one is exact (testing)
bool word_r32_allowed()
{
    static const bool allowed = [] {
        const char* e = std::getenv("RB200_WORD_RECIPROCAL");
        return !(e && std::strcmp(e, "33") == 0);
    }();
    return allowed;
}
}  // namespace

extern "C" int rb200_model_create(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint32_t freqs[256], rb200_model** out)
{
    if (!ctx || !freqs || !out) return RB200_E_ARG;
    *out = nullptr;
    DeviceGuard g(ctx->device);
    rb200_model* m = new (std::nothrow) rb200_model;
    if (!m) return RB200_E_NOMEM;
    m->ctx = ctx;
    m->coder = coder;
    m->scale_bits = scale_bits;
    int rc = RB200_OK;
    cudaError_t e = cudaSuccess;
    if (coder == RB200_CODER_WORD) {
        if (scale_bits != kWordScaleBits) { delete m; return RB200_E_ARG; }
        WordDeviceTables* t = new (std::nothrow) WordDeviceTables;
        if (!t) { delete m; return RB200_E_NOMEM; }
        rc = build_word_device_tables(freqs, *t);
        if (rc == RB200_OK) {
            m->wide = t->wide;
            m->enc_r32 = t->enc32_ok && word_r32_allowed();
            e = cudaMalloc(&m->d_word_dec, sizeof t->dec);
            if (e == cudaSuccess) e = cudaMalloc(&m->d_word_enc, sizeof t->enc);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_word_dec, t->dec, sizeof t->dec, cudaMemcpyHostToDevice);
            if (e == cudaSuccess)
                e = cudaMemcpy(m->d_word_enc, m->enc_r32 ? t->enc32 : t->enc, sizeof t->enc, cudaMemcpyHostToDevice);
        }
        delete t;
    } else if (coder == RB200_CODER_ALIAS) {
        AliasDeviceTables* t = new (std::nothrow) AliasDeviceTables;
        if (!t) { delete m; return RB200_E_NOMEM; }
        rc = build_alias_device_tables(freqs, scale_bits, *t);
        if (rc == RB200_OK) {
            const size_t remap_bytes = t->remap.size() * sizeof(uint16_t);
            e = cudaMalloc(&m->d_alias_dec, sizeof t->dec);
            if (e == cudaSuccess) e = cudaMalloc(&m->d_alias_enc, sizeof t->enc);
            if (e == cudaSuccess) e = cudaMalloc(&m->d_alias_remap, remap_bytes);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_alias_dec, t->dec, sizeof t->dec, cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_alias_enc, t->enc, sizeof t->enc, cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_alias_remap, t->remap.data(), remap_bytes, cudaMemcpyHostToDevice);
        }
        delete t;
    } else if (coder == RB200_CODER_BYTE) {
        ByteDeviceTables* t = new (std::nothrow) ByteDeviceTables;
        if (!t) { delete m; return RB200_E_NOMEM; }
        rc = build_byte_device_tables(freqs, scale_bits, *t);
        if (rc == RB200_OK) {
            e = cudaMalloc(&m->d_byte_dec, t->dec.size());
            if (e == cudaSuccess) e = cudaMalloc(&m->d_byte_enc, sizeof t->enc);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_byte_dec, t->dec.data(), t->dec.size(), cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_byte_enc, t->enc, sizeof t->enc, cudaMemcpyHostToDevice);
        }
        delete t;
    } else if (coder == RB200_CODER_RANS64) {
        Rans64DeviceTables* t = new (std::nothrow) Rans64DeviceTables;
        if (!t) { delete m; return RB200_E_NOMEM; }
        rc = build_rans64_device_tables(freqs, scale_bits, *t);
        if (rc == RB200_OK) {
            e = cudaMalloc(&m->d_r64_dec, t->dec.size());
            if (e == cudaSuccess) e = cudaMalloc(&m->d_r64_enc, sizeof t->enc);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_r64_dec, t->dec.data(), t->dec.size(), cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = cudaMemcpy(m->d_r64_enc, t->enc, sizeof t->enc, cudaMemcpyHostToDevice);
        }
        delete t;
    } else {
        delete m;
        return RB200_E_ARG;
    }
    std::memcpy(m->freqs, freqs, sizeof m->freqs);
    if (rc == RB200_OK && e == cudaSuccess) e = cudaMalloc(&m->d_freqs, sizeof m->freqs);
    if (rc == RB200_OK && e == cudaSuccess) e = cudaMemcpy(m->d_freqs, m->freqs, sizeof m->freqs, cudaMemcpyHostToDevice);
    if (rc != RB200_OK || e != cudaSuccess) {
        if (e != cudaSuccess) rc = cuda_fail(ctx, e, "model upload");
        rb200_model_destroy(m);
        return rc;
    }
    *out = m;
    return RB200_OK;
}

// ---------------------------------------------------------------------------
// geometry
// ---------------------------------------------------------------------------

extern "C" size_t rb200_chunk_count(size_t n, uint32_t chunk_syms)
{
    if (!chunk_syms) return 0;
    return n / chunk_syms + (n % chunk_syms != 0);      // no wrap-around for any n
}

// A chunk stream never exceeds 512 + 2 * symbols bytes, whatever the coder: the word coder emits
// <= one u16 per symbol (rans_word_sse41.h:85-89) after a 128-byte header; the byte coders emit
// <= two bytes per symbol at scale_bits <= 16 (state < 2^31, x_max >= 2^15; rans_byte.h:64-70);
// rans64 emits one u32 per 32 bits of information, <= scale_bits/8 <= 2 bytes per symbol plus at
// most one extra word per lane, after a 256-byte header.  Streams are padded to multiples of 16.
extern "C" size_t rb200_encode_bound(size_t n, uint32_t chunk_syms)
{
    if (!chunk_syms) return 0;
    const size_t full = n / chunk_syms, tail = n % chunk_syms;
    size_t b = full * round16(kBoundFixed + 2ull * chunk_syms);
    if (tail) b += round16(kBoundFixed + 2ull * tail);
    return b;
}

// ---------------------------------------------------------------------------
// device-resident hot path
// ---------------------------------------------------------------------------

namespace {


// directory + compaction after any encode kernel: sizes[] -> offsets[] + blob.  geom set: the GEOM instances, on grids
// sized for n_chunks (the bound's), with d_blob the container, in which they find the directory and the blob from the
// record (d_offsets unused).  choice set: the GATED instances, which run only when the record names `group`.  stored
// set (the stored encode, ungated): compact_stored_kernel, which copies the stored blocks' chunks from the input
// (with geom: compact_stored_varlen_kernel).
int finish_encode(rb200_ctx* ctx, uint8_t* scratch, uint32_t slot, uint32_t* sizes, uint64_t* tile_sums, uint32_t n_chunks,
                  uint8_t* d_blob, size_t blob_cap, uint64_t* d_offsets, const VarlenGeom* geom, const CoderChoice* choice, uint32_t group,
                  const StoredBlocks* stored = nullptr)
{
    if (!n_chunks) {
        RB_CUDA(ctx, cudaMemsetAsync(d_offsets, 0, sizeof(uint64_t), ctx->stream));
        return RB200_OK;
    }
    const uint32_t tiles = (n_chunks + kScanTile - 1) / kScanTile;
    auto scan = choice ? (geom ? scan_tiles_kernel<true, true> : scan_tiles_kernel<false, true>)
                       : (geom ? scan_tiles_kernel<true> : scan_tiles_kernel<false>);
    scan<<<tiles, 1024, 0, ctx->stream>>>(sizes, n_chunks, geom ? reinterpret_cast<uint64_t*>(d_blob) : d_offsets, tile_sums, geom, choice,
                                          group);
    int rc = check_launch(ctx, "scan_tiles_kernel");
    if (rc != RB200_OK) return rc;
    const uint32_t prefixed = tiles > kTilePrefixThreshold ? 1u : 0u;
    if (prefixed) {
        auto prefix = choice ? (geom ? tile_prefix_kernel<true, true> : tile_prefix_kernel<false, true>)
                             : (geom ? tile_prefix_kernel<true> : tile_prefix_kernel<false>);
        prefix<<<1, 1024, 0, ctx->stream>>>(tile_sums, tiles, geom, choice, group);
        rc = check_launch(ctx, "tile_prefix_kernel");
        if (rc != RB200_OK) return rc;
    }
    const uint32_t grid = (n_chunks + kCopyWarps - 1) / kCopyWarps;
    if (stored && geom) {
        compact_stored_varlen_kernel<<<grid, kCopyWarps * 32, 0, ctx->stream>>>(scratch, slot, sizes, tile_sums, prefixed, d_blob, ctx->d_status,
                                                                                geom, *stored);
        return check_launch(ctx, "compact_stored_varlen_kernel");
    }
    if (stored) {
        compact_stored_kernel<<<grid, kCopyWarps * 32, 0, ctx->stream>>>(scratch, slot, sizes, d_offsets, tile_sums, prefixed, n_chunks, d_blob,
                                                                         blob_cap, ctx->d_status, *stored);
        return check_launch(ctx, "compact_stored_kernel");
    }
    auto compact = choice ? (geom ? compact_kernel<true, true> : compact_kernel<false, true>)
                          : (geom ? compact_kernel<true> : compact_kernel<false>);
    compact<<<grid, kCopyWarps * 32, 0, ctx->stream>>>(scratch, slot, sizes, d_offsets, tile_sums, prefixed, n_chunks, d_blob, blob_cap,
                                                        ctx->d_status, geom, choice, group);
    return check_launch(ctx, "compact_kernel");
}

// Word-coder encode has three paths:
//   fused: ONE persistent launch -- workers encode, a scanner warp turns published sizes into end offsets
//          in chunk order, workers place chunk k after encoding chunk k+1 (placement.cuh);
//   ring:  the fused launch with every stream kept in its warp's shared-memory ring until it is placed with TMA bulk
//          copies (K2r, encode_ring.cuh): what does not fit the ring goes to per-warp spill slots; for chunks of
//          <= kEncRingMaxChunk symbols, whose worst-case stream fits a slot, and models the host knows satisfy word_ring_model (so not for
//          rb200_container_model_encode_async, whose model is built on the GPU);
//   split: three launches -- encode into per-chunk worst-case slots, tile scan, compaction.
// fused is faster as long as the scanner keeps up, i.e. for chunks of >= 4096 symbols; below that the split path
// is used (H100 SXM at a 400 W power limit, 1 GiB uniform bytes: 1.89 vs 2.21 ms per call at chunks of 8192, 2.10 vs
// 2.25 ms at 4096, but 2.80 vs 2.36 ms at 2048).  Where both fit, ring replaces fused (DESIGN.md section 4).
// RB200_ENCODE_PATH=split|fused forces one of those two.  Only the encode plans (plan_encode, plan_blocks_encode) ask.
int forced_encode_path()                     // RB200_ENCODE_PATH: 1 fused, 0 split, -1 not set
{
    static const int forced = [] {           // read once; thread-safe static initialisation
        const char* e = std::getenv("RB200_ENCODE_PATH");
        return !e ? -1 : (std::strcmp(e, "fused") == 0 ? 1 : (std::strcmp(e, "split") == 0 ? 0 : -1));
    }();
    return forced;
}

bool use_fused_encode(uint32_t chunk_syms)
{
    // two worst-case slots per resident warp: keep that scratch below ~2 GB (chunks of <= 64 Ki symbols)
    if (chunk_syms > 65536) return false;
    if (forced_encode_path() >= 0) return forced_encode_path() == 1;
    return chunk_syms >= 4096;
}

// How one encode call over n_chunks chunks runs, decided once: the path, the encode launch's shape, and the workspace
// both need.  Fused: one launch of `grid` CTAs with `slots` scratch slots (slots per worker warp x the warps of the grid; ring: a pair of spill slots per warp);
// in ctx->sizes the chunk counter (16 bytes), then look[n_chunks] (placement.cuh).  Split: the encode launch into one
// slot per chunk, then finish_encode; in ctx->sizes sizes[n_chunks], then the scan's tile sums.
struct EncodePlan {
    bool fused;
    bool ring;                         // word coder, fused: K2r instead of K2f
    uint32_t grid, threads, smem;      // the encode launch (dynamic shared memory in bytes)
    size_t slots;
    uint32_t slot_bytes;
    uint32_t n_chunks;
};

// A word model whose streams fit K2r's ring: no symbol holds all 4096 slots.  Such a symbol's x_max wraps to 0
// (word_enc_expand), so every step emits a word: 2 * chunk_syms + 128 bytes per chunk, so
// every stream would go largely through K2r's spill slots; K2f takes those models.
bool word_ring_model(const uint32_t freqs[256])
{
    for (int s = 0; s < 256; s++)
        if (freqs[s] >= kWordSlots) return false;
    return true;
}

// ring_model: the word model is known to satisfy word_ring_model (a model built on the GPU is not known to)
// split: the split path whatever the chunk size (rb200_container_stored_encode_async needs every stream's size first)
EncodePlan plan_encode(const rb200_ctx* ctx, int coder, uint32_t scale_bits, uint32_t n_chunks, uint32_t chunk_syms, bool ring_model,
                       bool split = false)
{
    EncodePlan p = {};
    p.n_chunks = n_chunks;
    p.slot_bytes = slot_bytes_for(chunk_syms);
    p.fused = !split && n_chunks && coder != RB200_CODER_RANS64 && use_fused_encode(chunk_syms);
    p.slots = n_chunks;
    const uint32_t sms = static_cast<uint32_t>(ctx->sms);
    if (coder == RB200_CODER_WORD) {
        p.threads = kEncWarps * 32;
        p.smem = kEncSmemBytes;
        p.ring = p.fused && ring_model && forced_encode_path() < 0 && chunk_syms <= kEncRingMaxChunk;
        if (p.ring) {
            p.threads = kEncRingWarps * 32;
            p.smem = kEncRingSmemBytes;
            p.grid = std::min((n_chunks + 1 + kEncRingWarps - 1) / kEncRingWarps, sms);
            p.slots = static_cast<size_t>(p.grid) * kEncRingWarps;     // one pair of spill slots per warp
            p.slot_bytes = kEncRingSpillBytes;
        } else if (p.fused) {
            const uint32_t want = (n_chunks + 1 + kEncWarps - 1) / kEncWarps;     // + 1: one warp of the grid is the scanner
            p.grid = std::min(want, sms * RB200_FUSED_MINBLOCKS);
            p.slots = static_cast<size_t>(p.grid) * kEncWarps * kFusedSlots;
        } else {
            p.grid = (n_chunks + kEncWarps - 1) / kEncWarps;
        }
    } else if (coder == RB200_CODER_RANS64) {
        p.threads = kRans64Warps * 32;
        p.smem = kRans64EncSmemBytes;
        p.grid = (n_chunks + kRans64Warps - 1) / kRans64Warps;
    } else {                           // alias / byte: persistent, at most one CTA per SM
        p.threads = kAliasEncWarps * 32;
        p.smem = alias_encode_smem(coder == RB200_CODER_ALIAS, scale_bits);
        p.grid = std::min((n_chunks + (p.fused ? 1 : 0) + kAliasEncWarps - 1) / kAliasEncWarps, sms);
        if (p.fused) p.slots = static_cast<size_t>(sms) * kAliasEncWarps * kAliasFusedSlots;
    }
    return p;
}

// Bytes of the u32 part of ctx->sizes (the fused path's counter, the split path's sizes[]); the u64 part follows.
size_t plan_head_bytes(const EncodePlan& p)
{
    return p.fused ? 16 : round16((static_cast<size_t>(p.n_chunks) + 1) * sizeof(uint32_t));
}

// Grows ctx->scratch and ctx->sizes to what `p` needs (the host pipeline does this once for its largest slice so that
// no slice has to stall on a reallocation).
int reserve_plan(rb200_ctx* ctx, const EncodePlan& p)
{
    const size_t n = p.n_chunks;
    const size_t longs = p.fused ? n : (n + kScanTile - 1) / kScanTile + 1;
    int rc = reserve(ctx, ctx->scratch, p.slots * p.slot_bytes + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->sizes, plan_head_bytes(p) + longs * sizeof(uint64_t));
    return rc;
}

// The workspace of a plan, as the encode kernels take it; the pointers of the other path are null.
struct EncodeWorkspace {
    uint8_t* scratch;
    uint32_t* counter;     // fused
    uint64_t* look;        // fused
    uint32_t* sizes;       // split
    uint64_t* tile_sums;   // split
};

// Reserves the workspace of a plan and lays it out; fused: zeroes the counter and look[] on the stream.
int prepare_workspace(rb200_ctx* ctx, const EncodePlan& p, EncodeWorkspace* ws)
{
    int rc = reserve_plan(ctx, p);
    if (rc != RB200_OK) return rc;
    uint8_t* scratch = static_cast<uint8_t*>(ctx->scratch.p);
    uint32_t* head = static_cast<uint32_t*>(ctx->sizes.p);
    uint64_t* tail = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(ctx->sizes.p) + plan_head_bytes(p));
    if (p.fused) {
        RB_CUDA(ctx, cudaMemsetAsync(ctx->sizes.p, 0, 16 + static_cast<size_t>(p.n_chunks) * sizeof(uint64_t), ctx->stream));
        *ws = EncodeWorkspace{scratch, head, tail, nullptr, nullptr};
    } else {
        *ws = EncodeWorkspace{scratch, nullptr, nullptr, head, tail};
    }
    return RB200_OK;
}

// Runs a plan: prepare its workspace; fused: `launch(ws)`, the one kernel; split: `launch(ws)` encodes into the slots
// (when there are chunks), then finish_encode (geom, choice, group: as there).  `launch` returns check_launch's code.
template <class Launch>
int run_encode(rb200_ctx* ctx, const EncodePlan& p, uint8_t* d_blob, size_t blob_cap, uint64_t* d_offsets, const VarlenGeom* geom,
               Launch launch, const CoderChoice* choice = nullptr, uint32_t group = 0)
{
    EncodeWorkspace ws = {};
    int rc = prepare_workspace(ctx, p, &ws);
    if (rc != RB200_OK) return rc;
    if (p.fused) return launch(ws);
    if (p.n_chunks) {
        rc = launch(ws);
        if (rc != RB200_OK) return rc;
    }
    return finish_encode(ctx, ws.scratch, p.slot_bytes, ws.sizes, ws.tile_sums, p.n_chunks, d_blob, blob_cap, d_offsets, geom, choice,
                         group);
}

// The encode tables of one encode call, in device memory.  Word: `word_gate` null runs the instance word_r32 names on
// word[word_r32]; set, both GATED instances run (word_kernels.cuh), each on its own table, and *word_gate picks one.
// choice set (the auto encode): the other coders' GATED instances, and those of the split path's directory and
// compaction, which run only when the record names `group`; scale_bits is then the largest of the group.
struct EncodeTables {
    int coder;
    uint32_t scale_bits;
    const WordEncEntry* word[2];       // the 33-bit and the 32-bit reciprocal tables
    int word_r32;
    const uint32_t* word_gate;
    const AliasEncEntry* enc;          // alias / byte
    const uint16_t* remap;             // alias
    const uint4* r64;                  // rans64
    bool word_ring = false;            // word: the model satisfies word_ring_model
    const CoderChoice* choice = nullptr;
    uint32_t group = 0;
};

EncodeTables model_tables(const rb200_model* m)
{
    return EncodeTables{m->coder, m->scale_bits, {m->d_word_enc, m->d_word_enc}, m->enc_r32, nullptr,
                        m->coder == RB200_CODER_ALIAS ? m->d_alias_enc : m->d_byte_enc, m->d_alias_remap, m->d_r64_enc,
                        word_ring_model(m->freqs)};
}

// The encode launch of plan p with tables t on workspace ws (split: into the slots; fused: the one kernel).
int launch_encoder(rb200_ctx* ctx, const EncodeTables& t, const EncodePlan& p, const uint8_t* d_in, size_t n, uint32_t chunk_syms,
                   uint32_t n_chunks, const EncodeWorkspace& ws, uint8_t* d_blob, size_t blob_cap, uint64_t* d_offsets, const VarlenGeom* geom)
{
    if (t.coder == RB200_CODER_WORD) {
        const WordEncEntry* table = t.word[t.word_r32 ? 1 : 0];
        if (p.ring) {
            auto kernel = t.word_r32 ? word_encode_ring_kernel<true> : word_encode_ring_kernel<false>;
            kernel<<<p.grid, p.threads, p.smem, ctx->stream>>>(d_in, n, chunk_syms, n_chunks, table, ws.scratch, ws.look, ws.counter,
                                                               d_blob, blob_cap, d_offsets, ctx->d_status);
            return check_launch(ctx, "word_encode_ring_kernel");
        }
        // the instance word_r32 names, or both GATED ones
        int rc = RB200_OK;
        const int r32_first = t.word_gate ? 0 : t.word_r32, r32_last = t.word_gate ? 1 : t.word_r32;
        for (int r32 = r32_first; r32 <= r32_last && rc == RB200_OK; r32++) {
            if (p.fused) {
                auto kernel = !t.word_gate ? (r32 ? word_encode_fused_kernel<true> : word_encode_fused_kernel<false>)
                              : !geom  ? (r32 ? word_encode_fused_kernel<true, true> : word_encode_fused_kernel<false, true>)
                                       : (r32 ? word_encode_fused_kernel<true, true, true> : word_encode_fused_kernel<false, true, true>);
                kernel<<<p.grid, p.threads, p.smem, ctx->stream>>>(d_in, n, chunk_syms, n_chunks, t.word[r32], ws.scratch, p.slot_bytes, ws.look,
                                                                   ws.counter, d_blob, blob_cap, d_offsets, ctx->d_status, t.word_gate, geom);
                rc = check_launch(ctx, "word_encode_fused_kernel");
            } else {
                auto kernel = !t.word_gate ? (r32 ? word_encode_kernel<true> : word_encode_kernel<false>)
                              : !geom  ? (r32 ? word_encode_kernel<true, true> : word_encode_kernel<false, true>)
                                       : (r32 ? word_encode_kernel<true, true, true> : word_encode_kernel<false, true, true>);
                kernel<<<p.grid, p.threads, p.smem, ctx->stream>>>(d_in, n, chunk_syms, n_chunks, t.word[r32], ws.scratch, p.slot_bytes, ws.sizes,
                                                                   ctx->d_status, t.word_gate, geom);
                rc = check_launch(ctx, "word_encode_kernel");
            }
        }
        return rc;
    }
    if (t.coder == RB200_CODER_RANS64) {
        auto kernel = t.choice ? (geom ? rans64_encode_kernel<true, true> : rans64_encode_kernel<false, true>)
                               : (geom ? rans64_encode_kernel<true> : rans64_encode_kernel<false>);
        kernel<<<p.grid, p.threads, p.smem, ctx->stream>>>(d_in, n, chunk_syms, n_chunks, t.scale_bits, t.r64, ws.scratch, p.slot_bytes,
                                                           ws.sizes, ctx->d_status, geom, t.choice, t.group);
        return check_launch(ctx, "rans64_encode_kernel");
    }
    const bool alias = t.coder == RB200_CODER_ALIAS;
    launch_alias_encode(ctx->stream, p.grid, p.smem, d_in, n, chunk_syms, n_chunks, t.scale_bits, t.enc, alias ? t.remap : nullptr,
                        ws.scratch, p.slot_bytes, ws.sizes, ws.look, ws.counter, d_blob, blob_cap, d_offsets, ctx->d_status, geom,
                        t.choice, t.group);
    return check_launch(ctx, alias ? "alias_encode_kernel" : "byte_encode_kernel");
}

// geom set (rb200_container_model_encode_varlen_async): n is the bound n_max, which fixes the plan and every launch
// shape, the GEOM instances read n, the chunk count and the blob's place from the record, and d_blob is the container.
int encode_device(rb200_ctx* ctx, const EncodeTables& t, const uint8_t* d_in, size_t n, uint32_t chunk_syms, uint8_t* d_blob,
                  size_t blob_cap, uint64_t* d_offsets, const VarlenGeom* geom = nullptr)
{
    const size_t n_chunks_sz = rb200_chunk_count(n, chunk_syms);
    if (n_chunks_sz >= (1ull << 31)) return RB200_E_ARG;
    const uint32_t n_chunks = static_cast<uint32_t>(n_chunks_sz);
    const EncodePlan p = plan_encode(ctx, t.coder, t.scale_bits, n_chunks, chunk_syms, t.word_ring);
    return run_encode(ctx, p, d_blob, blob_cap, d_offsets, geom, [&](const EncodeWorkspace& ws) {
        return launch_encoder(ctx, t, p, d_in, n, chunk_syms, n_chunks, ws, d_blob, blob_cap, d_offsets, geom);
    }, t.choice, t.group);
}

int decode_device(rb200_ctx* ctx, const rb200_model* model, const uint8_t* d_blob, size_t blob_size, const uint64_t* d_offsets,
                  uint32_t chunk_syms, uint8_t* d_out, size_t n)
{
    const size_t n_chunks_sz = rb200_chunk_count(n, chunk_syms);
    if (n_chunks_sz >= (1ull << 31)) return RB200_E_ARG;
    const uint32_t n_chunks = static_cast<uint32_t>(n_chunks_sz);
    if (!n_chunks) return RB200_OK;
    if (model->coder == RB200_CODER_WORD) {
        // persistent grid: 2 CTAs of 32 warps per SM, chunks handed out by an atomic counter (word_decode_tma.cuh)
        const uint32_t want = (n_chunks + DecShip::kWarps - 1) / DecShip::kWarps;
        const uint32_t full = static_cast<uint32_t>(ctx->sms) * DecShip::kMinBlocks;
        const uint32_t grid = want < full ? want : full;
        auto kernel = model->wide ? word_decode_tma_kernel<DecShip, true> : word_decode_tma_kernel<DecShip, false>;
        kernel<<<grid, DecShip::kWarps * 32, DecShip::kSmemBytes, ctx->stream>>>(d_blob, blob_size, d_offsets, model->d_word_dec, d_out, n,
                                                                                 chunk_syms, n_chunks, ctx->d_work, ctx->d_status, 0);
        return check_launch(ctx, "word_decode_tma_kernel");
    }
    if (model->coder == RB200_CODER_RANS64) {
        launch_rans64_decode(ctx->stream, d_blob, blob_size, d_offsets, model->scale_bits, model->d_r64_dec, d_out, n, chunk_syms,
                             n_chunks, ctx->d_status);
        return check_launch(ctx, "rans64_decode_kernel");
    }
    if (model->coder == RB200_CODER_BYTE) {
        launch_byte_decode(ctx->stream, d_blob, blob_size, d_offsets, model->scale_bits, model->d_byte_dec, d_out, n, chunk_syms,
                           n_chunks, ctx->d_status);
        return check_launch(ctx, "byte_decode_kernel");
    }
    launch_alias_decode(ctx->stream, d_blob, blob_size, d_offsets, model->scale_bits, model->d_alias_dec, d_out, n, chunk_syms, n_chunks,
                        ctx->d_status, ctx->d_work, static_cast<uint32_t>(ctx->sms));
    return check_launch(ctx, "alias_decode_persist_kernel");
}

}  // namespace

namespace {

int reserve_dir(rb200_ctx* ctx, size_t entries)
{
    if (entries <= ctx->h_dir_cap) return RB200_OK;
    if (ctx->h_dir) {
        RB_CUDA(ctx, cudaStreamSynchronize(ctx->s_in));
        RB_CUDA(ctx, cudaStreamSynchronize(ctx->s_out));
        RB_CUDA(ctx, cudaFreeHost(ctx->h_dir));
        ctx->h_dir = nullptr;
        ctx->h_dir_cap = 0;
    }
    const size_t want = entries + entries / 8 + 64;
    cudaError_t e = cudaMallocHost(&ctx->h_dir, want * sizeof(uint64_t));
    if (e != cudaSuccess) {
        ctx->h_dir = nullptr;
        cuda_fail(ctx, e, "cudaMallocHost(directory staging)");
        return RB200_E_NOMEM;
    }
    ctx->h_dir_cap = want;
    return RB200_OK;
}

// Runs `enqueue`, the part of a host pipeline that puts work on the three streams.  An error exit must not leave copies
// in flight: they target the caller's buffers and the context's staging, which a later reserve() may free.  So any
// non-OK result first drains the streams, and clears whatever the kernels flagged.
template <class Enqueue>
int run_pipeline(rb200_ctx* ctx, Enqueue enqueue)
{
    const int rc = enqueue();
    if (rc != RB200_OK) {
        cudaStreamSynchronize(ctx->s_in);
        cudaStreamSynchronize(ctx->stream);
        cudaStreamSynchronize(ctx->s_out);
        cudaMemsetAsync(ctx->d_status, 0, sizeof(uint32_t), ctx->stream);
        cudaMemsetAsync(ctx->d_work, 0, sizeof(DecodeWork), ctx->stream);
        cudaStreamSynchronize(ctx->stream);
    }
    return rc;
}

// One pipeline slice of a host-mode call: units [u0, u0 + units) = chunks [c0, c0 + cnt) = symbols [lo, lo + len).
// A unit is one chunk for rb200_encode / rb200_decode and one block for the per-block calls.
struct Slice {
    size_t u0, units, c0, cnt, lo, len;
};

// Slice plan for the host pipeline.  Steady-state slices are `RB200_SLICE_MIB` (default 32 MiB) of symbols:
// big enough that PCIe time dwarfs launch overhead and the per-slice host wake-up, small enough to overlap.
// The first and last three slices ramp (1/8, 1/4, 1/2 of that) so that the pipeline fill (first H2D) and
// drain (last D2H), which nothing overlaps, are short.  Returns the number of slices (<= kMaxSlices).
// Slices hold whole units of `unit_syms` symbols and `unit_chunks` chunks.
size_t plan_slices(size_t n, uint32_t unit_syms, uint32_t unit_chunks, Slice* out)
{
    static const size_t tuned = [] {        // tuning knob for the host pipeline (1..1024 MiB)
        const char* e = std::getenv("RB200_SLICE_MIB");
        const long v = e ? std::atol(e) : 0;
        return (v >= 1 && v <= 1024) ? static_cast<size_t>(v) << 20 : static_cast<size_t>(32u << 20);
    }();
    const size_t total = rb200_chunk_count(n, unit_syms);
    size_t tc = (tuned + unit_syms - 1) / unit_syms;                  // units per steady-state slice
    if (tc == 0) tc = 1;
    const size_t room = rb200_ctx::kMaxSlices - 8;
    if (total / tc >= room) tc = total / room + 1;
    size_t ramp[3] = {tc / 8, tc / 4, tc / 2};
    const bool ramped = total >= 4 * tc && ramp[0] > 0;
    size_t k = 0, c = 0;
    auto push = [&](size_t cnt) {
        if (cnt == 0) return;
        if (cnt > total - c) cnt = total - c;
        const size_t lo = c * unit_syms;
        const size_t len = (n - lo < cnt * unit_syms) ? n - lo : cnt * unit_syms;
        out[k++] = Slice{c, cnt, c * unit_chunks, cnt * unit_chunks, lo, len};
        c += cnt;
    };
    const size_t tail = ramped ? ramp[0] + ramp[1] + ramp[2] : 0;
    if (ramped)
        for (int r = 0; r < 3; r++) push(ramp[r]);
    while (total - c > tail) push((total - c - tail < tc) ? total - c - tail : tc);
    if (ramped)
        for (int r = 2; r >= 0; r--) push(ramp[r]);
    return k;
}

// A table of `unit_bytes` per unit that a host pipeline moves along with each slice (the per-block frequency tables),
// staged in ctx->st_aux: copied in before the slice runs when `in` is set, or out after it when `out` is set.
struct UnitTable {
    const void* in;
    void* out;
    size_t unit_bytes;
};

// Optional per-slice work of a host pipeline, enqueued on ctx->stream once the slice's bytes are on the device:
// `(i, d_data, d_len, cap)` after slice i's encode, whose staged container is d_data[0, *d_len) with *d_len <= cap;
// `(i, d_data, len)` before
// slice i's decode, whose blob bytes are d_data[0, len).  rb200_container_encode / _decode CRC the blob with it.
struct NoSliceHook {
    int operator()(size_t, const uint8_t*, const uint64_t*, size_t) const { return RB200_OK; }
    int operator()(size_t, const uint8_t*, size_t) const { return RB200_OK; }
};

// Host buffers -> blob, overlapped: slice i+1 is copied in while slice i is encoded and slice i-1 is
// copied out.  Every slice is its own container in a staging region; because containers end 16-byte
// aligned they concatenate, and the directory entries only need the running base added.  Directories are
// staged in pinned memory (an async copy to a pageable `offsets` would block the issuing thread).
// `plan_slice(slice)` is the encode plan of a slice; the plan of the largest slice is reserved up front, so that no
// slice stalls on a reallocation.  `encode_slice(slice, d_in, d_table, d_blob, cap, d_offsets)` enqueues one slice's
// encode on ctx->stream.
template <class PlanSlice, class EncodeSlice, class Hook = NoSliceHook>
int encode_pipeline(rb200_ctx* ctx, const uint8_t* in, size_t n, uint32_t chunk_syms, uint32_t unit_chunks, UnitTable tab,
                    PlanSlice plan_slice, EncodeSlice encode_slice, uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size,
                    Hook hook = Hook{})
{
    if (n == 0) {
        offsets[0] = 0;
        if (blob_size) *blob_size = 0;
        return RB200_OK;
    }
    const uint32_t unit_syms = chunk_syms * unit_chunks;
    const size_t n_units = rb200_chunk_count(n, unit_syms), n_chunks = n_units * unit_chunks;
    Slice sl[rb200_ctx::kMaxSlices];
    const size_t n_slices = plan_slices(n, unit_syms, unit_chunks, sl);
    const Slice* largest = &sl[0];
    for (size_t i = 1; i < n_slices; i++) largest = sl[i].units > largest->units ? &sl[i] : largest;
    const size_t slot = slot_bytes_for(chunk_syms);
    // slice i's container is built at bound(symbols before it); its directory at c0 + i (cnt + 1 entries)
    int rc = reserve(ctx, ctx->st_in, n + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_blob, n_chunks * slot + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_offsets, (n_chunks + n_slices) * sizeof(uint64_t));
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_aux, n_units * tab.unit_bytes);
    if (rc == RB200_OK) rc = reserve_dir(ctx, n_chunks + n_slices);
    if (rc == RB200_OK) rc = reserve_plan(ctx, plan_slice(*largest));
    if (rc != RB200_OK) return rc;
    uint8_t* d_in = static_cast<uint8_t*>(ctx->st_in.p);
    uint8_t* d_blob = static_cast<uint8_t*>(ctx->st_blob.p);
    uint64_t* d_off = static_cast<uint64_t*>(ctx->st_offsets.p);
    uint8_t* d_tab = static_cast<uint8_t*>(ctx->st_aux.p);
    const size_t tb = tab.unit_bytes;

    return run_pipeline(ctx, [&]() -> int {
        RB_CUDA(ctx, cudaEventRecord(ctx->ev_start, ctx->stream));       // staging buffers may still be in use upstream
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_in, ctx->ev_start, 0));
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_out, ctx->ev_start, 0));
        auto issue = [&](size_t i) -> int {      // H2D + kernels for slice i
            const Slice& s = sl[i];
            RB_CUDA(ctx, cudaMemcpyAsync(d_in + s.lo, in + s.lo, s.len, cudaMemcpyHostToDevice, ctx->s_in));
            if (tab.in)
                RB_CUDA(ctx, cudaMemcpyAsync(d_tab + s.u0 * tb, static_cast<const uint8_t*>(tab.in) + s.u0 * tb, s.units * tb,
                                             cudaMemcpyHostToDevice, ctx->s_in));
            RB_CUDA(ctx, cudaEventRecord(ctx->ev_in[i], ctx->s_in));
            RB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[i], 0));
            uint64_t* so = d_off + s.c0 + i;
            int r = encode_slice(s, d_in + s.lo, d_tab + s.u0 * tb, d_blob + s.c0 * slot, s.cnt * slot, so);
            if (r == RB200_OK) r = hook(i, d_blob + s.c0 * slot, so + s.cnt, s.cnt * slot);
            if (r != RB200_OK) return r;
            RB_CUDA(ctx, cudaMemcpyAsync(&ctx->h_slice_total[i], so + s.cnt, sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
            RB_CUDA(ctx, cudaEventRecord(ctx->ev_done[i], ctx->stream));
            return RB200_OK;
        };
        int r = issue(0);
        if (r != RB200_OK) return r;
        size_t base = 0;
        bool overflow = false;
        for (size_t i = 0; i < n_slices; i++) {
            if (i + 1 < n_slices) {
                r = issue(i + 1);
                if (r != RB200_OK) return r;
            }
            RB_CUDA(ctx, cudaEventSynchronize(ctx->ev_done[i]));          // slice i's size is now on the host
            const size_t total = static_cast<size_t>(ctx->h_slice_total[i]);
            const Slice& s = sl[i];
            if (base + total > blob_cap) {
                overflow = true;                                          // finish the slices, copy nothing more out
            } else if (!overflow) {
                RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_out, ctx->ev_done[i], 0));
                RB_CUDA(ctx, cudaMemcpyAsync(blob + base, d_blob + s.c0 * slot, total, cudaMemcpyDeviceToHost, ctx->s_out));
                RB_CUDA(ctx, cudaMemcpyAsync(ctx->h_dir + s.c0 + i, d_off + s.c0 + i, s.cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                                             ctx->s_out));
                if (tab.out)
                    RB_CUDA(ctx, cudaMemcpyAsync(static_cast<uint8_t*>(tab.out) + s.u0 * tb, d_tab + s.u0 * tb, s.units * tb,
                                                 cudaMemcpyDeviceToHost, ctx->s_out));
            }
            ctx->h_slice_total[i] = base;                                 // reuse as "base of slice i"
            base += total;
        }
        RB_CUDA(ctx, cudaEventRecord(ctx->ev_out, ctx->s_out));
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_out, 0));
        r = rb200_sync(ctx);
        if (r != RB200_OK) return r;
        if (overflow) return RB200_E_SPACE;
        for (size_t i = 0; i < n_slices; i++) {                           // rebase the directory into the caller's array
            const uint64_t add = ctx->h_slice_total[i];
            const uint64_t* src = ctx->h_dir + sl[i].c0 + i;
            uint64_t* dst = offsets + sl[i].c0;
            for (size_t c = 0; c < sl[i].cnt; c++) dst[c] = src[c] + add;
        }
        offsets[n_chunks] = base;
        if (blob_size) *blob_size = base;
        return RB200_OK;
    });
}

// blob -> host buffers, overlapped the same way; no host synchronisation until the end because the
// directory (and therefore every slice's byte range) is already on the host.
// `decode_slice(slice, d_blob, d_offsets, d_table, d_out)` enqueues one slice's decode on ctx->stream; d_offsets points
// at the slice's first directory entry.
template <class DecodeSlice, class Hook = NoSliceHook>
int decode_pipeline(rb200_ctx* ctx, const uint8_t* blob, size_t blob_size, const uint64_t* offsets, uint32_t chunk_syms,
                    uint32_t unit_chunks, UnitTable tab, DecodeSlice decode_slice, uint8_t* out, size_t n, Hook hook = Hook{})
{
    if (n == 0) return RB200_OK;
    const uint32_t unit_syms = chunk_syms * unit_chunks;
    const size_t n_units = rb200_chunk_count(n, unit_syms), n_chunks = n_units * unit_chunks;
    if (offsets[n_chunks] != blob_size) return RB200_E_STREAM;
    Slice sl[rb200_ctx::kMaxSlices];
    const size_t n_slices = plan_slices(n, unit_syms, unit_chunks, sl);
    int rc = reserve(ctx, ctx->st_blob, blob_size + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_offsets, (n_chunks + 1) * sizeof(uint64_t));
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_out, n + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->st_aux, n_units * tab.unit_bytes);
    if (rc == RB200_OK) rc = reserve_dir(ctx, n_chunks + 1);
    if (rc != RB200_OK) return rc;
    for (size_t c = 0; c < n_chunks; c++) {                          // the copies below trust these
        if (offsets[c] > offsets[c + 1] || offsets[c + 1] > blob_size) return RB200_E_STREAM;
        ctx->h_dir[c] = offsets[c];
    }
    ctx->h_dir[n_chunks] = offsets[n_chunks];
    uint8_t* d_blob = static_cast<uint8_t*>(ctx->st_blob.p);
    uint64_t* d_off = static_cast<uint64_t*>(ctx->st_offsets.p);
    uint8_t* d_out = static_cast<uint8_t*>(ctx->st_out.p);
    uint8_t* d_tab = static_cast<uint8_t*>(ctx->st_aux.p);
    const size_t tb = tab.unit_bytes;

    return run_pipeline(ctx, [&]() -> int {
        RB_CUDA(ctx, cudaEventRecord(ctx->ev_start, ctx->stream));
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_in, ctx->ev_start, 0));
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_out, ctx->ev_start, 0));
        RB_CUDA(ctx, cudaMemcpyAsync(d_off, ctx->h_dir, (n_chunks + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->s_in));
        for (size_t i = 0; i < n_slices; i++) {
            const Slice& s = sl[i];
            // bytes of chunks [c0, c1): from the (aligned) end of chunk c0-1 to the end of chunk c1-1
            const size_t b0 = s.c0 ? static_cast<size_t>(offsets[s.c0] & ~15ull) : 0;
            const size_t b1 = static_cast<size_t>(offsets[s.c0 + s.cnt] & ~15ull);
            if (b1 > b0) RB_CUDA(ctx, cudaMemcpyAsync(d_blob + b0, blob + b0, b1 - b0, cudaMemcpyHostToDevice, ctx->s_in));
            if (tab.in)
                RB_CUDA(ctx, cudaMemcpyAsync(d_tab + s.u0 * tb, static_cast<const uint8_t*>(tab.in) + s.u0 * tb, s.units * tb,
                                             cudaMemcpyHostToDevice, ctx->s_in));
            RB_CUDA(ctx, cudaEventRecord(ctx->ev_in[i], ctx->s_in));
            RB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[i], 0));
            int r = hook(i, d_blob + b0, b1 - b0);
            if (r == RB200_OK) r = decode_slice(s, d_blob, d_off + s.c0, d_tab + s.u0 * tb, d_out + s.lo);
            if (r != RB200_OK) return r;
            RB_CUDA(ctx, cudaEventRecord(ctx->ev_done[i], ctx->stream));
            RB_CUDA(ctx, cudaStreamWaitEvent(ctx->s_out, ctx->ev_done[i], 0));
            RB_CUDA(ctx, cudaMemcpyAsync(out + s.lo, d_out + s.lo, s.len, cudaMemcpyDeviceToHost, ctx->s_out));
        }
        RB_CUDA(ctx, cudaEventRecord(ctx->ev_out, ctx->s_out));
        RB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_out, 0));
        return rb200_sync(ctx);
    });
}

// Entry checks shared by the encode / decode calls.  RB200_MEM_DEVICE runs `device` once the blob (16 bytes) and the
// directory (8 bytes) are aligned for the kernels; RB200_MEM_HOST runs `host`, a slice pipeline.
template <class Device, class Host>
int by_mem_kind(int mem_kind, const void* blob, const uint64_t* offsets, Device device, Host host)
{
    if (mem_kind == RB200_MEM_DEVICE) {
        if ((reinterpret_cast<uintptr_t>(blob) & 15) || (reinterpret_cast<uintptr_t>(offsets) & 7)) return RB200_E_ARG;
        return device();
    }
    if (mem_kind != RB200_MEM_HOST) return RB200_E_ARG;
    return host();
}

// container invariant: the blob ends on a 16-byte boundary; the decoders index it in 16-byte vectors with 32 bits
bool blob_size_ok(size_t blob_size) { return (blob_size & 15) == 0 && (blob_size >> 36) == 0; }

// the host-buffer form of rb200_encode / rb200_decode (one chunk per pipeline unit)
template <class Hook = NoSliceHook>
int encode_host(rb200_ctx* ctx, const rb200_model* model, const uint8_t* in, size_t n, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                uint64_t* offsets, size_t* blob_size, Hook hook = Hook{})
{
    return encode_pipeline(
        ctx, in, n, chunk_syms, 1, UnitTable{},
        [&](const Slice& s) {
            return plan_encode(ctx, model->coder, model->scale_bits, static_cast<uint32_t>(s.cnt), chunk_syms, word_ring_model(model->freqs));
        },
        [&](const Slice& s, const uint8_t* d_in, uint8_t*, uint8_t* d_blob, size_t cap, uint64_t* d_off) {
            return encode_device(ctx, model_tables(model), d_in, s.len, chunk_syms, d_blob, cap, d_off);
        },
        blob, blob_cap, offsets, blob_size, hook);
}

template <class Hook = NoSliceHook>
int decode_host(rb200_ctx* ctx, const rb200_model* model, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                uint32_t chunk_syms, uint8_t* out, size_t n, Hook hook = Hook{})
{
    return decode_pipeline(
        ctx, blob, blob_size, offsets, chunk_syms, 1, UnitTable{},
        [&](const Slice& s, const uint8_t* d_blob, const uint64_t* d_off, uint8_t*, uint8_t* d_out) {
            return decode_device(ctx, model, d_blob, blob_size, d_off, chunk_syms, d_out, s.len);
        },
        out, n, hook);
}

}  // namespace

extern "C" int rb200_encode(rb200_ctx* ctx, const rb200_model* model, const uint8_t* in, size_t n, uint32_t chunk_syms,
                            uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    if (!ctx || !model || model->ctx != ctx || !blob || !offsets || (!in && n) || !chunk_ok(chunk_syms)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return by_mem_kind(
        mem_kind, blob, offsets, [&] { return encode_device(ctx, model_tables(model), in, n, chunk_syms, blob, blob_cap, offsets); },
        [&] { return encode_host(ctx, model, in, n, chunk_syms, blob, blob_cap, offsets, blob_size); });
}

extern "C" int rb200_decode(rb200_ctx* ctx, const rb200_model* model, const uint8_t* blob, size_t blob_size,
                            const uint64_t* offsets, uint32_t chunk_syms, uint8_t* out, size_t n, int mem_kind)
{
    if (!ctx || !model || model->ctx != ctx || !offsets || (!out && n) || (!blob && blob_size) || !chunk_ok(chunk_syms))
        return RB200_E_ARG;
    if (!blob_size_ok(blob_size)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return by_mem_kind(
        mem_kind, blob, offsets, [&] { return decode_device(ctx, model, blob, blob_size, offsets, chunk_syms, out, n); },
        [&] { return decode_host(ctx, model, blob, blob_size, offsets, chunk_syms, out, n); });
}

// ---------------------------------------------------------------------------
// histogram + per-block models: block_kernels.cuh
// ---------------------------------------------------------------------------

extern "C" int rb200_histogram(rb200_ctx* ctx, const uint8_t* in, size_t n, uint64_t counts[256], int mem_kind)
{
    if (!ctx || !counts || (!in && n)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    int rc = reserve(ctx, ctx->st_aux, 256 * sizeof(unsigned long long));
    if (rc != RB200_OK) return rc;
    const uint8_t* d_in = in;
    if (mem_kind == RB200_MEM_HOST) {
        rc = reserve(ctx, ctx->st_in, n + 16);
        if (rc != RB200_OK) return rc;
        if (n) RB_CUDA(ctx, cudaMemcpyAsync(ctx->st_in.p, in, n, cudaMemcpyHostToDevice, ctx->stream));
        d_in = static_cast<const uint8_t*>(ctx->st_in.p);
    } else if (mem_kind != RB200_MEM_DEVICE) {
        return RB200_E_ARG;
    }
    unsigned long long* d_counts = static_cast<unsigned long long*>(ctx->st_aux.p);
    RB_CUDA(ctx, cudaMemsetAsync(d_counts, 0, 256 * sizeof(unsigned long long), ctx->stream));
    if (n) {
        launch_histogram(ctx->stream, static_cast<uint32_t>(ctx->sms), d_in, n, d_counts);
        rc = check_launch(ctx, "histogram_kernel");
        if (rc != RB200_OK) return rc;
    }
    RB_CUDA(ctx, cudaMemcpyAsync(counts, d_counts, 256 * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RB200_OK;
}

extern "C" int rb200_model_from_data(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* data, size_t n, int mem_kind,
                                     uint32_t freqs_out[256], rb200_model** out)
{
    if (!ctx || !out || (!data && n) || scale_bits < 8 || scale_bits > 16) return RB200_E_ARG;
    if (n >> 32) return RB200_E_ARG;                 // the reference counts in 32 bits (main.cpp:52)
    if (n == 0) return RB200_E_MODEL;                // normalize_freqs divides by the total
    uint64_t counts[256];
    int rc = rb200_histogram(ctx, data, n, counts, mem_kind);
    if (rc != RB200_OK) return rc;
    uint32_t freqs[256], cum[257];
    for (int s = 0; s < 256; s++) freqs[s] = static_cast<uint32_t>(counts[s]);
    rc = rb200_normalize_freqs(freqs, cum, 1u << scale_bits);
    if (rc != RB200_OK) return rc;
    rc = rb200_model_create(ctx, coder, scale_bits, freqs, out);
    if (rc == RB200_OK && freqs_out) std::memcpy(freqs_out, freqs, sizeof freqs);
    return rc;
}

extern "C" int rb200_blocks_build_models(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                         uint16_t* block_freqs, int mem_kind)
{
    if (!ctx || !in || !block_freqs || !n_blocks || !block_size) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    const size_t n = static_cast<size_t>(n_blocks) * block_size;
    const size_t fbytes = static_cast<size_t>(n_blocks) * 256 * sizeof(uint16_t);
    const uint8_t* d_in = in;
    uint16_t* d_freqs = block_freqs;
    int rc;
    if (mem_kind == RB200_MEM_HOST) {
        rc = reserve(ctx, ctx->st_in, n + 16);
        if (rc == RB200_OK) rc = reserve(ctx, ctx->st_aux, fbytes);
        if (rc != RB200_OK) return rc;
        RB_CUDA(ctx, cudaMemcpyAsync(ctx->st_in.p, in, n, cudaMemcpyHostToDevice, ctx->stream));
        d_in = static_cast<const uint8_t*>(ctx->st_in.p);
        d_freqs = static_cast<uint16_t*>(ctx->st_aux.p);
    } else if (mem_kind != RB200_MEM_DEVICE) {
        return RB200_E_ARG;
    }
    launch_block_models(ctx->stream, d_in, n_blocks, block_size, d_freqs, ctx->d_status);
    rc = check_launch(ctx, "block_model_kernel");
    if (rc != RB200_OK) return rc;
    if (mem_kind == RB200_MEM_HOST) {
        RB_CUDA(ctx, cudaMemcpyAsync(block_freqs, d_freqs, fbytes, cudaMemcpyDeviceToHost, ctx->stream));
        return rb200_sync(ctx);
    }
    return RB200_OK;
}

namespace {

constexpr size_t kBlockFreqBytes = 256 * sizeof(uint16_t);     // one block's frequency table

// The plan of a per-block encode over n_blocks blocks (n_blocks x block_size / chunk_syms < 2^31 chunks).  The word
// coder: the fused kernel (CTA 0 the scanner, then as many worker CTAs as are resident at once, at most one per block
// and as many as kBlockFusedScratchMax holds)
// whenever it builds the models, or the split sequence (one CTA per block) when use_fused_encode says so.  The byte and
// rans64 and alias coders: the split sequence (block_coder_encode_kernel), in slots of the same worst case as
// plan_encode's.
// K5f holds kBlockFusedSlots worst-case slots (2 x chunk_syms + 512 bytes) per warp of every CTA: about 4x a block's
// bytes per CTA.  The flat path leaves the fused kernel above 64 Ki symbols per chunk (use_fused_encode), but K5f is
// the only per-block path that builds models, so it takes any chunk; its worker CTAs are capped instead, so that the
// scratch stays within kBlockFusedScratchMax (one worker at least).  Up to 64 Ki symbols per chunk the cap binds only
// at 32 chunks of 64 Ki per block, by a few of ~260 CTAs on an H100; without it, 64 blocks of 2^24 symbols would take
// 65 x 256 MiB of scratch where the split path takes 2 GiB.
constexpr uint64_t kBlockFusedScratchMax = 2ull << 30;

EncodePlan plan_blocks_encode(const rb200_ctx* ctx, int coder, uint32_t sb, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                              bool build)
{
    EncodePlan p = {};
    p.n_chunks = n_blocks * (block_size / chunk_syms);
    p.slot_bytes = slot_bytes_for(chunk_syms);
    p.fused = coder == RB200_CODER_WORD && (build || use_fused_encode(chunk_syms));
    p.threads = block_threads(block_size, chunk_syms);
    p.smem = block_coder_encode_smem(static_cast<uint32_t>(coder), sb, p.threads);
    if (!p.fused) {
        p.grid = n_blocks;
        p.slots = p.n_chunks;
        return p;
    }
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, block_encode_fused_for(build, false, false, p.threads), static_cast<int>(p.threads), p.smem);
    const uint64_t cta_scratch = static_cast<uint64_t>(p.threads / 32) * kBlockFusedSlots * p.slot_bytes;
    const uint64_t fit = kBlockFusedScratchMax / cta_scratch;                                  // CTAs, the scanner's included
    const uint64_t workers = std::min<uint64_t>(static_cast<uint64_t>(ctx->sms) * std::max(per_sm, 1) - 1,   // the scanner CTA takes one slot
                                                std::max<uint64_t>(fit, 2) - 1);
    p.grid = static_cast<uint32_t>(std::max<uint64_t>(std::min<uint64_t>(workers, n_blocks), 1) + 1);
    p.slots = static_cast<size_t>(p.grid) * (p.threads / 32) * kBlockFusedSlots;
    return p;
}

// Per-block encode.  The word coder (scale_bits 12), default: ONE persistent launch (block_encode_fused_kernel: [model,]
// tables, encode, directory, placement); build_models makes the kernel run count_freqs + normalize_freqs per block first
// and write d_freqs.  RB200_ENCODE_PATH=split keeps the round-1 sequence (encode into per-chunk slots, tile scan,
// compaction), which the byte, rans64 and alias coders always run (block_coder_encode_kernel, models of 1 << sb).
// choice set (with build_models; an auto encode's launch group): the GATED instances of the encoder, the scan, prefix
// and compaction, which run only when the record names `group`; sb is then the largest scale_bits of the group.  geom
// set as well (the device-count encode): n_blocks is the bound n_blocks_max, which fixes the plan and every launch
// shape, the GEOM instances take the count, the directory's and the blob's places from the record, and d_blob is the
// container, of capacity blob_cap.
int blocks_encode_device(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* d_in, uint32_t n_blocks, uint32_t block_size,
                         uint16_t* d_freqs, bool build_models, uint32_t chunk_syms, uint8_t* d_blob, size_t blob_cap, uint64_t* d_offsets,
                         const CoderChoice* choice = nullptr, uint32_t group = 0, const BlocksVarlenGeom* geom = nullptr)
{
    if (static_cast<uint64_t>(n_blocks) * (block_size / chunk_syms) >= (1ull << 31)) return RB200_E_ARG;
    const EncodePlan p = plan_blocks_encode(ctx, coder, sb, n_blocks, block_size, chunk_syms, build_models);
    // the word coder's model-building encodes run K5f: its split GATED and GEOM instances serve the stored encodes only
    if (!p.fused && coder == RB200_CODER_WORD && (build_models || choice || geom)) return RB200_E_ARG;
    return run_encode(ctx, p, d_blob, blob_cap, d_offsets, geom ? &geom->v : nullptr, [&](const EncodeWorkspace& ws) {
        if (p.fused) {
            block_encode_fused_for(build_models, choice != nullptr, geom != nullptr, p.threads)<<<p.grid, p.threads, p.smem, ctx->stream>>>(
                d_in, n_blocks, block_size, d_freqs, chunk_syms, ws.scratch, p.slot_bytes, ws.look, ws.counter, d_blob, blob_cap, d_offsets,
                ctx->d_status, choice, group, geom, block_size / chunk_syms);
            return check_launch(ctx, "block_encode_fused_kernel");
        }
        launch_block_encode(ctx->stream, static_cast<uint32_t>(coder), sb, build_models, p.grid, p.threads, p.smem, d_in, block_size, d_freqs,
                            chunk_syms, ws.scratch, p.slot_bytes, ws.sizes, ctx->d_status, choice, group, geom);
        return check_launch(ctx, "block_coder_encode_kernel");
    }, choice, group);
}

// Host mode runs the slice pipeline over whole blocks; the frequency tables go in with each slice when the caller supplies
// them, and come back with it when the kernel builds them.  `hook` as in encode_pipeline.
template <class Hook = NoSliceHook>
int blocks_encode_host(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                       uint16_t* block_freqs, bool build, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap, uint64_t* offsets,
                       size_t* blob_size, Hook hook = Hook{})
{
    const UnitTable freqs = build ? UnitTable{nullptr, block_freqs, kBlockFreqBytes} : UnitTable{block_freqs, nullptr, kBlockFreqBytes};
    return encode_pipeline(
        ctx, in, static_cast<size_t>(n_blocks) * block_size, chunk_syms, block_size / chunk_syms, freqs,
        [&](const Slice& s) { return plan_blocks_encode(ctx, coder, sb, static_cast<uint32_t>(s.units), block_size, chunk_syms, build); },
        [&](const Slice& s, const uint8_t* d_in, uint8_t* d_freqs, uint8_t* d_blob, size_t cap, uint64_t* d_off) {
            return blocks_encode_device(ctx, coder, sb, d_in, static_cast<uint32_t>(s.units), block_size, reinterpret_cast<uint16_t*>(d_freqs),
                                        build, chunk_syms, d_blob, cap, d_off);
        },
        blob, blob_cap, offsets, blob_size, hook);
}

int blocks_encode_entry(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                        uint16_t* block_freqs, bool build, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap, uint64_t* offsets,
                        size_t* blob_size, int mem_kind)
{
    if (!ctx || !in || !block_freqs || !blob || !offsets || !container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return by_mem_kind(
        mem_kind, blob, offsets,
        [&] { return blocks_encode_device(ctx, coder, sb, in, n_blocks, block_size, block_freqs, build, chunk_syms, blob, blob_cap, offsets); },
        [&] {
            return blocks_encode_host(ctx, coder, sb, in, n_blocks, block_size, block_freqs, build, chunk_syms, blob, blob_cap, offsets,
                                      blob_size);
        });
}

int blocks_decode_device(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* d_blob, size_t blob_size, const uint64_t* d_off,
                         const uint16_t* d_freqs, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, uint8_t* d_out)
{
    launch_block_decode(ctx->stream, static_cast<uint32_t>(coder), sb, d_blob, blob_size, d_off, d_freqs, n_blocks, block_size, chunk_syms,
                        d_out, ctx->d_status);
    return check_launch(ctx, "block_decode_kernel");
}

// the host-buffer form of rb200_blocks_decode: the slice pipeline over whole blocks, each slice's tables copied in with it
template <class Hook = NoSliceHook>
int blocks_decode_host(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                       const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, uint8_t* out,
                       Hook hook = Hook{})
{
    return decode_pipeline(
        ctx, blob, blob_size, offsets, chunk_syms, block_size / chunk_syms, UnitTable{block_freqs, nullptr, kBlockFreqBytes},
        [&](const Slice& s, const uint8_t* d_blob, const uint64_t* d_off, uint8_t* d_freqs, uint8_t* d_out) {
            return blocks_decode_device(ctx, coder, sb, d_blob, blob_size, d_off, reinterpret_cast<const uint16_t*>(d_freqs),
                                        static_cast<uint32_t>(s.units), block_size, chunk_syms, d_out);
        },
        out, static_cast<size_t>(n_blocks) * block_size, hook);
}

int blocks_decode_entry(rb200_ctx* ctx, int coder, uint32_t sb, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                        const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, uint8_t* out, int mem_kind)
{
    if (!ctx || !blob || !offsets || !block_freqs || !out || !container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    if (!blob_size_ok(blob_size)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    const uint32_t per_block = block_size / chunk_syms;
    if (static_cast<uint64_t>(n_blocks) * per_block >= (1ull << 31)) return RB200_E_ARG;
    return by_mem_kind(
        mem_kind, blob, offsets,
        [&] { return blocks_decode_device(ctx, coder, sb, blob, blob_size, offsets, block_freqs, n_blocks, block_size, chunk_syms, out); },
        [&] { return blocks_decode_host(ctx, coder, sb, blob, blob_size, offsets, block_freqs, n_blocks, block_size, chunk_syms, out); });
}

// The byte / rans64 (version 3) and alias (version 4) per-block calls' own checks before the shared entries: the coder
// and scale_bits of `version`, fewer than 2^31 chunks (RB200_E_ARG, nothing launched); a HOST-mode caller table that
// does not sum to 1 << sb (RB200_E_MODEL).
int blocks_coder_args(uint16_t version, int coder, uint32_t sb, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                      const uint16_t* caller_freqs, int mem_kind)
{
    if (coder < 0 || !container_blocks_coder_ok(version, static_cast<uint32_t>(coder), sb)) return RB200_E_ARG;
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    if (static_cast<uint64_t>(n_blocks) * (block_size / chunk_syms) >= (1ull << 31)) return RB200_E_ARG;
    if (caller_freqs && mem_kind == RB200_MEM_HOST && !container_block_models_sum_to(caller_freqs, n_blocks, 1u << sb)) return RB200_E_MODEL;
    return RB200_OK;
}

}  // namespace

extern "C" int rb200_blocks_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                   const uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                                   uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    return blocks_encode_entry(ctx, RB200_CODER_WORD, 12, in, n_blocks, block_size, const_cast<uint16_t*>(block_freqs), false, chunk_syms,
                               blob, blob_cap, offsets, blob_size, mem_kind);
}

extern "C" int rb200_blocks_model_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                         uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                                         uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    return blocks_encode_entry(ctx, RB200_CODER_WORD, 12, in, n_blocks, block_size, block_freqs, true, chunk_syms, blob, blob_cap, offsets,
                               blob_size, mem_kind);
}

extern "C" int rb200_blocks_decode(rb200_ctx* ctx, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                                   const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                   uint8_t* out, int mem_kind)
{
    return blocks_decode_entry(ctx, RB200_CODER_WORD, 12, blob, blob_size, offsets, block_freqs, n_blocks, block_size, chunk_syms, out,
                               mem_kind);
}

extern "C" int rb200_blocks_coder_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                         uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob,
                                         size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    if (!block_freqs) return RB200_E_ARG;
    const int rc = blocks_coder_args(kContainerVersionBlocksCoder, coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs, mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_encode_entry(ctx, coder, scale_bits, in, n_blocks, block_size, const_cast<uint16_t*>(block_freqs), false, chunk_syms,
                               blob, blob_cap, offsets, blob_size, mem_kind);
}

extern "C" int rb200_blocks_coder_model_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                               uint32_t block_size, uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob,
                                               size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    const int rc = blocks_coder_args(kContainerVersionBlocksCoder, coder, scale_bits, n_blocks, block_size, chunk_syms, nullptr, mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_encode_entry(ctx, coder, scale_bits, in, n_blocks, block_size, block_freqs, true, chunk_syms, blob, blob_cap, offsets,
                               blob_size, mem_kind);
}

extern "C" int rb200_blocks_coder_decode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* blob, size_t blob_size,
                                         const uint64_t* offsets, const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size,
                                         uint32_t chunk_syms, uint8_t* out, int mem_kind)
{
    const int rc = blocks_coder_args(kContainerVersionBlocksCoder, coder, scale_bits, n_blocks, block_size, chunk_syms, nullptr, mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_decode_entry(ctx, coder, scale_bits, blob, blob_size, offsets, block_freqs, n_blocks, block_size, chunk_syms, out, mem_kind);
}

extern "C" int rb200_blocks_alias_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                         const uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                                         uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    if (!block_freqs) return RB200_E_ARG;
    const int rc = blocks_coder_args(kContainerVersionBlocksAlias, RB200_CODER_ALIAS, scale_bits, n_blocks, block_size, chunk_syms,
                                     block_freqs, mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_encode_entry(ctx, RB200_CODER_ALIAS, scale_bits, in, n_blocks, block_size, const_cast<uint16_t*>(block_freqs), false,
                               chunk_syms, blob, blob_cap, offsets, blob_size, mem_kind);
}

extern "C" int rb200_blocks_alias_model_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                               uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                                               uint64_t* offsets, size_t* blob_size, int mem_kind)
{
    const int rc = blocks_coder_args(kContainerVersionBlocksAlias, RB200_CODER_ALIAS, scale_bits, n_blocks, block_size, chunk_syms, nullptr,
                                     mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_encode_entry(ctx, RB200_CODER_ALIAS, scale_bits, in, n_blocks, block_size, block_freqs, true, chunk_syms, blob, blob_cap,
                               offsets, blob_size, mem_kind);
}

extern "C" int rb200_blocks_alias_decode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* blob, size_t blob_size,
                                         const uint64_t* offsets, const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size,
                                         uint32_t chunk_syms, uint8_t* out, int mem_kind)
{
    const int rc = blocks_coder_args(kContainerVersionBlocksAlias, RB200_CODER_ALIAS, scale_bits, n_blocks, block_size, chunk_syms, nullptr,
                                     mem_kind);
    if (rc != RB200_OK) return rc;
    return blocks_decode_entry(ctx, RB200_CODER_ALIAS, scale_bits, blob, blob_size, offsets, block_freqs, n_blocks, block_size, chunk_syms,
                               out, mem_kind);
}

// ---------------------------------------------------------------------------
// CRC-32 and the container in host or device memory: crc_kernels.cuh, container_host.cpp
// ---------------------------------------------------------------------------

namespace {

// zlib crc32 of d[0, n) into `slot`, on ctx->stream; with n_dev set the length is min(*n_dev, n); with off_dev set the
// bytes start *off_dev bytes after d (crc32_kernel)
int launch_crc(rb200_ctx* ctx, const uint8_t* d, uint64_t n, const uint64_t* n_dev, uint32_t crc_in, CrcSlot* slot,
               const uint64_t* off_dev = nullptr)
{
    const uint32_t sms = static_cast<uint32_t>(ctx->sms);
    crc32_kernel<<<n_dev ? sms : crc32_grid(sms, n), kCrcThreads, kCrcSmemBytes, ctx->stream>>>(d, n, n_dev, off_dev, crc_in,
                                                                                                ctx->d_crc_work, slot);
    return check_launch(ctx, "crc32_kernel");
}

// brings slots [0, count) to ctx->h_crc and waits for them
int fetch_crc(rb200_ctx* ctx, size_t count)
{
    if (!count) return RB200_OK;
    RB_CUDA(ctx, cudaMemcpyAsync(ctx->h_crc, ctx->d_crc, count * sizeof(CrcSlot), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RB200_OK;
}

// the CRC of the whole blob from the per-slice CRCs a host pipeline left in slots [0, count), joined in slice order
int joined_slice_crc(rb200_ctx* ctx, size_t count, uint32_t* crc)
{
    const int rc = fetch_crc(ctx, count);
    if (rc != RB200_OK) return rc;
    uint32_t c = 0;
    for (size_t i = 0; i < count; i++) c = crc32_combine(c, ctx->h_crc[i].crc, ctx->h_crc[i].len);
    *crc = c;
    return RB200_OK;
}

// The per-slice hook of the container calls: CRC each slice's blob bytes into slot i when `on`.  Counts the slices.
struct SliceCrc {
    rb200_ctx* ctx;
    bool on;
    size_t* slices;
    int operator()(size_t i, const uint8_t* d, const uint64_t* d_len, size_t cap) const
    {
        *slices = i + 1;
        return on ? launch_crc(ctx, d, cap, d_len, 0, ctx->d_crc + i) : RB200_OK;
    }
    int operator()(size_t i, const uint8_t* d, size_t len) const
    {
        *slices = i + 1;
        return on ? launch_crc(ctx, d, len, nullptr, 0, ctx->d_crc + i) : RB200_OK;
    }
};

// rb200_container_decode / rb200_container_blocks_decode / rb200_container_blocks_coder_decode once the buffers are
// checked: header, model and directory validated by the shared parser for `version`, then the blob CRC, then the decode
// (a model and rb200_decode's kernels for version 1, the per-block decoder of the header's coder reading its tables in
// place for versions 2 and 3).  DEVICE: the prefix is read through pinned memory, both CRCs are taken on the GPU, and
// nothing is decoded unless every check passes.
int container_decode_impl(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap, uint64_t* n_symbols,
                          bool device, uint16_t version)
{
    ContainerHeader h;
    const uint8_t* prefix = buf;
    int rc;
    if (device) {
        if (size < sizeof(ContainerHeader)) return RB200_E_STREAM;
        rc = reserve_dir(ctx, sizeof(ContainerHeader) / sizeof(uint64_t));
        if (rc != RB200_OK) return rc;
        RB_CUDA(ctx, cudaMemcpyAsync(ctx->h_dir, buf, sizeof(ContainerHeader), cudaMemcpyDeviceToHost, ctx->stream));
        RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        rc = container_parse_header(reinterpret_cast<const uint8_t*>(ctx->h_dir), size, version, &h);
        if (rc != RB200_OK) return rc;
        const size_t boff = container_blob_offset(h);
        rc = reserve_dir(ctx, boff / sizeof(uint64_t));
        if (rc != RB200_OK) return rc;
        const uint64_t covered = container_dir_end(h) - sizeof(ContainerHeader);     // model and directory: what the CRC covers after the header
        RB_CUDA(ctx, cudaMemcpyAsync(ctx->h_dir, buf, boff, cudaMemcpyDeviceToHost, ctx->stream));
        rc = launch_crc(ctx, buf + sizeof(ContainerHeader), covered, nullptr, 0, ctx->d_crc);
        if (rc == RB200_OK) rc = fetch_crc(ctx, 1);
        if (rc != RB200_OK) return rc;
        prefix = reinterpret_cast<const uint8_t*>(ctx->h_dir);
        rc = container_check_prefix(h, prefix, crc32_combine(container_header_crc(h), ctx->h_crc[0].crc, covered));
    } else {
        rc = container_parse_header(buf, size, version, &h);
        if (rc == RB200_OK)
            rc = container_check_prefix(h, buf, container_meta_crc(h, buf + sizeof(ContainerHeader),
                                                                   reinterpret_cast<const uint64_t*>(buf + container_dir_offset(h))));
    }
    if (rc != RB200_OK) return rc;
    if (n_symbols) *n_symbols = h.n_symbols;
    if (out_cap < h.n_symbols) return RB200_E_SPACE;
    if (h.n_symbols && !out) return RB200_E_ARG;
    if (!container_geometry_decodable(h.chunk_syms, h.blob_bytes)) return RB200_E_ARG;  // what rb200_decode accepts
    const uint8_t* blob = buf + container_blob_offset(h);
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + container_dir_offset(h));
    const bool blob_crc = (h.flags & RB200_CONTAINER_CRC_BLOB) != 0;
    if (device && blob_crc) {
        rc = launch_crc(ctx, blob, h.blob_bytes, nullptr, 0, ctx->d_crc);
        if (rc == RB200_OK) rc = fetch_crc(ctx, 1);
        if (rc == RB200_OK) rc = container_check_blob(h, ctx->h_crc[0].crc);
        if (rc != RB200_OK) return rc;
    }
    // the decode: DEVICE enqueues it and synchronises; HOST runs a slice pipeline that CRCs each slice's blob bytes
    auto decode = [&](auto on_device, auto on_host) -> int {
        if (device) {
            const int r = on_device();
            const int st = rb200_sync(ctx);
            return r == RB200_OK ? st : r;
        }
        size_t slices = 0;
        int r = on_host(SliceCrc{ctx, blob_crc, &slices});
        uint32_t crc = 0;
        if (r == RB200_OK && blob_crc) r = joined_slice_crc(ctx, slices, &crc);
        if (r == RB200_OK) r = container_check_blob(h, crc);
        return r;
    };
    if (version != kContainerVersion) {       // per-block models: word at 12 (version 2), byte / rans64 (3), alias (4)
        const uint16_t* block_freqs = reinterpret_cast<const uint16_t*>(buf + sizeof(ContainerHeader));     // read in place
        return decode(
            [&] {
                return blocks_decode_device(ctx, h.coder, h.scale_bits, blob, h.blob_bytes, offsets, block_freqs, h.n_blocks, h.block_size,
                                            h.chunk_syms, out);
            },
            [&](SliceCrc hook) {
                return blocks_decode_host(ctx, h.coder, h.scale_bits, blob, h.blob_bytes, offsets, block_freqs, h.n_blocks, h.block_size,
                                          h.chunk_syms, out, hook);
            });
    }
    const uint32_t* freqs = reinterpret_cast<const uint32_t*>(prefix + sizeof(ContainerHeader));
    if (!container_model_decodable(h.coder, freqs)) return RB200_E_MODEL;                 // what rb200_model_create accepts
    rb200_model* model = nullptr;
    rc = rb200_model_create(ctx, h.coder, h.scale_bits, freqs, &model);
    if (rc != RB200_OK) return rc;
    rc = decode([&] { return decode_device(ctx, model, blob, h.blob_bytes, offsets, h.chunk_syms, out, h.n_symbols); },
                [&](SliceCrc hook) { return decode_host(ctx, model, blob, h.blob_bytes, offsets, h.chunk_syms, out, h.n_symbols, hook); });
    rb200_model_destroy(model);
    return rc;
}

// Alignment of a container call's buffers: 16 bytes in DEVICE mode (the kernels' vector loads), 8 in HOST mode.
bool container_mem_ok(int mem_kind, const void* a, const void* b)
{
    if (mem_kind != RB200_MEM_HOST && mem_kind != RB200_MEM_DEVICE) return false;
    const uintptr_t align = mem_kind == RB200_MEM_DEVICE ? 15 : 7;
    return !(reinterpret_cast<uintptr_t>(a) & align) && !(reinterpret_cast<uintptr_t>(b) & align);
}

}  // namespace

extern "C" int rb200_crc32(rb200_ctx* ctx, const uint8_t* data, size_t n, uint32_t crc_in, uint32_t* crc_out, int mem_kind)
{
    if (!ctx || !crc_out || (!data && n) || (mem_kind != RB200_MEM_HOST && mem_kind != RB200_MEM_DEVICE)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    const uint8_t* d = data;
    if (mem_kind == RB200_MEM_HOST) {
        const int rc = reserve(ctx, ctx->st_in, n + 16);
        if (rc != RB200_OK) return rc;
        if (n) RB_CUDA(ctx, cudaMemcpyAsync(ctx->st_in.p, data, n, cudaMemcpyHostToDevice, ctx->stream));
        d = static_cast<const uint8_t*>(ctx->st_in.p);
    }
    int rc = launch_crc(ctx, d, n, nullptr, crc_in, ctx->d_crc);
    if (rc == RB200_OK) rc = fetch_crc(ctx, 1);
    if (rc == RB200_OK) *crc_out = ctx->h_crc[0].crc;
    return rc;
}

extern "C" int rb200_container_encode(rb200_ctx* ctx, const rb200_model* model, const uint8_t* in, size_t n, uint32_t chunk_syms,
                                      uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind)
{
    if (!ctx || !model || model->ctx != ctx || !out || (!in && n) || !chunk_ok(chunk_syms)) return RB200_E_ARG;
    if (!container_mem_ok(mem_kind, out, nullptr)) return RB200_E_ARG;
    const bool device = mem_kind == RB200_MEM_DEVICE;
    if (!container_model_ok(static_cast<uint32_t>(model->coder), model->scale_bits, model->freqs)) return RB200_E_MODEL;
    const size_t n_chunks = rb200_chunk_count(n, chunk_syms);
    if (n_chunks >= (1ull << 31)) return RB200_E_ARG;
    ContainerHeader h = container_header(model->coder, model->scale_bits, chunk_syms, n, n_chunks, 0, flags);
    const size_t dir_off = container_dir_offset(h), dir_end = container_dir_end(h), boff = container_blob_offset(h);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    const bool blob_crc = (h.flags & RB200_CONTAINER_CRC_BLOB) != 0;
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + dir_off);
    if (device) {            // asynchronous: directory CRC, blob CRC, then the header from blob_bytes = dir[n_chunks]
        int rc = encode_device(ctx, model_tables(model), in, n, chunk_syms, out + boff, out_cap - boff, dir);
        if (rc == RB200_OK) rc = launch_crc(ctx, out + dir_off, dir_end - dir_off, nullptr, 0, ctx->d_crc);
        if (rc == RB200_OK && blob_crc) rc = launch_crc(ctx, out + boff, out_cap - boff, dir + n_chunks, 0, ctx->d_crc + 1);
        if (rc != RB200_OK) return rc;
        container_finish_kernel<<<1, 32, 0, ctx->stream>>>(out, h, dir_off, boff, out_cap, model->d_freqs, ctx->d_crc, ctx->d_status, nullptr,
                                                           nullptr);
        return check_launch(ctx, "container_finish_kernel");
    }
    size_t blob_bytes = 0, slices = 0;
    int rc = encode_host(ctx, model, in, n, chunk_syms, out + boff, out_cap - boff, dir, &blob_bytes, SliceCrc{ctx, blob_crc, &slices});
    if (rc == RB200_OK && blob_crc) rc = joined_slice_crc(ctx, slices, &h.blob_crc);
    if (rc != RB200_OK) return rc;
    h.blob_bytes = blob_bytes;
    h.meta_crc = container_meta_crc(h, model->freqs, dir);
    std::memcpy(out, &h, sizeof h);
    std::memcpy(out + sizeof h, model->freqs, sizeof model->freqs);
    std::memset(out + dir_end, 0, boff - dir_end);
    if (out_size) *out_size = boff + blob_bytes;
    return RB200_OK;
}

extern "C" int rb200_container_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                      uint64_t* n_symbols, int mem_kind)
{
    if (!ctx || !buf || (!out && out_cap)) return RB200_E_ARG;
    if (!container_mem_ok(mem_kind, buf, out)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return container_decode_impl(ctx, buf, size, out, out_cap, n_symbols, mem_kind == RB200_MEM_DEVICE, kContainerVersion);
}

namespace {

// The launch groups of an auto encode, one per distinct encoder instance its candidates need: word (both GATED K2 or
// K2f instances), alias and byte per SB instance of RB200_ALIAS_SB_DISPATCH, rans64.  A group's scale_bits is the
// largest of its candidates': it sizes the alias encoder's shared memory (no other plan depends on it), and the GATED
// kernels take the chosen one from the record.
struct AutoPlan {
    CandidateList list;
    int coder[kMaxCandidates];
    uint32_t sb[kMaxCandidates];
    uint32_t n_groups;
};

AutoPlan plan_auto(const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm)
{
    AutoPlan a = {};
    uint32_t key[kMaxCandidates];
    a.list.n = n_candidates;
    a.list.tolerance_ppm = tolerance_ppm;
    for (uint32_t i = 0; i < n_candidates; i++) {
        const int coder = static_cast<int>(candidates[i] >> 8);
        const uint32_t sb = candidates[i] & 0xffu;
        const bool by_sb = (coder == RB200_CODER_ALIAS || coder == RB200_CODER_BYTE) && (sb == 16 || sb == 14 || sb == 12);
        const uint32_t k = static_cast<uint32_t>(coder) << 8 | (by_sb ? sb : 0u);
        uint32_t g = 0;
        while (g < a.n_groups && key[g] != k) g++;
        if (g == a.n_groups) {
            key[g] = k;
            a.coder[g] = coder;
            a.sb[g] = sb;
            a.n_groups++;
        }
        a.sb[g] = std::max(a.sb[g], sb);
        a.list.pair[i] = candidates[i];
        a.list.group[i] = g;
    }
    return a;
}

// the argument rules of every per-block container encode, with n_blocks the count (fixed calls) or its bound
// n_blocks_max (device-count call)
bool blocks_container_args_ok(const rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                              const uint8_t* out, int mem_kind)
{
    if (!ctx || !in || !out || !container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return false;
    if (!container_mem_ok(mem_kind, out, nullptr)) return false;
    return static_cast<uint64_t>(n_blocks) * (block_size / chunk_syms) < (1ull << 31);
}

// The per-block containers (version 2: the word coder at 12; version 3: byte / rans64; version 4: alias) in device
// memory, enqueue only: the block encoder writes every block's model (built, or the caller's tables copied in first),
// the directory and the blob straight into their place in `out`; then as rb200_container_encode, except that one CRC
// launch covers model and directory, which are contiguous, and the header kernel reads blob_bytes = dir[n_chunks].
// a set (the auto encode, with models built): the choice kernel (after a memset of its sums), one gated encode group per
// distinct encoder instance of the list, then the CRCs and the per-block header kernel, which writes the chosen
// version, coder and scale_bits; the layout of versions 2-4 is the same, so the host lays the container out without
// knowing the choice.  d_n_blocks set as well: h.n_blocks is the bound n_blocks_max, which sizes every launch; the plan
// kernel reads *d_n_blocks into the record at every run (for a list of one it also writes the choice record, and no
// choice kernel runs), and every later kernel is its GEOM instance.  Arguments are checked by the caller.
int blocks_container_encode(rb200_ctx* ctx, const ContainerHeader& h, const uint8_t* in, const uint16_t* caller_freqs,
                            const uint32_t* d_n_blocks, uint8_t* out, size_t out_cap, const AutoPlan* a = nullptr)
{
    const uint32_t n_blocks = h.n_blocks, block_size = h.block_size, chunk_syms = h.chunk_syms;
    const size_t dir_off = container_dir_offset(h), dir_end = container_dir_end(h), boff = container_blob_offset(h);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    cudaStream_t s = ctx->stream;
    BlocksChoice* r = ctx->d_blocks_choice;
    BlocksVarlenGeom* geom = d_n_blocks ? ctx->d_blocks_geom : nullptr;
    uint16_t* model = reinterpret_cast<uint16_t*>(out + sizeof(ContainerHeader));
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + dir_off);
    uint8_t* blob = geom ? out : out + boff;                 // GEOM: the container, in which the kernels place the blob
    const size_t blob_cap = geom ? out_cap : out_cap - boff;
    int rc = RB200_OK;
    if (caller_freqs) RB_CUDA(ctx, cudaMemcpyAsync(model, caller_freqs, dir_off - sizeof(ContainerHeader), cudaMemcpyDeviceToDevice, s));
    if (a) {
        for (uint32_t k = 0; k < a->n_groups && rc == RB200_OK; k++)    // every group's workspace before the first launch
            rc = reserve_plan(ctx, plan_blocks_encode(ctx, a->coder[k], a->sb[k], n_blocks, block_size, chunk_syms, true));
        if (rc != RB200_OK) return rc;
        const bool one = geom && a->list.n == 1;
        if (!one) RB_CUDA(ctx, cudaMemsetAsync(&r->done, 0, sizeof(BlocksChoice) - offsetof(BlocksChoice, done), s));
        if (geom) {
            blocks_varlen_plan_kernel<<<1, 32, 0, s>>>(d_n_blocks, n_blocks, block_size, chunk_syms, out_cap, one ? a->list.pair[0] : 0u, geom,
                                                       r, ctx->d_status);
            rc = check_launch(ctx, "blocks_varlen_plan_kernel");
        }
        if (rc == RB200_OK && !one) {
            auto choice = geom ? blocks_choice_kernel<true> : blocks_choice_kernel<false>;
            choice<<<n_blocks, kBlocksChoiceWarps * 32, 0, s>>>(a->list, in, block_size, chunk_syms, r, ctx->d_status, geom);
            rc = check_launch(ctx, "blocks_choice_kernel");
        }
        for (uint32_t k = 0; k < a->n_groups && rc == RB200_OK; k++)
            rc = blocks_encode_device(ctx, a->coder[k], a->sb[k], in, n_blocks, block_size, model, true, chunk_syms, blob, blob_cap, dir,
                                      &r->choice, k, geom);
    } else {
        rc = blocks_encode_device(ctx, h.coder, h.scale_bits, in, n_blocks, block_size, model, !caller_freqs, chunk_syms, blob, blob_cap, dir);
    }
    if (rc == RB200_OK)
        rc = launch_crc(ctx, out + sizeof(ContainerHeader), dir_end - sizeof(ContainerHeader), geom ? &geom->meta_len : nullptr, 0, ctx->d_crc);
    if (rc == RB200_OK && (h.flags & RB200_CONTAINER_CRC_BLOB)) {
        if (geom) {
            varlen_blob_len_kernel<<<1, 32, 0, s>>>(out, &geom->v);
            rc = check_launch(ctx, "varlen_blob_len_kernel");
            if (rc == RB200_OK) rc = launch_crc(ctx, out, out_cap, &geom->v.blob_len, 0, ctx->d_crc + 1, &geom->v.blob_off);
        } else {
            rc = launch_crc(ctx, out + boff, out_cap - boff, dir + h.n_chunks, 0, ctx->d_crc + 1);
        }
    }
    if (rc != RB200_OK) return rc;
    if (!a) {
        container_finish_kernel<<<1, 32, 0, s>>>(out, h, dir_off, boff, out_cap, nullptr, ctx->d_crc, ctx->d_status, nullptr, nullptr);
        return check_launch(ctx, "container_finish_kernel");
    }
    auto finish = geom ? container_blocks_finish_kernel<true> : container_blocks_finish_kernel<false>;
    finish<<<1, 32, 0, s>>>(out, h, dir_off, boff, out_cap, ctx->d_crc, ctx->d_status, r, geom);
    return check_launch(ctx, "container_blocks_finish_kernel");
}

// The fixed per-block container encodes: in device memory blocks_container_encode; in host memory the slice pipeline,
// then the CRCs and the header on the host.  Arguments are checked by the caller.
int container_blocks_encode_impl(rb200_ctx* ctx, ContainerHeader h, const uint8_t* in, const uint16_t* block_freqs, uint8_t* out,
                                 size_t out_cap, size_t* out_size, int mem_kind)
{
    if (mem_kind == RB200_MEM_DEVICE) return blocks_container_encode(ctx, h, in, block_freqs, nullptr, out, out_cap);
    const bool build = block_freqs == nullptr;
    const uint32_t n_blocks = h.n_blocks, block_size = h.block_size, chunk_syms = h.chunk_syms;
    if (!build && !container_block_models_sum_to(block_freqs, n_blocks, 1u << h.scale_bits)) return RB200_E_MODEL;
    const size_t dir_off = container_dir_offset(h), dir_end = container_dir_end(h), boff = container_blob_offset(h);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    const bool blob_crc = (h.flags & RB200_CONTAINER_CRC_BLOB) != 0;
    uint16_t* model = reinterpret_cast<uint16_t*>(out + sizeof(ContainerHeader));
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + dir_off);
    if (!build) std::memcpy(model, block_freqs, dir_off - sizeof(ContainerHeader));
    size_t blob_bytes = 0, slices = 0;
    int rc = blocks_encode_host(ctx, h.coder, h.scale_bits, in, n_blocks, block_size, model, build, chunk_syms, out + boff, out_cap - boff,
                                dir, &blob_bytes, SliceCrc{ctx, blob_crc, &slices});
    if (rc == RB200_OK && blob_crc) rc = joined_slice_crc(ctx, slices, &h.blob_crc);
    if (rc != RB200_OK) return rc;
    h.blob_bytes = blob_bytes;
    h.meta_crc = container_meta_crc(h, model, dir);
    std::memcpy(out, &h, sizeof h);
    std::memset(out + dir_end, 0, boff - dir_end);
    if (out_size) *out_size = boff + blob_bytes;
    return RB200_OK;
}

}  // namespace

extern "C" int rb200_container_blocks_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                             const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap,
                                             size_t* out_size, int mem_kind)
{
    if (!blocks_container_args_ok(ctx, in, n_blocks, block_size, chunk_syms, out, mem_kind)) return RB200_E_ARG;
    return container_blocks_encode_impl(ctx, container_blocks_header(n_blocks, block_size, chunk_syms, 0, flags), in, block_freqs, out,
                                        out_cap, out_size, mem_kind);
}

namespace {

// rb200_container_blocks_coder_encode (version 3) and rb200_container_blocks_alias_encode (version 4)
int container_blocks_coder_encode(rb200_ctx* ctx, uint16_t version, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                  uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags, uint8_t* out,
                                  size_t out_cap, size_t* out_size, int mem_kind)
{
    if (coder < 0 || !container_blocks_coder_ok(version, static_cast<uint32_t>(coder), scale_bits)) return RB200_E_ARG;
    if (!blocks_container_args_ok(ctx, in, n_blocks, block_size, chunk_syms, out, mem_kind)) return RB200_E_ARG;
    return container_blocks_encode_impl(
        ctx, container_blocks_coder_header(version, coder, scale_bits, n_blocks, block_size, chunk_syms, 0, flags), in, block_freqs, out,
        out_cap, out_size, mem_kind);
}

}  // namespace

extern "C" int rb200_container_blocks_coder_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                                   uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags,
                                                   uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind)
{
    return container_blocks_coder_encode(ctx, kContainerVersionBlocksCoder, coder, scale_bits, in, n_blocks, block_size, block_freqs,
                                         chunk_syms, flags, out, out_cap, out_size, mem_kind);
}

extern "C" int rb200_container_blocks_alias_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                                   uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags,
                                                   uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind)
{
    return container_blocks_coder_encode(ctx, kContainerVersionBlocksAlias, RB200_CODER_ALIAS, scale_bits, in, n_blocks, block_size,
                                         block_freqs, chunk_syms, flags, out, out_cap, out_size, mem_kind);
}

extern "C" int rb200_container_blocks_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                             uint64_t* n_symbols, int mem_kind)
{
    if (!ctx || !buf || (!out && out_cap)) return RB200_E_ARG;
    if (!container_mem_ok(mem_kind, buf, out)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return container_decode_impl(ctx, buf, size, out, out_cap, n_symbols, mem_kind == RB200_MEM_DEVICE, kContainerVersionBlocks);
}

extern "C" int rb200_container_blocks_coder_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                   uint64_t* n_symbols, int mem_kind)
{
    if (!ctx || !buf || (!out && out_cap)) return RB200_E_ARG;
    if (!container_mem_ok(mem_kind, buf, out)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return container_decode_impl(ctx, buf, size, out, out_cap, n_symbols, mem_kind == RB200_MEM_DEVICE, kContainerVersionBlocksCoder);
}

extern "C" int rb200_container_blocks_alias_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                   uint64_t* n_symbols, int mem_kind)
{
    if (!ctx || !buf || (!out && out_cap)) return RB200_E_ARG;
    if (!container_mem_ok(mem_kind, buf, out)) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    return container_decode_impl(ctx, buf, size, out, out_cap, n_symbols, mem_kind == RB200_MEM_DEVICE, kContainerVersionBlocksAlias);
}

namespace {

// the argument rules the async decodes share: device memory, buf and out 16-byte aligned, d_n_symbols 8-byte aligned
bool async_args_ok(const rb200_ctx* ctx, const uint8_t* buf, const uint8_t* out, const uint64_t* d_n_symbols)
{
    return ctx && buf && out && !(reinterpret_cast<uintptr_t>(d_n_symbols) & 7) && container_mem_ok(RB200_MEM_DEVICE, buf, out);
}

// The async decode of a container of `version` (container_decode.cuh), or of any per-block version
// (kContainerVersionAnyBlocks), in its own workspace: plan, meta CRC, blob CRC, the prefix check, version 1's model
// check and table build, the verdict, then every decoder of the version (of versions 2-4) on its fixed grid; the
// verdict's go names the one that runs.  Lengths and positions the host cannot know come from the plan on the device;
// the host passes only bounds it knows (size).  No copy, no synchronisation, no allocation.
int container_decode_async(rb200_ctx* ctx, uint16_t version, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                           uint64_t* d_n_symbols)
{
    DeviceGuard g(ctx->device);
    const bool any = version == kContainerVersionAnyBlocks;
    ContainerAsyncWork* w = any ? ctx->d_async_any : ctx->d_async[version - 1];
    const bool stored = version == kContainerVersionBlocksStored, v6 = version == kContainerVersionStored;
    const int first = kDecoderFirst[any ? kContainerVersionBlocks - 1 : version - 1];
    const int last = kDecoderFirst[any ? kContainerVersionBlocksAlias : version];
    const uint32_t sms = static_cast<uint32_t>(ctx->sms);
    const uint64_t after_head = size > sizeof(ContainerHeader) ? size - sizeof(ContainerHeader) : 0;
    cudaStream_t s = ctx->stream;
    if (v6) {
        container_stored_plan_kernel<<<1, 32, 0, s>>>(buf, size, w);
    } else {
        auto plan = stored ? container_plan_kernel<true> : container_plan_kernel<false>;
        plan<<<1, 32, 0, s>>>(buf, size, version, w);
    }
    int rc = check_launch(ctx, "container_plan_kernel");
    if (rc != RB200_OK) return rc;
    crc32_kernel<<<crc32_grid(sms, after_head), kCrcThreads, kCrcSmemBytes, s>>>(buf + sizeof(ContainerHeader), after_head, &w->plan.meta_len,
                                                                                 nullptr, 0, &w->crc_work, &w->crc[0]);
    rc = check_launch(ctx, "crc32_kernel(meta)");
    if (rc != RB200_OK) return rc;
    crc32_kernel<<<crc32_grid(sms, size), kCrcThreads, kCrcSmemBytes, s>>>(buf, size, &w->plan.blob_len, &w->plan.blob_off, 0,
                                                                           &w->crc_work, &w->crc[1]);
    rc = check_launch(ctx, "crc32_kernel(blob)");
    if (rc != RB200_OK) return rc;
    if (v6) {
        container_stored_check_kernel<<<sms * kPrefixCtasPerSm, kPrefixWarps * 32, 0, s>>>(buf, w);
    } else {
        auto prefix = stored ? container_prefix_check_kernel<true> : container_prefix_check_kernel<false>;
        prefix<<<sms * kPrefixCtasPerSm, kPrefixWarps * 32, 0, s>>>(buf, w);
    }
    rc = check_launch(ctx, "container_prefix_check_kernel");
    if (rc != RB200_OK) return rc;
    if (version == kContainerVersion || v6) {
        container_table_kernel<<<1, kTableThreads, 0, s>>>(buf, w);
        rc = check_launch(ctx, "container_table_kernel");
        if (rc != RB200_OK) return rc;
    }
    // version 6 runs the STORED twins of version 1's decoders, with version 1's ids
    container_verdict_kernel<<<1, 32, 0, s>>>(buf, out_cap, d_n_symbols, w, ctx->d_status, v6 ? kContainerVersion : version);
    rc = check_launch(ctx, "container_verdict_kernel");
    for (int i = first; i < last && rc == RB200_OK; i++) {
        const DecoderLaunch& l = ctx->async_decoders[i];
        l.kernel<<<l.grid, l.threads, l.smem, s>>>(buf, out, w, ctx->d_status);
        rc = check_launch(ctx, l.name);
    }
    return rc;
}

}  // namespace

// Six launches: the checks and the block decoder.
extern "C" int rb200_container_blocks_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                   uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionBlocks, buf, size, out, out_cap, d_n_symbols);
}

// Seventeen launches: the checks, the table kernel and every decoder variant rb200_decode can pick.
extern "C" int rb200_container_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                            uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersion, buf, size, out, out_cap, d_n_symbols);
}

// Nine launches: the checks and the block decoder variants of the byte and rans64 coders (RB200_BLOCK_DISPATCH).
extern "C" int rb200_container_blocks_coder_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                         uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionBlocksCoder, buf, size, out, out_cap, d_n_symbols);
}

// Eight launches: the checks and the block decoder variants of the alias coder (RB200_BLOCK_DISPATCH).
extern "C" int rb200_container_blocks_alias_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                         uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionBlocksAlias, buf, size, out, out_cap, d_n_symbols);
}

// Thirteen launches: the checks and the STORED block decoder variants of RB200_BLOCK_DISPATCH (version 5).
extern "C" int rb200_container_blocks_stored_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                          uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionBlocksStored, buf, size, out, out_cap, d_n_symbols);
}

// Seventeen launches: version 6's checks, the table kernel and the STORED twin of every decoder variant of version 1.
extern "C" int rb200_container_stored_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                   uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionStored, buf, size, out, out_cap, d_n_symbols);
}

// Thirteen launches: the checks and every block decoder variant of RB200_BLOCK_DISPATCH (versions 2, 3 and 4).
extern "C" int rb200_container_blocks_any_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                                       uint64_t* d_n_symbols)
{
    if (!async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return container_decode_async(ctx, kContainerVersionAnyBlocks, buf, size, out, out_cap, d_n_symbols);
}

namespace {

// the argument rules of both model encodes, with n the length (fixed call) or its bound n_max (varlen call)
bool model_encode_args_ok(const rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, size_t n, uint32_t chunk_syms,
                          const uint8_t* out)
{
    if (!ctx || !in || !out || !container_mem_ok(RB200_MEM_DEVICE, out, nullptr)) return false;
    if (coder < RB200_CODER_WORD || coder > RB200_CODER_RANS64 || scale_bits < 8 || scale_bits > 16) return false;
    if (coder == RB200_CODER_WORD && scale_bits != kWordScaleBits) return false;
    if (!chunk_ok(chunk_syms) || (n >> 32)) return false;            // counts of 32 bits, as rb200_model_from_data
    return rb200_chunk_count(n, chunk_syms) < (1ull << 31);
}

// the encode tables the model kernel builds in the workspace; the word coder's gate is its r32
EncodeTables workspace_tables(ModelAsyncWork* w, int coder, uint32_t scale_bits)
{
    return EncodeTables{coder, scale_bits, {w->word_enc, w->word_enc32}, 0, &w->r32,
                        coder == RB200_CODER_ALIAS ? w->alias_enc : w->byte_enc, w->alias_remap, w->r64_enc};
}

// The body of both model encodes (model_kernels.cuh): histogram, model kernel, the coder's encoder, the CRCs and the
// header.  d_n null: n symbols, every length by value.  d_n set: n is the bound n_max, which sizes every launch; the plan
// kernel reads *d_n into the record at every run, and every later kernel is its GEOM instance.  a set (the auto encode):
// the choice kernel, the CHOSEN model kernel, every group's gated encode, the CHOSEN header kernel; coder and
// scale_bits are then the first candidate's, for the host-side layout only (it does not depend on them).
int model_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, size_t n, const uint64_t* d_n, uint32_t chunk_syms,
                 uint32_t flags, uint8_t* out, size_t out_cap, const AutoPlan* a = nullptr)
{
    const size_t n_chunks = rb200_chunk_count(n, chunk_syms);
    const ContainerHeader h = container_header(coder, scale_bits, chunk_syms, n, n_chunks, 0, flags);
    const size_t dir_off = container_dir_offset(h), dir_end = container_dir_end(h), boff = container_blob_offset(h);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    cudaStream_t s = ctx->stream;
    ModelAsyncWork* w = ctx->d_model_async;
    VarlenGeom* geom = d_n ? &w->geom : nullptr;
    int rc = RB200_OK;
    if (a) {                 // every group's workspace first, so that no group's launch is followed by a reallocation
        for (uint32_t k = 0; k < a->n_groups && rc == RB200_OK; k++)
            rc = reserve_plan(ctx, plan_encode(ctx, a->coder[k], a->sb[k], static_cast<uint32_t>(n_chunks), chunk_syms, false));
        if (rc != RB200_OK) return rc;
    }
    if (geom) {
        varlen_plan_kernel<<<1, 32, 0, s>>>(d_n, n, chunk_syms, out_cap, geom, ctx->d_status);
        rc = check_launch(ctx, "varlen_plan_kernel");
        if (rc != RB200_OK) return rc;
    }
    RB_CUDA(ctx, cudaMemsetAsync(w->counts, 0, sizeof w->counts, s));
    launch_histogram(s, static_cast<uint32_t>(ctx->sms), in, n, w->counts, geom);
    rc = check_launch(ctx, "histogram_kernel");
    if (rc != RB200_OK) return rc;
    if (a) {
        coder_choice_kernel<<<1, a->list.n * 32, 0, s>>>(a->list, n_chunks, w, geom, ctx->d_status);
        rc = check_launch(ctx, "coder_choice_kernel");
        if (rc != RB200_OK) return rc;
    }
    auto model = a ? (geom ? container_model_kernel<true, true> : container_model_kernel<false, true>)
                   : (geom ? container_model_kernel<true> : container_model_kernel<false>);
    model<<<1, kModelThreads, 0, s>>>(static_cast<uint32_t>(coder), scale_bits, word_r32_allowed() ? 1u : 0u, w, ctx->d_status);
    rc = check_launch(ctx, "container_model_kernel");
    if (rc != RB200_OK) return rc;
    const bool blob_crc = (h.flags & RB200_CONTAINER_CRC_BLOB) != 0;
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + dir_off);
    uint8_t* blob = geom ? out : out + boff;
    if (a) {
        for (uint32_t k = 0; k < a->n_groups && rc == RB200_OK; k++) {
            EncodeTables t = workspace_tables(w, a->coder[k], a->sb[k]);
            t.choice = &w->choice;
            t.group = k;
            rc = encode_device(ctx, t, in, n, chunk_syms, blob, out_cap - boff, dir, geom);
        }
    } else {
        rc = encode_device(ctx, workspace_tables(w, coder, scale_bits), in, n, chunk_syms, blob, out_cap - boff, dir, geom);
    }
    if (rc == RB200_OK) rc = launch_crc(ctx, out + dir_off, dir_end - dir_off, geom ? &geom->dir_len : nullptr, 0, ctx->d_crc);
    if (rc == RB200_OK && blob_crc) {
        if (geom) {
            varlen_blob_len_kernel<<<1, 32, 0, s>>>(out, geom);
            rc = check_launch(ctx, "varlen_blob_len_kernel");
            if (rc == RB200_OK) rc = launch_crc(ctx, out, out_cap, &geom->blob_len, 0, ctx->d_crc + 1, &geom->blob_off);
        } else {
            rc = launch_crc(ctx, out + boff, out_cap - boff, dir + n_chunks, 0, ctx->d_crc + 1);
        }
    }
    if (rc != RB200_OK) return rc;
    auto finish = a ? (geom ? container_finish_kernel<true, true> : container_finish_kernel<false, true>)
                    : (geom ? container_finish_kernel<true> : container_finish_kernel<false>);
    finish<<<1, 32, 0, s>>>(out, h, dir_off, boff, out_cap, w->freqs, ctx->d_crc, ctx->d_status, geom, &w->choice);
    return check_launch(ctx, "container_finish_kernel");
}

}  // namespace

// rb200_model_from_data + rb200_container_encode (device memory) + rb200_model_destroy with kernels alone: five to seven
// launches and one memset, no copy, no synchronisation; the encode workspace grows as in rb200_container_encode.
extern "C" int rb200_container_model_encode_async(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, size_t n,
                                                  uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!model_encode_args_ok(ctx, coder, scale_bits, in, n, chunk_syms, out)) return RB200_E_ARG;
    if (n == 0) return RB200_E_MODEL;                                // normalize_freqs divides by the total
    return model_encode(ctx, coder, scale_bits, in, n, nullptr, chunk_syms, flags, out, out_cap);
}

// rb200_container_model_encode_async with the length read from device memory at every run: the plan kernel, then the
// same stages on launch shapes sized for n_max, each taking the length from the plan's record.  Eight to eleven launches
// and one or two memsets, no copy, no synchronisation; the workspace grows as the fixed call's for n_max.
extern "C" int rb200_container_model_encode_varlen_async(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in,
                                                         const uint64_t* d_n, size_t n_max, uint32_t chunk_syms, uint32_t flags,
                                                         uint8_t* out, size_t out_cap)
{
    if (!d_n || (reinterpret_cast<uintptr_t>(d_n) & 7) || n_max == 0) return RB200_E_ARG;
    if (!model_encode_args_ok(ctx, coder, scale_bits, in, n_max, chunk_syms, out)) return RB200_E_ARG;
    return model_encode(ctx, coder, scale_bits, in, n_max, d_n, chunk_syms, flags, out, out_cap);
}

// Either call above with the pair chosen on the GPU at every run (coder_choice_kernel): the choice kernel, the CHOSEN
// model kernel, one gated encode group per distinct encoder instance of the list, the CHOSEN header kernel.  No copy,
// no synchronisation; the workspace grows for every group's plan.
extern "C" int rb200_container_model_encode_auto_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                       uint32_t tolerance_ppm, const uint8_t* in, const uint64_t* d_n, size_t n,
                                                       uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (d_n && ((reinterpret_cast<uintptr_t>(d_n) & 7) || n == 0)) return RB200_E_ARG;
    for (uint32_t i = 0; i < n_candidates; i++)
        if (!model_encode_args_ok(ctx, static_cast<int>(candidates[i] >> 8), candidates[i] & 0xffu, in, n, chunk_syms, out)) return RB200_E_ARG;
    if (!d_n && n == 0) return RB200_E_MODEL;                        // normalize_freqs divides by the total
    const AutoPlan a = plan_auto(candidates, n_candidates, tolerance_ppm);
    return model_encode(ctx, static_cast<int>(candidates[0] >> 8), candidates[0] & 0xffu, in, n, d_n, chunk_syms, flags, out, out_cap, &a);
}

// rb200_container_blocks_encode / _coder_encode / _alias_encode (DEVICE, models built) with the pair chosen on the GPU
// at every run: the choice kernel (after a memset of its sums), one gated encode group per distinct encoder instance
// of the list, the model + directory CRC, the optional blob CRC, the per-block header kernel.
extern "C" int rb200_container_blocks_model_encode_auto_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                              uint32_t tolerance_ppm, const uint8_t* in, uint32_t n_blocks,
                                                              uint32_t block_size, uint32_t chunk_syms, uint32_t flags, uint8_t* out,
                                                              size_t out_cap)
{
    if (!blocks_candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!blocks_container_args_ok(ctx, in, n_blocks, block_size, chunk_syms, out, RB200_MEM_DEVICE)) return RB200_E_ARG;
    const AutoPlan a = plan_auto(candidates, n_candidates, tolerance_ppm);
    return blocks_container_encode(ctx, container_blocks_header(n_blocks, block_size, chunk_syms, 0, flags), in, nullptr, nullptr, out,
                                   out_cap, &a);
}

// rb200_container_blocks_model_encode_auto_async with the block count read from device memory at every run: the plan
// kernel, then the same stages on launch shapes sized for n_blocks_max, each taking the count, the directory's and the
// blob's places and the CRC lengths from the plan's record.  One candidate: the plan kernel writes the choice record and
// no choice kernel runs.
extern "C" int rb200_container_blocks_model_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                                uint32_t tolerance_ppm, const uint8_t* in, const uint32_t* d_n_blocks,
                                                                uint32_t n_blocks_max, uint32_t block_size, uint32_t chunk_syms,
                                                                uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!d_n_blocks || (reinterpret_cast<uintptr_t>(d_n_blocks) & 3) || n_blocks_max == 0) return RB200_E_ARG;
    if (!blocks_candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!blocks_container_args_ok(ctx, in, n_blocks_max, block_size, chunk_syms, out, RB200_MEM_DEVICE)) return RB200_E_ARG;
    const AutoPlan a = plan_auto(candidates, n_candidates, tolerance_ppm);
    return blocks_container_encode(ctx, container_blocks_header(n_blocks_max, block_size, chunk_syms, 0, flags), in, nullptr, d_n_blocks,
                                   out, out_cap, &a);
}

namespace {

// rb200_container_blocks_stored_encode_async: the choice kernel (after a memset of its sums) or, for one candidate,
// blocks_one_pair_kernel; one GATED split encoder per launch group of the list, all into one workspace of one
// worst-case slot per chunk (slot_bytes_for does not depend on the coder), so that every stream's size is known before
// anything is placed; blocks_store_kernel; the scan, the tile prefix and compact_stored_kernel, ungated; the model +
// directory CRC, the optional blob CRC and container_blocks_stored_finish_kernel (version 5).  The workspace: the split plan's, then the
// per-block verdicts after its tile sums.  d_n_blocks set (rb200_container_blocks_stored_encode_varlen_async): n_blocks
// is the bound n_blocks_max, which sizes the workspace and every launch; blocks_varlen_plan_kernel reads *d_n_blocks into
// the record at every run (for one candidate it also writes the choice record), and every later kernel is its GEOM
// instance.  Arguments are checked by the caller.
int blocks_stored_encode(rb200_ctx* ctx, const AutoPlan& a, const uint8_t* in, uint32_t n_blocks, const uint32_t* d_n_blocks,
                         uint32_t block_size, uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    const ContainerHeader h = container_blocks_header(n_blocks, block_size, chunk_syms, 0, flags);
    const size_t dir_off = container_dir_offset(h), dir_end = container_dir_end(h), boff = container_blob_offset(h);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    cudaStream_t s = ctx->stream;
    BlocksChoice* r = ctx->d_blocks_choice;
    BlocksVarlenGeom* geom = d_n_blocks ? ctx->d_blocks_geom : nullptr;
    const uint32_t per_block = block_size / chunk_syms, n_chunks = static_cast<uint32_t>(h.n_chunks);
    EncodePlan p = {};
    p.n_chunks = n_chunks;
    p.slots = n_chunks;
    p.slot_bytes = slot_bytes_for(chunk_syms);
    p.threads = block_threads(block_size, chunk_syms);
    const size_t longs = (n_chunks + kScanTile - 1) / kScanTile + 1;
    int rc = reserve(ctx, ctx->scratch, p.slots * p.slot_bytes + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->sizes, plan_head_bytes(p) + longs * sizeof(uint64_t) + n_blocks * sizeof(uint32_t));
    if (rc != RB200_OK) return rc;
    uint8_t* scratch = static_cast<uint8_t*>(ctx->scratch.p);
    uint32_t* sizes = static_cast<uint32_t*>(ctx->sizes.p);
    uint64_t* tile_sums = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(ctx->sizes.p) + plan_head_bytes(p));
    uint32_t* stored = reinterpret_cast<uint32_t*>(tile_sums + longs);
    uint16_t* model = reinterpret_cast<uint16_t*>(out + sizeof(ContainerHeader));
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + dir_off);
    const bool one = a.list.n == 1;
    if (!one) RB_CUDA(ctx, cudaMemsetAsync(&r->done, 0, sizeof(BlocksChoice) - offsetof(BlocksChoice, done), s));
    if (geom) {
        blocks_varlen_plan_kernel<<<1, 32, 0, s>>>(d_n_blocks, n_blocks, block_size, chunk_syms, out_cap, one ? a.list.pair[0] : 0u, geom, r,
                                                   ctx->d_status);
        rc = check_launch(ctx, "blocks_varlen_plan_kernel");
    } else if (one) {
        blocks_one_pair_kernel<<<1, 32, 0, s>>>(a.list.pair[0], r);
        rc = check_launch(ctx, "blocks_one_pair_kernel");
    }
    if (rc == RB200_OK && !one) {
        auto choice = geom ? blocks_choice_kernel<true> : blocks_choice_kernel<false>;
        choice<<<n_blocks, kBlocksChoiceWarps * 32, 0, s>>>(a.list, in, block_size, chunk_syms, r, ctx->d_status, geom);
        rc = check_launch(ctx, "blocks_choice_kernel");
    }
    for (uint32_t k = 0; k < a.n_groups && rc == RB200_OK; k++) {
        launch_block_encode(s, static_cast<uint32_t>(a.coder[k]), a.sb[k], true, n_blocks, p.threads,
                            block_coder_encode_smem(static_cast<uint32_t>(a.coder[k]), a.sb[k], p.threads), in, block_size, model, chunk_syms,
                            scratch, p.slot_bytes, sizes, ctx->d_status, &r->choice, k, geom);
        rc = check_launch(ctx, "block_coder_encode_kernel");
    }
    if (rc != RB200_OK) return rc;
    const uint32_t store_grid = (n_blocks + kStoreWarps - 1) / kStoreWarps;
    if (geom) {
        blocks_store_varlen_kernel<<<store_grid, kStoreWarps * 32, 0, s>>>(sizes, per_block, chunk_syms, model, stored, geom);
        rc = check_launch(ctx, "blocks_store_varlen_kernel");
    } else {
        blocks_store_kernel<<<store_grid, kStoreWarps * 32, 0, s>>>(sizes, n_blocks, per_block, chunk_syms, model, stored);
        rc = check_launch(ctx, "blocks_store_kernel");
    }
    const StoredBlocks st = {in, stored, per_block, chunk_syms};
    if (rc == RB200_OK)
        rc = geom ? finish_encode(ctx, scratch, p.slot_bytes, sizes, tile_sums, n_chunks, out, out_cap, nullptr, &geom->v, nullptr, 0, &st)
                  : finish_encode(ctx, scratch, p.slot_bytes, sizes, tile_sums, n_chunks, out + boff, out_cap - boff, dir, nullptr, nullptr, 0, &st);
    if (rc == RB200_OK)
        rc = launch_crc(ctx, out + sizeof(ContainerHeader), dir_end - sizeof(ContainerHeader), geom ? &geom->meta_len : nullptr, 0, ctx->d_crc);
    if (rc == RB200_OK && (flags & RB200_CONTAINER_CRC_BLOB)) {
        if (geom) {
            varlen_blob_len_kernel<<<1, 32, 0, s>>>(out, &geom->v);
            rc = check_launch(ctx, "varlen_blob_len_kernel");
            if (rc == RB200_OK) rc = launch_crc(ctx, out, out_cap, &geom->v.blob_len, 0, ctx->d_crc + 1, &geom->v.blob_off);
        } else {
            rc = launch_crc(ctx, out + boff, out_cap - boff, dir + n_chunks, 0, ctx->d_crc + 1);
        }
    }
    if (rc != RB200_OK) return rc;
    if (geom) {
        container_blocks_stored_finish_varlen_kernel<<<1, 32, 0, s>>>(out, h, out_cap, ctx->d_crc, ctx->d_status, r, geom);
        return check_launch(ctx, "container_blocks_stored_finish_varlen_kernel");
    }
    container_blocks_stored_finish_kernel<<<1, 32, 0, s>>>(out, h, dir_off, boff, out_cap, ctx->d_crc, ctx->d_status, r);
    return check_launch(ctx, "container_blocks_stored_finish_kernel");
}

}  // namespace

// The auto encode's choice and model-building encoders, with every block whose coded chunks would take more than its
// stored size stored verbatim (version 5).  Eight to eleven launches and one memset, no copy, no synchronisation.
extern "C" int rb200_container_blocks_stored_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                          uint32_t tolerance_ppm, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                                          uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!blocks_candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!blocks_container_args_ok(ctx, in, n_blocks, block_size, chunk_syms, out, RB200_MEM_DEVICE)) return RB200_E_ARG;
    return blocks_stored_encode(ctx, plan_auto(candidates, n_candidates, tolerance_ppm), in, n_blocks, nullptr, block_size, chunk_syms, flags,
                                out, out_cap);
}

// rb200_container_blocks_stored_encode_async with the block count read from device memory at every run: the plan kernel,
// then the same stages on launch shapes sized for n_blocks_max, each taking the count, the directory's and the blob's
// places and the CRC lengths from the plan's record.  One candidate: the plan kernel writes the choice record.
extern "C" int rb200_container_blocks_stored_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                                 uint32_t tolerance_ppm, const uint8_t* in, const uint32_t* d_n_blocks,
                                                                 uint32_t n_blocks_max, uint32_t block_size, uint32_t chunk_syms,
                                                                 uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!d_n_blocks || (reinterpret_cast<uintptr_t>(d_n_blocks) & 3) || n_blocks_max == 0) return RB200_E_ARG;
    if (!blocks_candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!blocks_container_args_ok(ctx, in, n_blocks_max, block_size, chunk_syms, out, RB200_MEM_DEVICE)) return RB200_E_ARG;
    return blocks_stored_encode(ctx, plan_auto(candidates, n_candidates, tolerance_ppm), in, n_blocks_max, d_n_blocks, block_size, chunk_syms,
                                flags, out, out_cap);
}

namespace {

// rb200_container_stored_encode_async (version 6): the histogram, coder_choice_kernel and the CHOSEN model kernel of the
// auto encode; one GATED split encoder per launch group of the list, all into one workspace of one worst-case slot per
// chunk (slot_bytes_for does not depend on the coder), so that every stream's size is known before anything is placed;
// chunks_store_kernel (the bitmap and the per-chunk verdicts); the scan, the tile prefix and
// chunks_stored_compaction_kernel, ungated; the CRC of everything between the model and the blob, the optional blob CRC
// and container_stored_finish_kernel.  The workspace: the split plan's, then the verdicts after its tile sums.
// d_n set (rb200_container_stored_encode_varlen_async): n is the bound n_max, which sizes the workspace and every
// launch; stored_varlen_plan_kernel reads *d_n into the record at every run, and every later kernel is its GEOM
// instance.  Arguments are checked by the caller.
int stored_encode(rb200_ctx* ctx, const AutoPlan& a, const uint8_t* in, size_t n, const uint64_t* d_n, uint32_t chunk_syms, uint32_t flags,
                  uint8_t* out, size_t out_cap)
{
    const uint32_t n_chunks = static_cast<uint32_t>(rb200_chunk_count(n, chunk_syms));
    const ContainerHeader h = container_header(static_cast<int>(a.list.pair[0] >> 8), a.list.pair[0] & 0xffu, chunk_syms, n, n_chunks, 0, flags);
    const size_t boff = container_bitmap_blob_offset(n_chunks);
    if (out_cap < boff) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    cudaStream_t s = ctx->stream;
    ModelAsyncWork* w = ctx->d_model_async;
    StoredVarlenGeom* sg = d_n ? ctx->d_stored_geom : nullptr;
    const VarlenGeom* geom = sg ? &sg->v : nullptr;
    EncodePlan p = {};
    p.n_chunks = n_chunks;
    p.slots = n_chunks;
    p.slot_bytes = slot_bytes_for(chunk_syms);
    const size_t longs = (n_chunks + kScanTile - 1) / kScanTile + 1;
    int rc = reserve(ctx, ctx->scratch, p.slots * p.slot_bytes + 16);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->sizes, plan_head_bytes(p) + longs * sizeof(uint64_t) + n_chunks * sizeof(uint32_t));
    if (rc != RB200_OK) return rc;
    uint8_t* scratch = static_cast<uint8_t*>(ctx->scratch.p);
    uint32_t* sizes = static_cast<uint32_t*>(ctx->sizes.p);
    uint64_t* tile_sums = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(ctx->sizes.p) + plan_head_bytes(p));
    uint32_t* stored = reinterpret_cast<uint32_t*>(tile_sums + longs);
    const EncodeWorkspace ws = {scratch, nullptr, nullptr, sizes, tile_sums};
    uint64_t* dir = reinterpret_cast<uint64_t*>(out + kContainerDirOffset);
    if (sg) {
        stored_varlen_plan_kernel<<<1, 32, 0, s>>>(d_n, n, chunk_syms, out_cap, sg, &w->geom, ctx->d_status);
        rc = check_launch(ctx, "stored_varlen_plan_kernel");
        if (rc != RB200_OK) return rc;
    }
    RB_CUDA(ctx, cudaMemsetAsync(w->counts, 0, sizeof w->counts, s));
    launch_histogram(s, static_cast<uint32_t>(ctx->sms), in, n, w->counts, geom);
    rc = check_launch(ctx, "histogram_kernel");
    if (rc != RB200_OK) return rc;
    coder_choice_kernel<<<1, a.list.n * 32, 0, s>>>(a.list, n_chunks, w, geom, ctx->d_status);
    rc = check_launch(ctx, "coder_choice_kernel");
    if (rc != RB200_OK) return rc;
    auto model = geom ? container_model_kernel<true, true> : container_model_kernel<false, true>;
    model<<<1, kModelThreads, 0, s>>>(h.coder, h.scale_bits, word_r32_allowed() ? 1u : 0u, w, ctx->d_status);
    rc = check_launch(ctx, "container_model_kernel");
    for (uint32_t k = 0; k < a.n_groups && rc == RB200_OK; k++) {
        EncodeTables t = workspace_tables(w, a.coder[k], a.sb[k]);
        t.choice = &w->choice;
        t.group = k;
        const EncodePlan pk = plan_encode(ctx, a.coder[k], a.sb[k], n_chunks, chunk_syms, false, true);
        rc = launch_encoder(ctx, t, pk, in, n, chunk_syms, n_chunks, ws, nullptr, 0, nullptr, geom);
    }
    if (rc != RB200_OK) return rc;
    const uint32_t store_grid = static_cast<uint32_t>((container_bitmap_words(n_chunks) * 32 + kChunkStoreThreads - 1) / kChunkStoreThreads);
    if (geom) {
        chunks_store_varlen_kernel<<<store_grid, kChunkStoreThreads, 0, s>>>(sizes, chunk_syms, out, stored, geom);
        rc = check_launch(ctx, "chunks_store_varlen_kernel");
    } else {
        chunks_store_kernel<<<store_grid, kChunkStoreThreads, 0, s>>>(sizes, n_chunks, n, chunk_syms, out, stored);
        rc = check_launch(ctx, "chunks_store_kernel");
    }
    if (rc != RB200_OK) return rc;
    // the scan and the tile prefix ungated; the compaction copies stored chunks from the input.  GEOM: the scan writes
    // the directory into the container `out` at the record's place, and the prefix and the compaction use the record's
    // tile count, whichever the host chose from the bound's
    const uint32_t tiles = (n_chunks + kScanTile - 1) / kScanTile;
    auto scan = geom ? scan_tiles_kernel<true> : scan_tiles_kernel<false>;
    scan<<<tiles, 1024, 0, s>>>(sizes, n_chunks, geom ? reinterpret_cast<uint64_t*>(out) : dir, tile_sums, geom, nullptr, 0);
    rc = check_launch(ctx, "scan_tiles_kernel");
    const uint32_t prefixed = tiles > kTilePrefixThreshold ? 1u : 0u;
    if (rc == RB200_OK && prefixed) {
        auto prefix = geom ? tile_prefix_kernel<true> : tile_prefix_kernel<false>;
        prefix<<<1, 1024, 0, s>>>(tile_sums, tiles, geom, nullptr, 0);
        rc = check_launch(ctx, "tile_prefix_kernel");
    }
    if (rc != RB200_OK) return rc;
    const StoredBlocks st = {in, stored, 1, chunk_syms, n};
    const uint32_t copy_grid = (n_chunks + kCopyWarps - 1) / kCopyWarps;
    if (geom) {
        chunks_stored_compaction_varlen_kernel<<<copy_grid, kCopyWarps * 32, 0, s>>>(scratch, p.slot_bytes, sizes, tile_sums, prefixed, out,
                                                                                     ctx->d_status, geom, st);
        rc = check_launch(ctx, "chunks_stored_compaction_varlen_kernel");
    } else {
        chunks_stored_compaction_kernel<<<copy_grid, kCopyWarps * 32, 0, s>>>(scratch, p.slot_bytes, sizes, dir, tile_sums, prefixed, n_chunks,
                                                                              out + boff, out_cap - boff, ctx->d_status, st);
        rc = check_launch(ctx, "chunks_stored_compaction_kernel");
    }
    if (rc == RB200_OK)
        rc = launch_crc(ctx, out + kContainerDirOffset, boff - kContainerDirOffset, sg ? &sg->meta_len : nullptr, 0, ctx->d_crc);
    if (rc == RB200_OK && (flags & RB200_CONTAINER_CRC_BLOB)) {
        if (sg) {
            varlen_blob_len_kernel<<<1, 32, 0, s>>>(out, &sg->v);
            rc = check_launch(ctx, "varlen_blob_len_kernel");
            if (rc == RB200_OK) rc = launch_crc(ctx, out, out_cap, &sg->v.blob_len, 0, ctx->d_crc + 1, &sg->v.blob_off);
        } else {
            rc = launch_crc(ctx, out + boff, out_cap - boff, dir + n_chunks, 0, ctx->d_crc + 1);
        }
    }
    if (rc != RB200_OK) return rc;
    if (sg) {
        container_stored_finish_varlen_kernel<<<1, 32, 0, s>>>(out, h, out_cap, w->freqs, ctx->d_crc, ctx->d_status, &w->choice, sg);
        return check_launch(ctx, "container_stored_finish_varlen_kernel");
    }
    container_stored_finish_kernel<<<1, 32, 0, s>>>(out, h, boff, out_cap, w->freqs, ctx->d_crc, ctx->d_status, &w->choice);
    return check_launch(ctx, "container_stored_finish_kernel");
}

}  // namespace

// The auto encode's choice, model and split encoders, with every chunk whose stream is longer than its symbols stored
// verbatim (version 6).  Ten to fourteen launches and one memset, no copy, no synchronisation.
extern "C" int rb200_container_stored_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                                   const uint8_t* in, size_t n, uint32_t chunk_syms, uint32_t flags, uint8_t* out,
                                                   size_t out_cap)
{
    if (!candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    for (uint32_t i = 0; i < n_candidates; i++)
        if (!model_encode_args_ok(ctx, static_cast<int>(candidates[i] >> 8), candidates[i] & 0xffu, in, n, chunk_syms, out)) return RB200_E_ARG;
    if (n == 0) return RB200_E_MODEL;                                // normalize_freqs divides by the total
    return stored_encode(ctx, plan_auto(candidates, n_candidates, tolerance_ppm), in, n, nullptr, chunk_syms, flags, out, out_cap);
}

// rb200_container_stored_encode_async with the length read from device memory at every run: the plan kernel, then the
// same stages on launch shapes sized for n_max, each taking the length, the chunk count, the bitmap's and the blob's
// places and the CRC lengths from the plan's record.
extern "C" int rb200_container_stored_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                          uint32_t tolerance_ppm, const uint8_t* in, const uint64_t* d_n, size_t n_max,
                                                          uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!d_n || (reinterpret_cast<uintptr_t>(d_n) & 7) || n_max == 0) return RB200_E_ARG;
    if (!candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    for (uint32_t i = 0; i < n_candidates; i++)
        if (!model_encode_args_ok(ctx, static_cast<int>(candidates[i] >> 8), candidates[i] & 0xffu, in, n_max, chunk_syms, out))
            return RB200_E_ARG;
    return stored_encode(ctx, plan_auto(candidates, n_candidates, tolerance_ppm), in, n_max, d_n, chunk_syms, flags, out, out_cap);
}

namespace {

// a grid of every CTA of the byte-plane kernels that is resident at once: they stride over what they move
uint32_t planes_grid(const rb200_ctx* ctx) { return static_cast<uint32_t>(ctx->sms) * kPlanesCtasPerSm; }

// The list a tensor-list call reads, in device memory, with its prefix workspace (count + 1 u64)
struct TensorList {
    const rb200_tensor_ref* refs;
    uint32_t count;
    uint64_t* prefix;
};

// geom set: the varlen split, m from the record; base set: the delta split; list set: the segmented split (geom set too)
int launch_split(rb200_ctx* ctx, uint32_t w, const uint8_t* in, const uint8_t* base, uint64_t m, const PlanesVarlenGeom* geom, const TensorList* list,
                 uint8_t* planes, uint64_t stride)
{
    if (list) {
        auto split = w == 2 ? tensors_split_kernel<2> : w == 4 ? tensors_split_kernel<4> : tensors_split_kernel<8>;
        split<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(list->refs, list->prefix, list->count, geom, planes, stride);
        return check_launch(ctx, "tensors_split_kernel");
    }
    if (base) {
        auto split = w == 2 ? delta_split_kernel<2> : w == 4 ? delta_split_kernel<4> : delta_split_kernel<8>;
        split<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(in, base, m, planes, stride);
        return check_launch(ctx, "delta_split_kernel");
    }
    if (geom) {
        auto split = w == 2 ? planes_split_varlen_kernel<2> : w == 4 ? planes_split_varlen_kernel<4> : planes_split_varlen_kernel<8>;
        split<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(in, geom, planes, stride);
        return check_launch(ctx, "planes_split_varlen_kernel");
    }
    auto split = w == 2 ? planes_split_kernel<2> : w == 4 ? planes_split_kernel<4> : planes_split_kernel<8>;
    split<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(in, m, planes, stride);
    return check_launch(ctx, "planes_split_kernel");
}

// base set: the delta interleave, out = base + the decoded difference; list set: the segmented interleave into its refs
int launch_interleave(rb200_ctx* ctx, uint32_t w, const uint8_t* planes, uint64_t stride, const uint8_t* base, const TensorList* list, uint8_t* out,
                      const PlanesWork* r)
{
    if (list) {
        auto interleave = w == 2 ? tensors_interleave_kernel<2> : w == 4 ? tensors_interleave_kernel<4> : tensors_interleave_kernel<8>;
        interleave<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(planes, stride, list->refs, list->prefix, list->count, r);
        return check_launch(ctx, "tensors_interleave_kernel");
    }
    if (base) {
        auto interleave = w == 2 ? delta_interleave_kernel<2> : w == 4 ? delta_interleave_kernel<4> : delta_interleave_kernel<8>;
        interleave<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(planes, stride, base, out, r);
        return check_launch(ctx, "delta_interleave_kernel");
    }
    auto interleave = w == 2 ? planes_interleave_kernel<2> : w == 4 ? planes_interleave_kernel<4> : planes_interleave_kernel<8>;
    interleave<<<planes_grid(ctx), kPlanesThreads, 0, ctx->stream>>>(planes, stride, out, r);
    return check_launch(ctx, "planes_interleave_kernel");
}

// The split, then per plane the whole version 6 encode (stored_encode, unchanged) and a place kernel, then the version
// 7 header.  Plane 0 is encoded in place; the others into one staging area of rb200_container_stored_bound(n / w)
// bytes, from which their place kernel copies them to the end of the previous plane, whose size only the device knows.
// d_n set (rb200_container_planes_encode_varlen_async): n is the bound n_max, which sizes the workspaces, the planes'
// stride and every version 6 encode's bound; planes_varlen_plan_kernel reads *d_n into the context's PlanesVarlenGeom
// first, the split and the finish are their varlen forms, and every plane's version 6 encode is the varlen one, with
// the record's m as its length.  Arguments are checked here, with n_max for n.
// base set (rb200_container_delta_encode_async, never with d_n): the delta split, the base's CRC (crc32_kernel into the
// call's DeltaWork) right after it, and the delta finish, which writes version 8 with the CRC in reserved.
// refs set (rb200_container_tensors_encode_async, with n = n_max): the varlen encode with tensors_plan_kernel in place
// of its plan (the list checked, its prefix, the record, the directory), the segmented split, the directory's CRC
// (crc32_kernel into the call's TensorsWork) right after it, plane 0 after the directory, and the tensors finish, which
// writes version 9.  Arguments are checked here, with n_max for n and the list for in.
int planes_encode(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm, uint32_t w, const uint8_t* in,
                  const uint8_t* base, size_t n, const uint64_t* d_n, const rb200_tensor_ref* refs, uint32_t count, uint32_t chunk_syms,
                  uint32_t flags, uint8_t* out, size_t out_cap)
{
    const uint8_t* src = refs ? reinterpret_cast<const uint8_t*>(refs) : in;
    if (!container_planes_w_ok(w) || n == 0 || n % w || ((n / w) >> 32) || (reinterpret_cast<uintptr_t>(src) & 15)) return RB200_E_ARG;
    const size_t m = n / w;
    if (!candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    for (uint32_t i = 0; i < n_candidates; i++)
        if (!model_encode_args_ok(ctx, static_cast<int>(candidates[i] >> 8), candidates[i] & 0xffu, src, m, chunk_syms, out)) return RB200_E_ARG;
    const uint64_t dir_bytes = refs ? container_tensors_dir_bytes(count) : 0;
    const size_t plane_cap = rb200_container_stored_bound(m, chunk_syms), table_end = container_planes_table_end(w, dir_bytes);
    if (out_cap < rb200_container_planes_bound(n, w, chunk_syms) + dir_bytes) return RB200_E_SPACE;
    DeviceGuard g(ctx->device);
    const uint64_t stride = round16(m);
    int rc = reserve(ctx, ctx->planes_in, w * stride);
    if (rc == RB200_OK) rc = reserve(ctx, ctx->planes_enc_stage, plane_cap);
    if (rc == RB200_OK && refs) rc = reserve(ctx, ctx->tensors_enc_prefix, (count + 1ull) * sizeof(uint64_t));
    if (rc != RB200_OK) return rc;
    uint8_t* planes = static_cast<uint8_t*>(ctx->planes_in.p);
    uint8_t* stage = static_cast<uint8_t*>(ctx->planes_enc_stage.p);
    PlanesVarlenGeom* geom = d_n || refs ? ctx->d_planes_geom : nullptr;
    const TensorList list = {refs, count, static_cast<uint64_t*>(ctx->tensors_enc_prefix.p)};
    const AutoPlan a = plan_auto(candidates, n_candidates, tolerance_ppm);
    if (refs) {
        tensors_plan_kernel<<<1, kTensorsPlanThreads, 0, ctx->stream>>>(refs, count, w, n, list.prefix, geom,
                                                                        reinterpret_cast<uint64_t*>(out + container_planes_table_end(w, 0)));
        rc = check_launch(ctx, "tensors_plan_kernel");
        if (rc != RB200_OK) return rc;
    } else if (geom) {
        planes_varlen_plan_kernel<<<1, 32, 0, ctx->stream>>>(d_n, n, w, geom);
        rc = check_launch(ctx, "planes_varlen_plan_kernel");
        if (rc != RB200_OK) return rc;
    }
    rc = launch_split(ctx, w, in, base, m, geom, refs ? &list : nullptr, planes, stride);
    if (rc == RB200_OK && base) rc = launch_crc(ctx, base, n, nullptr, 0, &ctx->d_delta_enc->crc);
    if (rc == RB200_OK && refs)
        rc = launch_crc(ctx, out + container_planes_table_end(w, 0), 8ull * count, nullptr, 0, &ctx->d_tensors_enc->crc);
    const uint32_t units = w + static_cast<uint32_t>(dir_bytes / 16);
    for (uint32_t p = 0; p < w && rc == RB200_OK; p++) {
        uint8_t* dst = p ? stage : out + table_end;
        rc = stored_encode(ctx, a, planes + p * stride, m, geom ? &geom->m : nullptr, chunk_syms, flags, dst, plane_cap);
        if (rc != RB200_OK) break;
        planes_place_kernel<<<p ? planes_grid(ctx) : 1, kPlanesThreads, 0, ctx->stream>>>(out, dst, p, units, out_cap, ctx->d_planes_enc,
                                                                                         ctx->d_status);
        rc = check_launch(ctx, "planes_place_kernel");
    }
    if (rc != RB200_OK) return rc;
    ContainerHeader h{};
    h.magic = kContainerMagic;
    h.version = kContainerVersionPlanes;
    h.lanes = RB200_LANES;
    h.chunk_syms = chunk_syms;
    h.n_symbols = n;
    h.flags = flags;
    h.block_size = h.n_blocks = w;
    if (refs) {
        h.version = kContainerVersionTensors;
        h.n_blocks = count;
        tensors_finish_kernel<<<1, 32, 0, ctx->stream>>>(out, h, dir_bytes, geom, ctx->d_tensors_enc, ctx->d_planes_enc, ctx->d_status);
        return check_launch(ctx, "tensors_finish_kernel");
    }
    if (base) {
        delta_finish_kernel<<<1, 32, 0, ctx->stream>>>(out, h, ctx->d_delta_enc, ctx->d_planes_enc, ctx->d_status);
        return check_launch(ctx, "delta_finish_kernel");
    }
    if (geom) {
        planes_finish_varlen_kernel<<<1, 32, 0, ctx->stream>>>(out, h, geom, ctx->d_planes_enc, ctx->d_status);
        return check_launch(ctx, "planes_finish_varlen_kernel");
    }
    planes_finish_kernel<<<1, 32, 0, ctx->stream>>>(out, h, ctx->d_planes_enc, ctx->d_status);
    return check_launch(ctx, "planes_finish_kernel");
}

}  // namespace

// planes_encode without a device length: 2 + w * (11 to 15) launches and w memsets, no copy, no synchronisation.
extern "C" int rb200_container_planes_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                                   uint32_t elem_bytes, const uint8_t* in, size_t n, uint32_t chunk_syms, uint32_t flags,
                                                   uint8_t* out, size_t out_cap)
{
    return planes_encode(ctx, candidates, n_candidates, tolerance_ppm, elem_bytes, in, nullptr, n, nullptr, nullptr, 0, chunk_syms, flags, out,
                         out_cap);
}

// rb200_container_planes_encode_async with the length read from device memory at every run: the plan kernel, the
// varlen split, per plane version 6's varlen encode and the place kernel, the varlen finish, all sized for n_max: the
// fixed call's launches plus the plan kernel, plus w version 6 plan kernels, plus w blob-length kernels with the blob
// CRC.
extern "C" int rb200_container_planes_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                          uint32_t tolerance_ppm, uint32_t elem_bytes, const uint8_t* in, const uint64_t* d_n,
                                                          size_t n_max, uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!d_n || (reinterpret_cast<uintptr_t>(d_n) & 7) || n_max == 0) return RB200_E_ARG;
    return planes_encode(ctx, candidates, n_candidates, tolerance_ppm, elem_bytes, in, nullptr, n_max, d_n, nullptr, 0, chunk_syms, flags, out,
                         out_cap);
}

namespace {

// The plan kernel, then per plane the whole version 6 async decode (container_decode_async, unchanged) into a
// workspace -- plane 0 in place, the others after a fetch into staging -- and a record kernel, then the verdict and the
// interleave: 2 + 19 w launches, no copy, no synchronisation.
// base set (rb200_container_delta_decode_async): version 8's plan, and between the verdict (delta_verdict_kernel, which
// also writes the base's length) and the delta interleave the base's CRC and its check: 4 + 19 w launches.
// refs set (rb200_container_tensors_decode_async, with out_cap = n_max and no out): version 9's plan (tensors_open_kernel,
// with count; plane 0 after the directory), and between the verdict and the segmented interleave the directory's CRC
// and its check (tensors_check_kernel, which also writes d_lengths and the prefix): 4 + 19 w launches.  Arguments are
// checked by the callers.
int planes_decode(rb200_ctx* ctx, uint32_t w, const uint8_t* buf, size_t size, const uint8_t* base, const rb200_tensor_ref* refs, uint32_t count,
                  uint8_t* out, size_t out_cap, uint64_t* d_n_symbols)
{
    DeviceGuard g(ctx->device);
    const uint64_t table_end = container_planes_table_end(w, refs ? container_tensors_dir_bytes(count) : 0);
    // every plane of n <= out_cap bytes has n / w <= out_cap / w symbols, and fewer than 2^32
    const uint64_t stride = round16(std::min<uint64_t>(out_cap / w, 0xffffffffull));
    const uint64_t stage_cap = round16(std::max<uint64_t>(size > table_end ? size - table_end : 0, sizeof(ContainerHeader)));
    int rc = reserve(ctx, ctx->planes_out, std::max<uint64_t>(w * stride, 16));
    if (rc == RB200_OK) rc = reserve(ctx, ctx->planes_dec_stage, stage_cap);
    if (rc == RB200_OK && refs) rc = reserve(ctx, ctx->tensors_dec_prefix, (count + 1ull) * sizeof(uint64_t));
    if (rc != RB200_OK) return rc;
    uint8_t* planes = static_cast<uint8_t*>(ctx->planes_out.p);
    uint8_t* stage = static_cast<uint8_t*>(ctx->planes_dec_stage.p);
    PlanesWork* r = ctx->d_planes_dec;
    const TensorList list = {refs, count, static_cast<uint64_t*>(ctx->tensors_dec_prefix.p)};
    cudaStream_t s = ctx->stream;
    if (refs)
        tensors_open_kernel<<<1, 32, 0, s>>>(buf, size, w, count, r, ctx->d_tensors_dec);
    else if (base)
        delta_plan_kernel<<<1, 32, 0, s>>>(buf, size, w, r);
    else
        planes_plan_kernel<<<1, 32, 0, s>>>(buf, size, w, r);
    rc = check_launch(ctx, refs ? "tensors_open_kernel" : base ? "delta_plan_kernel" : "planes_plan_kernel");
    for (uint32_t p = 0; p < w && rc == RB200_OK; p++) {
        if (p) {
            planes_fetch_kernel<<<planes_grid(ctx), kPlanesThreads, 0, s>>>(buf, stage, stage_cap, p, r);
            rc = check_launch(ctx, "planes_fetch_kernel");
            if (rc == RB200_OK) rc = container_decode_async(ctx, kContainerVersionStored, stage, stage_cap, planes + p * stride, stride, nullptr);
        } else {
            rc = container_decode_async(ctx, kContainerVersionStored, buf + table_end, size > table_end ? size - table_end : 0, planes, stride,
                                        nullptr);
        }
        if (rc != RB200_OK) break;
        planes_record_kernel<<<1, 32, 0, s>>>(p, ctx->d_async[kContainerVersionStored - 1], r);
        rc = check_launch(ctx, "planes_record_kernel");
    }
    if (rc != RB200_OK) return rc;
    if (base) {
        DeltaWork* d = ctx->d_delta_dec;
        delta_verdict_kernel<<<1, 32, 0, s>>>(w, out_cap, d_n_symbols, r, ctx->d_status, d);
        rc = check_launch(ctx, "delta_verdict_kernel");
        if (rc == RB200_OK) rc = launch_crc(ctx, base, out_cap, &d->base_n, 0, &d->crc);
        if (rc != RB200_OK) return rc;
        delta_check_kernel<<<1, 32, 0, s>>>(buf, d, r, ctx->d_status);
        rc = check_launch(ctx, "delta_check_kernel");
    } else {
        planes_verdict_kernel<<<1, 32, 0, s>>>(w, out_cap, refs ? nullptr : d_n_symbols, r, ctx->d_status);
        rc = check_launch(ctx, "planes_verdict_kernel");
    }
    if (rc == RB200_OK && refs) {
        TensorsWork* t = ctx->d_tensors_dec;
        rc = launch_crc(ctx, buf + container_planes_table_end(w, 0), 8ull * count, &t->dir_len, 0, &t->crc);
        if (rc != RB200_OK) return rc;
        tensors_check_kernel<<<1, kTensorsPlanThreads, 0, s>>>(buf, w, count, refs, list.prefix, d_n_symbols, t, r, ctx->d_status);
        rc = check_launch(ctx, "tensors_check_kernel");
    }
    return rc == RB200_OK ? launch_interleave(ctx, w, planes, stride, base, refs ? &list : nullptr, out, r) : rc;
}

}  // namespace

extern "C" int rb200_container_planes_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size, uint8_t* out,
                                                   size_t out_cap, uint64_t* d_n_symbols)
{
    if (!container_planes_w_ok(elem_bytes) || !async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    return planes_decode(ctx, elem_bytes, buf, size, nullptr, nullptr, 0, out, out_cap, d_n_symbols);
}

// The version 7 encode of the difference from base: planes_encode with base set, 3 + w * (11 to 15) launches.
extern "C" int rb200_container_delta_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                                  uint32_t elem_bytes, const uint8_t* in, const uint8_t* base, size_t n, uint32_t chunk_syms,
                                                  uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!base || (reinterpret_cast<uintptr_t>(base) & 15)) return RB200_E_ARG;
    return planes_encode(ctx, candidates, n_candidates, tolerance_ppm, elem_bytes, in, base, n, nullptr, nullptr, 0, chunk_syms, flags, out,
                         out_cap);
}

// The version 7 decode applied to base: planes_decode with base set.  out == base applies the delta in place; any other
// overlap of the two, each taken as out_cap bytes long (the most the decode writes, and the most of base it reads), is
// refused, since the interleave's threads would read base bytes that others have already written.
extern "C" int rb200_container_delta_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size, const uint8_t* base,
                                                  uint8_t* out, size_t out_cap, uint64_t* d_n_symbols)
{
    if (!container_planes_w_ok(elem_bytes) || !async_args_ok(ctx, buf, out, d_n_symbols)) return RB200_E_ARG;
    if (!base || (reinterpret_cast<uintptr_t>(base) & 15)) return RB200_E_ARG;
    const uintptr_t o = reinterpret_cast<uintptr_t>(out), b = reinterpret_cast<uintptr_t>(base);
    if (o != b && o < b + out_cap && b < o + out_cap) return RB200_E_ARG;
    return planes_decode(ctx, elem_bytes, buf, size, base, nullptr, 0, out, out_cap, d_n_symbols);
}

// The version 7 varlen encode of a list's concatenated bytes, read through the list: planes_encode with refs set.
// Launches: the version 7 varlen call's (1 + 1 + w x (the version 6 varlen encode + 1) + 1), with tensors_plan_kernel
// and tensors_finish_kernel in place of its plan and finish kernels, plus one for the directory's CRC -- whatever T is.
extern "C" int rb200_container_tensors_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                                    uint32_t elem_bytes, const rb200_tensor_ref* d_refs, uint32_t count, size_t n_max,
                                                    uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap)
{
    if (!d_refs || !count || count > kContainerTensorsMax) return RB200_E_ARG;
    return planes_encode(ctx, candidates, n_candidates, tolerance_ppm, elem_bytes, nullptr, nullptr, n_max, nullptr, d_refs, count, chunk_syms,
                         flags, out, out_cap);
}

// The version 7 decode into a list's outputs: planes_decode with refs set, with n_max as the workspaces' bound.
// Launches: version 7's 2 + 19 w, plus the directory's CRC and tensors_check_kernel -- whatever T is.
extern "C" int rb200_container_tensors_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size,
                                                    const rb200_tensor_ref* d_refs, uint32_t count, size_t n_max, uint64_t* d_lengths)
{
    if (!container_planes_w_ok(elem_bytes) || !d_refs || !async_args_ok(ctx, buf, reinterpret_cast<const uint8_t*>(d_refs), d_lengths))
        return RB200_E_ARG;
    if (!count || count > kContainerTensorsMax || n_max == 0) return RB200_E_ARG;
    return planes_decode(ctx, elem_bytes, buf, size, nullptr, d_refs, count, nullptr, n_max, d_lengths);
}

extern "C" int rb200_container_blocks_auto_costs(rb200_ctx* ctx, uint64_t* costs, uint32_t n)
{
    if (!ctx || !costs || n > kMaxCandidates) return RB200_E_ARG;
    DeviceGuard g(ctx->device);
    RB_CUDA(ctx, cudaMemcpyAsync(costs, ctx->d_blocks_choice->choice.costs, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
    RB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RB200_OK;
}

// ---------------------------------------------------------------------------
// multi-GPU: gathering the shards' blobs over NCCL
// ---------------------------------------------------------------------------
#include "gather_nccl.cuh"

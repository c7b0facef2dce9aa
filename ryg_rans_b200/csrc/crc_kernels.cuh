// crc_kernels.cuh -- zlib's CRC-32 (IEEE polynomial, reflected, init and xor-out ~0) on sm_90a, and the GF(2)
// algebra that joins CRCs of adjacent pieces (zlib's crc32_combine), shared by the host and the kernels.
//
// The CRC register after a message is linear in (initial register, message): with R(c, D) the register after D
// starting from c,   R(c, A || B) = R(R(c, A), B)   and   R(c, D) = shift(c, |D|) ^ R(0, D),
// where shift(c, len) multiplies c by x^(8 len) mod P.  zlib's crc32(D, crc_in) = ~R(~crc_in, D).  So the kernel
// cuts the buffer into one contiguous segment per thread, computes each segment's R(0, D_t) on its own, shifts it
// by the bytes that follow the segment and XORs everything together; one thread then applies crc_in and the
// xor-out.  Multiplying by x^(8 len) takes one product per set bit of len from the table of x^(8 2^k), k < 64,
// so lengths past 2^32 cost nothing extra.
//
// Per-segment method: slicing-by-4 over 32-bit words with the four 256-entry tables in shared memory, each entry
// replicated 32 times with lane l reading replica l.  The replica of entry i for lane l sits at word i * 32 + l,
// i.e. always in bank l, so the random table indices of a warp never conflict (DESIGN.md section 4 has the
// alternatives and the numbers).  The 128 KiB of tables leave one 1024-thread CTA per SM.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "container_format.h"
#include "device_utils.cuh"

namespace rb200 {

constexpr uint32_t kCrcPoly = 0xEDB88320u;   // reflected IEEE 802.3 polynomial
constexpr uint32_t kCrcOne = 0x80000000u;    // x^0 in the reflected representation

// a * b mod P (reflected): zlib's multmodp, with a fixed trip count so that a == 0 is fine
__host__ __device__ constexpr uint32_t crc32_mulmod(uint32_t a, uint32_t b)
{
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        p ^= b & (0u - ((a >> (31 - i)) & 1u));
        b = (b >> 1) ^ (kCrcPoly & (0u - (b & 1u)));
    }
    return p;
}

struct CrcPowers {
    uint32_t p[64];   // x^(8 * 2^k) mod P
};

__host__ __device__ constexpr CrcPowers crc32_make_powers()
{
    CrcPowers t{};
    uint32_t x = kCrcOne >> 8;                                  // x^8
    for (int k = 0; k < 64; k++) {
        t.p[k] = x;
        x = crc32_mulmod(x, x);
    }
    return t;
}

constexpr CrcPowers kCrcPowersHost = crc32_make_powers();
__constant__ CrcPowers kCrcPowersDev = crc32_make_powers();

__host__ __device__ inline uint32_t crc32_power(int k)
{
#ifdef __CUDA_ARCH__
    return kCrcPowersDev.p[k];
#else
    return kCrcPowersHost.p[k];
#endif
}

// c * x^(8 len) mod P: the register c followed by len zero bytes
__host__ __device__ inline uint32_t crc32_shift(uint32_t c, uint64_t len)
{
    for (int k = 0; len; k++, len >>= 1)
        if (len & 1) c = crc32_mulmod(c, crc32_power(k));
    return c;
}

// zlib's crc32_combine: crc32(A || B) from crc32(A), crc32(B) and |B|
__host__ __device__ inline uint32_t crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b)
{
    return crc32_shift(crc_a, len_b) ^ crc_b;
}

// zlib's crc32(D, crc_in) from acc = R(0, D) and |D|
__host__ __device__ inline uint32_t crc32_finish(uint32_t crc_in, uint64_t len, uint32_t acc)
{
    return ~(crc32_shift(~crc_in, len) ^ acc);
}

// One CRC result: what the kernel computed and over how many bytes (the host pipeline joins slices with it).
struct CrcSlot {
    uint64_t len;
    uint32_t crc;
    uint32_t pad;
};

// Accumulator and CTA counter of crc32_kernel.  Zero between launches: the last CTA resets them.
struct CrcWork {
    uint32_t acc;
    uint32_t done;
};

constexpr int kCrcThreads = 1024;
constexpr int kCrcTableWords = 4 * 256 * 32;
constexpr size_t kCrcSmemBytes = (kCrcTableWords + 64) * sizeof(uint32_t);

namespace crc_detail {

// R(0, D) for the bytes of one thread's segment, bit by bit (the finalise kernel's 34-byte pieces)
__device__ __forceinline__ uint32_t raw_bytes_bitwise(const uint8_t* p, uint32_t len)
{
    uint32_t c = 0;
    for (uint32_t i = 0; i < len; i++) {
        c ^= p[i];
#pragma unroll
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (kCrcPoly & (0u - (c & 1u)));
    }
    return c;
}

// c * x^(8 len) with the powers in shared memory (lanes index it divergently; __constant__ would serialise)
__device__ __forceinline__ uint32_t shift_smem(uint32_t c, uint64_t len, const uint32_t* pow)
{
    for (int k = 0; len; k++, len >>= 1)
        if (len & 1) c = crc32_mulmod(c, pow[k]);
    return c;
}

// x^(8 len) mod P by the whole warp: lane l takes bits l and l + 32 of len, then a butterfly of products
__device__ __forceinline__ uint32_t x8pow_warp(uint64_t len)
{
    const int l = threadIdx.x & 31;
    uint32_t f = ((len >> l) & 1) ? kCrcPowersDev.p[l] : kCrcOne;
    if ((len >> (l + 32)) & 1) f = crc32_mulmod(f, kCrcPowersDev.p[l + 32]);
#pragma unroll
    for (int m = 16; m; m >>= 1) f = crc32_mulmod(f, __shfl_xor_sync(0xffffffffu, f, m));
    return f;
}

// crc32_finish by a whole warp (every lane returns the result)
__device__ __forceinline__ uint32_t finish_warp(uint32_t crc_in, uint64_t len, uint32_t acc)
{
    return ~(crc32_mulmod(~crc_in, x8pow_warp(len)) ^ acc);
}

__device__ __forceinline__ uint32_t step_word(uint32_t c, uint32_t w, uint32_t tab)
{
    const uint32_t v = c ^ w;
    // table j (entry = byte followed by j zero bytes) at tab + j * 32 KiB; entry i of this lane at + i * 128
    return lds_u32_ro(tab + 3 * 32768 + ((v << 7) & 0x7f80u)) ^ lds_u32_ro(tab + 2 * 32768 + ((v >> 1) & 0x7f80u)) ^
           lds_u32_ro(tab + 1 * 32768 + ((v >> 9) & 0x7f80u)) ^ lds_u32_ro(tab + ((v >> 17) & 0x7f80u));
}

__device__ __forceinline__ uint32_t step_vec(uint32_t c, uint4 v, uint32_t tab)
{
    c = step_word(c, v.x, tab);
    c = step_word(c, v.y, tab);
    c = step_word(c, v.z, tab);
    return step_word(c, v.w, tab);
}

__device__ __forceinline__ uint32_t step_byte(uint32_t c, uint32_t b, uint32_t tab)
{
    return lds_u32_ro(tab + (((c ^ b) & 0xffu) << 7)) ^ (c >> 8);
}

}  // namespace crc_detail

// zlib crc32(data[0, n), crc_in) -> slot.  With n_dev set the length is min(*n_dev, n): a length the device wrote
// (a directory's last entry), bounded by the buffer.  With off_dev set the bytes start *off_dev bytes after data (a
// position the device wrote), and n still bounds them from data.  Any n and any alignment of data.  work must be zero
// (it is left zero).
__global__ void __launch_bounds__(kCrcThreads, 1)
    crc32_kernel(const uint8_t* __restrict__ data, uint64_t n, const uint64_t* __restrict__ n_dev, const uint64_t* __restrict__ off_dev,
                 uint32_t crc_in, CrcWork* work, CrcSlot* slot)
{
    using namespace crc_detail;
    extern __shared__ uint4 crc_smem_v[];
    uint32_t* tabs = reinterpret_cast<uint32_t*>(crc_smem_v);
    uint32_t* pow = tabs + kCrcTableWords;
    {   // entry i of table j: R(0, byte i then j zero bytes); 32 replicas, 128 contiguous bytes
        const uint32_t j = threadIdx.x >> 8, i = threadIdx.x & 255;
        uint32_t c = i;
        for (uint32_t k = 0; k < 8 * (j + 1); k++) c = (c >> 1) ^ (kCrcPoly & (0u - (c & 1u)));
        uint4* dst = reinterpret_cast<uint4*>(tabs + (j * 256 + i) * 32);
#pragma unroll
        for (int r = 0; r < 8; r++) dst[r] = make_uint4(c, c, c, c);
        if (threadIdx.x < 64) pow[threadIdx.x] = kCrcPowersDev.p[threadIdx.x];
    }
    __syncthreads();
    if (off_dev) {
        const uint64_t skip = *off_dev < n ? *off_dev : n;
        data += skip;
        n -= skip;
    }
    if (n_dev && *n_dev < n) n = *n_dev;

    // thread t owns span bytes [t L, (t + 1) L) of the 16-aligned span that starts a0 bytes before data
    const uint64_t a0 = reinterpret_cast<uintptr_t>(data) & 15;
    const uint8_t* base = data - a0;
    const uint64_t span = a0 + n;
    const uint64_t threads = static_cast<uint64_t>(gridDim.x) * kCrcThreads;
    uint64_t L = (span + threads - 1) / threads;
    L = (L + 31) & ~31ull;
    const uint64_t t = static_cast<uint64_t>(blockIdx.x) * kCrcThreads + threadIdx.x;
    uint64_t p = t * L;
    const uint64_t e = p + L < span ? p + L : span;
    if (p < a0) p = a0;
    uint32_t contrib = 0;
    if (p < e) {
        const uint32_t tab = smem_addr(tabs) + (threadIdx.x & 31) * 4;
        uint32_t c = 0;
        for (; p < e && (p & 15); p++) c = step_byte(c, base[p], tab);              // unaligned head (thread 0 only)
        const uint4* v = reinterpret_cast<const uint4*>(base + p);
        const uint64_t pairs = (e - p) >> 5;
        if (pairs) {
            uint4 x0 = __ldg(v), x1 = __ldg(v + 1);
            for (uint64_t k = 1; k < pairs; k++) {
                const uint4 y0 = __ldg(v + 2 * k), y1 = __ldg(v + 2 * k + 1);
                c = step_vec(step_vec(c, x0, tab), x1, tab);
                x0 = y0;
                x1 = y1;
            }
            c = step_vec(step_vec(c, x0, tab), x1, tab);
            p += pairs << 5;
        }
        if (e - p >= 16) {
            c = step_vec(c, __ldg(reinterpret_cast<const uint4*>(base + p)), tab);
            p += 16;
        }
        for (; p < e; p++) c = step_byte(c, base[p], tab);                          // ragged tail (last thread only)
        contrib = shift_smem(c, span - e, pow);
    }
    contrib = __reduce_xor_sync(0xffffffffu, contrib);
    if ((threadIdx.x & 31) == 0 && contrib) {
        atomicXor(&work->acc, contrib);
        __threadfence();
    }
    __syncthreads();
    __shared__ uint32_t last;
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&work->done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || threadIdx.x >= 32) return;
    __threadfence();
    const uint32_t acc = threadIdx.x == 0 ? atomicExch(&work->acc, 0u) : 0u;
    const uint32_t crc = finish_warp(crc_in, n, __shfl_sync(0xffffffffu, acc, 0));
    if (threadIdx.x == 0) {
        work->done = 0;
        slot->len = n;
        slot->crc = crc;
    }
}

inline void configure_crc_kernels()
{
    cudaFuncSetAttribute(crc32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCrcSmemBytes));
}

// CTAs for a length known on the host: about 256 bytes per thread at least, at most one CTA per SM
inline uint32_t crc32_grid(uint32_t sms, uint64_t n)
{
    const uint64_t want = (n + kCrcThreads * 256ull - 1) / (kCrcThreads * 256ull);
    return want < 1 ? 1 : (want > sms ? sms : static_cast<uint32_t>(want));
}

// The last step of a device-memory container encode, one warp.  The encoder has written the directory at
// out + dir_off and the blob at out + blob_off.  crc32_kernel has put into slots[0] the CRC of out[head, dir_end),
// where head is what this kernel writes in front of it: header and model `freqs` (version 1, head = 1088: the model
// comes from the rb200_model and is CRC'd here) or the header alone (version 2, freqs == nullptr, head = 64: the
// block encoder wrote the models in place, so slots[0] covers model and directory); with RB200_CONTAINER_CRC_BLOB
// the blob's CRC is in slots[1].  Reads blob_bytes from the directory, completes the header (h arrives with
// blob_bytes and both CRCs zero), and writes the head and the zero pad in front of the blob -- only when the status
// word is clear (an encoder error leaves the buffer as it is) and the blob fits out_cap (else it flags kStatSpace).
// GEOM (rb200_container_model_encode_varlen_async, version 1): n_symbols, n_chunks and the blob offset from the record
// (VarlenGeom); h arrives with coder, scale_bits, chunk_syms and flags.  Writes nothing when geom->go == 0.
// CHOSEN (rb200_container_model_encode_auto_async, version 1): coder and scale_bits from the choice record.
// BITMAP (rb200_container_stored_encode_async, version 6): slots[0] covers out[head, blob_off) -- directory, the pad
// after it and the stored-chunk bitmap, all written by then -- so meta_crc spans everything before the blob.
template <bool GEOM, bool CHOSEN, bool BITMAP = false>
__device__ __forceinline__ void container_finish(uint8_t* out, ContainerHeader h, uint64_t dir_off, uint64_t blob_off, uint64_t out_cap,
                                                 const uint32_t* __restrict__ freqs, const CrcSlot* __restrict__ slots, uint32_t* status,
                                                 const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice)
{
    if (GEOM) {
        if (!geom->go) return;
        h.n_symbols = geom->n;
        h.n_chunks = geom->n_chunks;
        dir_off = kContainerDirOffset;
        blob_off = geom->blob_off;
    }
    if (CHOSEN) {
        h.coder = static_cast<uint8_t>(choice->coder);
        h.scale_bits = static_cast<uint8_t>(choice->scale_bits);
    }
    using namespace crc_detail;
    __shared__ uint4 sbuf_v[kContainerDirOffset / 16];
    uint32_t* sbuf = reinterpret_cast<uint32_t*>(sbuf_v);
    const uint32_t lane = threadIdx.x;
    if (*status) return;                              // the encoder has flagged an error: rb200_sync reports it
    const uint64_t blob_bytes = reinterpret_cast<const uint64_t*>(out + dir_off)[h.n_chunks];
    if (blob_bytes > out_cap - blob_off) {            // the encoder has flagged it; leave the buffer as it is
        if (lane == 0) atomicOr(status, kStatSpace);
        return;
    }
    const uint32_t head = freqs ? static_cast<uint32_t>(kContainerDirOffset) : static_cast<uint32_t>(sizeof(ContainerHeader));
    if (lane == 0) {
        ContainerHeader* sh = reinterpret_cast<ContainerHeader*>(sbuf);
        *sh = h;
        sh->blob_bytes = blob_bytes;
    }
    if (freqs)
        for (uint32_t i = lane; i < 256; i += 32) sbuf[16 + i] = freqs[i];
    __syncwarp();
    // CRC of the head: head / 32 bytes per lane (34 or 2), each shifted past the bytes after it
    const uint32_t piece = head / 32;
    uint32_t c = raw_bytes_bitwise(reinterpret_cast<const uint8_t*>(sbuf) + lane * piece, piece);
    c = __reduce_xor_sync(0xffffffffu, crc32_shift(c, head - piece * (lane + 1)));
    const uint32_t head_crc = finish_warp(0, head, c);
    const uint64_t dir_end = dir_off + (h.n_chunks + 1) * sizeof(uint64_t);
    const uint64_t meta_end = BITMAP ? blob_off : dir_end;
    const uint32_t meta = crc32_mulmod(head_crc, x8pow_warp(meta_end - head)) ^ slots[0].crc;     // crc32_combine
    __syncwarp();
    if (lane == 0) {
        sbuf[offsetof(ContainerHeader, meta_crc) / 4] = meta;
        sbuf[offsetof(ContainerHeader, blob_crc) / 4] = (h.flags & RB200_CONTAINER_CRC_BLOB) ? slots[1].crc : 0u;
    }
    __syncwarp();
    uint4* dst = reinterpret_cast<uint4*>(out);
    for (uint32_t i = lane; i < head / 16; i += 32) dst[i] = sbuf_v[i];
    if (!BITMAP && lane == 0 && blob_off > dir_end) *reinterpret_cast<uint64_t*>(out + dir_end) = 0;   // the 8-byte pad
}

template <bool GEOM = false, bool CHOSEN = false>
__global__ void __launch_bounds__(32)
    container_finish_kernel(uint8_t* out, ContainerHeader h, uint64_t dir_off, uint64_t blob_off, uint64_t out_cap,
                            const uint32_t* __restrict__ freqs, const CrcSlot* __restrict__ slots, uint32_t* status,
                            const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice)
{
    container_finish<GEOM, CHOSEN>(out, h, dir_off, blob_off, out_cap, freqs, slots, status, geom, choice);
}

// The per-block header kernel of rb200_container_blocks_model_encode_auto_async (versions 2-4): version, coder and
// scale_bits from the choice record r; the layout of the three versions is the same, so h carries the rest.
// GEOM (rb200_container_blocks_model_encode_varlen_async): n_blocks, n_symbols, n_chunks, the directory and the blob
// offset from the record (BlocksVarlenGeom); h arrives with block_size, chunk_syms and flags.  Writes nothing when
// geom->v.go == 0.
template <bool GEOM>
__global__ void __launch_bounds__(32)
    container_blocks_finish_kernel(uint8_t* out, ContainerHeader h, uint64_t dir_off, uint64_t blob_off, uint64_t out_cap,
                                   const CrcSlot* __restrict__ slots, uint32_t* status, const BlocksChoice* __restrict__ r,
                                   const BlocksVarlenGeom* __restrict__ geom)
{
    if (GEOM && !geom->v.go) return;
    h.version = static_cast<uint16_t>(r->version);
    if (GEOM) {
        h.n_blocks = geom->n_blocks;
        h.n_symbols = geom->v.n;
        h.n_chunks = geom->v.n_chunks;
        dir_off = geom->v.dir_off;
        blob_off = geom->v.blob_off;
    }
    container_finish<false, true>(out, h, dir_off, blob_off, out_cap, nullptr, slots, status, nullptr, &r->choice);
}

// The header kernel of rb200_container_blocks_stored_encode_async: container_blocks_finish_kernel's with version 5 (coder
// and scale_bits from the record)
__global__ void __launch_bounds__(32)
    container_blocks_stored_finish_kernel(uint8_t* out, ContainerHeader h, uint64_t dir_off, uint64_t blob_off, uint64_t out_cap,
                                          const CrcSlot* __restrict__ slots, uint32_t* status, const BlocksChoice* __restrict__ r)
{
    h.version = kContainerVersionBlocksStored;
    container_finish<false, true>(out, h, dir_off, blob_off, out_cap, nullptr, slots, status, nullptr, &r->choice);
}

// The header kernel of rb200_container_stored_encode_async: container_finish_kernel's CHOSEN instance with version 6,
// meta_crc over the bitmap as well (BITMAP), and the model section from freqs
__global__ void __launch_bounds__(32)
    container_stored_finish_kernel(uint8_t* out, ContainerHeader h, uint64_t blob_off, uint64_t out_cap, const uint32_t* __restrict__ freqs,
                                   const CrcSlot* __restrict__ slots, uint32_t* status, const CoderChoice* __restrict__ choice)
{
    h.version = kContainerVersionStored;
    container_finish<false, true, true>(out, h, kContainerDirOffset, blob_off, out_cap, freqs, slots, status, nullptr, choice);
}

// The GEOM header kernels of the two device-size stored encodes: n_symbols, n_chunks (version 5: n_blocks and the
// directory's place too) and the blob offset from the record; h arrives with the bound's geometry, chunk_syms and flags.
// Write nothing when the plan failed.
__global__ void __launch_bounds__(32)
    container_blocks_stored_finish_varlen_kernel(uint8_t* out, ContainerHeader h, uint64_t out_cap, const CrcSlot* __restrict__ slots,
                                                 uint32_t* status, const BlocksChoice* __restrict__ r, const BlocksVarlenGeom* __restrict__ geom)
{
    if (!geom->v.go) return;
    h.version = kContainerVersionBlocksStored;
    h.n_blocks = geom->n_blocks;
    h.n_symbols = geom->v.n;
    h.n_chunks = geom->v.n_chunks;
    container_finish<false, true>(out, h, geom->v.dir_off, geom->v.blob_off, out_cap, nullptr, slots, status, nullptr, &r->choice);
}

__global__ void __launch_bounds__(32)
    container_stored_finish_varlen_kernel(uint8_t* out, ContainerHeader h, uint64_t out_cap, const uint32_t* __restrict__ freqs,
                                          const CrcSlot* __restrict__ slots, uint32_t* status, const CoderChoice* __restrict__ choice,
                                          const StoredVarlenGeom* __restrict__ geom)
{
    if (!geom->v.go) return;
    h.version = kContainerVersionStored;
    h.n_symbols = geom->v.n;
    h.n_chunks = geom->v.n_chunks;
    container_finish<false, true, true>(out, h, kContainerDirOffset, geom->v.blob_off, out_cap, freqs, slots, status, nullptr, choice);
}

}  // namespace rb200

// planes_kernels.cuh -- the byte-plane container (version 7): rb200_container_planes_encode_async and
// rb200_container_planes_decode_async (rans_b200.cu).  Every plane is a version 6 container written and read by the
// version 6 calls' own stages; the kernels here only move bytes between the element layout and the planes, place the
// planes and write or check the version 7 header and table.
//
// Encode, in stream order on the context's stream:
//   planes_split_kernel<W>      the n input bytes into W planes of m = n / W bytes, at a stride of round16(m), in a
//                               context workspace: 16 elements per thread, W 16-byte loads, the byte transpose in
//                               registers (PRMT), one 16-byte store per plane
//   plane 0's version 6 encode  in place, at 64 + 16 W
//   planes_place_kernel(0)      plane 0's verdict (the status word is clear: its header was written) and table entry
//   for p = 1 .. W-1: plane p's version 6 encode into a staging area, then planes_place_kernel(p): its verdict, its size
//                               from its header, its offset from entry p - 1, the copy to there and its table entry
//   planes_finish_kernel        the version 7 header and meta_crc, only when every plane was placed
// Encode with the length in device memory (rb200_container_planes_encode_varlen_async), launch shapes and workspaces
// sized for n_max:
//   planes_varlen_plan_kernel   *d_n checked, n and the plane length m into the context's PlanesVarlenGeom
//   planes_split_varlen_kernel<W>  the split body with m from the record, at the stride round16(n_max / W)
//   per plane: version 6's varlen encode with &geom->m as its length, then planes_place_kernel, as above
//   planes_finish_varlen_kernel the finish body with n from the record
// Decode:
//   planes_plan_kernel          the header (its W must be the caller's), the table, every plane's header and meta_crc,
//                               into the call's record
//   plane 0's version 6 decode  in place from 64 + 16 W, into plane 0 of a workspace; planes_record_kernel(0)
//   for p = 1 .. W-1: planes_fetch_kernel(p) copies [offset, offset + size) into staging when the record passed (else a
//                               zero header, which version 6's plan rejects), plane p's version 6 decode from there,
//                               planes_record_kernel(p)
//   planes_verdict_kernel       *d_n_symbols, then kStatStream / kStatSpace or the record's go
//   planes_interleave_kernel<W> the planes into out, only when go is set
// The delta container (version 8, rb200_container_delta_encode_async / _decode_async) runs the same host bodies with a
// base tensor; its kernels are thin wrappers around the bodies above, or the version 7 kernels themselves:
//   encode: delta_split_kernel<W> (the split of d, the zigzag difference from base), crc32_kernel over base into the
//           call's DeltaWork, every plane as above, delta_finish_kernel (the finish with version 8, reserved = the CRC)
//   decode: delta_plan_kernel (the plan with version 8's rules), every plane as above, delta_verdict_kernel (the verdict,
//           then the base's length: n when go, else 0), crc32_kernel over that many bytes of base, delta_check_kernel
//           (a CRC other than the header's: kStatBase, go cleared), delta_interleave_kernel<W> (d and base into out)
// The tensor-list container (version 9, rb200_container_tensors_encode_async / _decode_async) runs the same host bodies
// with a list of rb200_tensor_ref in device memory in place of in / out:
//   encode: tensors_plan_kernel (one CTA: the list checked, the exclusive prefix of its element counts into a context
//           workspace, PlanesVarlenGeom {n, m} -- {0, UINT64_MAX} for a bad list, which every plane's version 6 varlen
//           plan refuses -- and, only for a good list, the directory into out), tensors_split_kernel<W> (the segmented
//           split), crc32_kernel over the directory into the call's TensorsWork, every plane as the varlen encode's,
//           tensors_finish_kernel (the finish with version 9, n_blocks = T, reserved = the directory's CRC)
//   decode: tensors_open_kernel (the plan with version 9's rules and T == count), every plane as above,
//           planes_verdict_kernel with n_max for out_cap, crc32_kernel over the directory (its length 8 T from the
//           plan, 0 for a rejected header), tensors_check_kernel (the CRC against reserved, the directory's rules and
//           every length against its ref's capacity, else go cleared; then the directory's prefix into a workspace),
//           tensors_interleave_kernel<W> (the segmented inverse scatter into the refs)
#pragma once
#include "container_decode.cuh"
#include "container_format.h"
#include "crc_kernels.cuh"

namespace rb200 {

// The call-private record of a byte-plane call (one for the encode, one for the decode): the outcome of the call's own
// checks, so that status bits left by earlier calls that were not synchronised do not change what it writes.
struct PlanesWork {
    PlaneEntry table[8];        // decode: the table, when ok
    uint64_t n;                 // decode: the header's n, when ok
    uint32_t ok;                // decode: the header, the table, every plane's header and meta_crc passed
    uint32_t go;                // decode: every check passed; the interleave runs
    uint32_t plane_go[8];       // encode: plane p was written and placed; decode: plane p's version 6 verdict passed
};

// The length of rb200_container_planes_encode_varlen_async, in device memory: written by planes_varlen_plan_kernel from
// *d_n at every run, read by the split, by every plane's version 6 varlen encode (m is its length) and by the finish.
// For a bad *d_n, n is 0 and m is UINT64_MAX, above every plane's bound: version 6's plan then refuses it (kStatArg)
// and writes nothing, so no plane is placed and no header written.
struct PlanesVarlenGeom {
    uint64_t n;                 // input bytes, 1 <= n <= n_max and a multiple of w; 0 for a bad *d_n
    uint64_t m;                 // symbols per plane, n / w; UINT64_MAX for a bad *d_n
};

// The base tensor's CRC of a delta call (one for the encode, one for the decode): crc32_kernel's result, and on decode
// the length it covers (the header's n once every check passed, else 0: the base is then not read).
struct DeltaWork {
    CrcSlot crc;
    uint64_t base_n;
};

// The directory's CRC of a tensor-list call (one for the encode, one for the decode): crc32_kernel's result, and on
// decode the length it covers (8 T once the header passed, else 0: the directory is then not read).
struct TensorsWork {
    CrcSlot crc;
    uint64_t dir_len;
};

constexpr uint32_t kPlanesThreads = 256;
constexpr uint32_t kPlanesCtasPerSm = 8;

// 16 elements of W bytes in x (4 W words, element e at bytes e W .. e W + W - 1) -> y[4 k + j] = byte k of elements
// 4 j .. 4 j + 3: three PRMTs per output word, every index a constant once unrolled
template <int W>
__device__ __forceinline__ void planes_transpose(const uint32_t (&x)[4 * W], uint32_t (&y)[4 * W])
{
#pragma unroll
    for (int k = 0; k < W; k++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int b0 = 4 * j * W + k, b1 = b0 + W, b2 = b1 + W, b3 = b2 + W;
            const uint32_t lo = __byte_perm(x[b0 >> 2], x[b1 >> 2], (b0 & 3) | ((b1 & 3) + 4) << 4);
            const uint32_t hi = __byte_perm(x[b2 >> 2], x[b3 >> 2], (b2 & 3) | ((b3 & 3) + 4) << 4);
            y[4 * k + j] = __byte_perm(lo, hi, 0x5410);
        }
}

// the inverse: byte b of x is byte b % W of element b / W, which is byte (b / W) % 4 of y[4 (b % W) + b / W / 4]
template <int W>
__device__ __forceinline__ void planes_untranspose(const uint32_t (&y)[4 * W], uint32_t (&x)[4 * W])
{
#pragma unroll
    for (int t = 0; t < 4 * W; t++) {
        int word[4], sel[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int b = 4 * t + i, e = b / W;
            word[i] = 4 * (b % W) + (e >> 2);
            sel[i] = e & 3;
        }
        const uint32_t lo = __byte_perm(y[word[0]], y[word[1]], sel[0] | (sel[1] + 4) << 4);
        const uint32_t hi = __byte_perm(y[word[2]], y[word[3]], sel[2] | (sel[3] + 4) << 4);
        x[t] = __byte_perm(lo, hi, 0x5410);
    }
}

// The version 8 transform of one element of W bytes (the low 8 W bits of x and b): d = zigzag((x - b) mod 2^(8 W)), and
// its inverse x = b + unzigzag(d).  For the ragged ends; the groups of 16 take the lane forms below.
template <int W>
__device__ __forceinline__ uint64_t delta_zigzag(uint64_t x, uint64_t b)
{
    const uint64_t s = (x - b) << (64 - 8 * W);                      // the difference in the top 8 W bits
    return ((s << 1) ^ static_cast<uint64_t>(static_cast<int64_t>(s) >> 63)) >> (64 - 8 * W);
}
template <int W>
__device__ __forceinline__ uint64_t delta_unzigzag(uint64_t d, uint64_t b)
{
    const uint64_t x = b + ((d >> 1) ^ (0ull - (d & 1)));
    return W == 8 ? x : x & ((1ull << (8 * W)) - 1);
}

// The transform on 4 W words of element data (element e at bytes e W .. e W + W - 1), in place: 16-bit lanes of a word
// for W = 2, the word for W = 4, pairs of words for W = 8.  forward: x -> d from x and b; inverse: d -> x from d and b.
template <int W>
__device__ __forceinline__ void delta_forward(uint32_t (&x)[4 * W], const uint32_t (&b)[4 * W])
{
#pragma unroll
    for (int i = 0; i < 4 * W; i += W == 8 ? 2 : 1) {
        if (W == 2) {
            const uint32_t s = __vsub2(x[i], b[i]);
            x[i] = ((s << 1) & 0xfffefffeu) ^ (((s >> 15) & 0x00010001u) * 0xffffu);
        } else if (W == 4) {
            const uint32_t s = x[i] - b[i];
            x[i] = (s << 1) ^ static_cast<uint32_t>(static_cast<int32_t>(s) >> 31);
        } else {
            const uint64_t s = (static_cast<uint64_t>(x[i + 1]) << 32 | x[i]) - (static_cast<uint64_t>(b[i + 1]) << 32 | b[i]);
            const uint64_t d = (s << 1) ^ static_cast<uint64_t>(static_cast<int64_t>(s) >> 63);
            x[i] = static_cast<uint32_t>(d);
            x[i + 1] = static_cast<uint32_t>(d >> 32);
        }
    }
}
template <int W>
__device__ __forceinline__ void delta_inverse(uint32_t (&x)[4 * W], const uint32_t (&b)[4 * W])
{
#pragma unroll
    for (int i = 0; i < 4 * W; i += W == 8 ? 2 : 1) {
        if (W == 2) {
            x[i] = __vadd2(b[i], ((x[i] >> 1) & 0x7fff7fffu) ^ ((x[i] & 0x00010001u) * 0xffffu));
        } else if (W == 4) {
            x[i] = b[i] + ((x[i] >> 1) ^ (0u - (x[i] & 1u)));
        } else {
            const uint64_t d = static_cast<uint64_t>(x[i + 1]) << 32 | x[i];
            const uint64_t v = (static_cast<uint64_t>(b[i + 1]) << 32 | b[i]) + ((d >> 1) ^ (0ull - (d & 1)));
            x[i] = static_cast<uint32_t>(v);
            x[i + 1] = static_cast<uint32_t>(v >> 32);
        }
    }
}

// W 16-byte loads of 16 elements into 4 W words
template <int W>
__device__ __forceinline__ void planes_load_group(const uint4* src, uint32_t (&x)[4 * W])
{
#pragma unroll
    for (int i = 0; i < W; i++) {
        const uint4 v = __ldcs(src + i);
        x[4 * i] = v.x;
        x[4 * i + 1] = v.y;
        x[4 * i + 2] = v.z;
        x[4 * i + 3] = v.w;
    }
}

// in (m elements of W bytes, 16-byte aligned) -> plane k at planes + k * stride (stride a multiple of 16).  Grid-stride
// over groups of 16 elements; the ragged end (fewer than 16 elements) a byte per thread.  DELTA (version 8): the planes
// of d, the difference of in from base (16-byte aligned too), W more loads per group; the ragged end an element per
// thread.
template <int W, bool DELTA = false>
__device__ __forceinline__ void planes_split(const uint8_t* __restrict__ in, const uint8_t* __restrict__ base, uint64_t m,
                                             uint8_t* __restrict__ planes, uint64_t stride)
{
    const uint64_t groups = m / 16, step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (uint64_t g = tid; g < groups; g += step) {
        uint32_t x[4 * W], y[4 * W];
        planes_load_group<W>(reinterpret_cast<const uint4*>(in) + g * W, x);
        if (DELTA) {
            uint32_t b[4 * W];
            planes_load_group<W>(reinterpret_cast<const uint4*>(base) + g * W, b);
            delta_forward<W>(x, b);
        }
        planes_transpose<W>(x, y);
#pragma unroll
        for (int k = 0; k < W; k++)
            *reinterpret_cast<uint4*>(planes + k * stride + g * 16) = make_uint4(y[4 * k], y[4 * k + 1], y[4 * k + 2], y[4 * k + 3]);
    }
    const uint64_t tail = groups * 16;
    if (DELTA) {
        if (tid < m - tail) {
            const uint64_t e = tail + tid;
            uint64_t x = 0, b = 0;
#pragma unroll
            for (int k = 0; k < W; k++) {
                x |= static_cast<uint64_t>(in[e * W + k]) << (8 * k);
                b |= static_cast<uint64_t>(base[e * W + k]) << (8 * k);
            }
            const uint64_t d = delta_zigzag<W>(x, b);
#pragma unroll
            for (int k = 0; k < W; k++) planes[k * stride + e] = static_cast<uint8_t>(d >> (8 * k));
        }
    } else if (tid < (m - tail) * W) {
        const uint64_t e = tail + tid / W, k = tid % W;
        planes[k * stride + e] = in[e * W + k];
    }
}

template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    planes_split_kernel(const uint8_t* __restrict__ in, uint64_t m, uint8_t* __restrict__ planes, uint64_t stride)
{
    planes_split<W>(in, nullptr, m, planes, stride);
}

// The split of the varlen encode: m from the record, nothing for a bad length.  The grid is the fixed call's, so a
// short length costs no extra CTAs.
template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    planes_split_varlen_kernel(const uint8_t* __restrict__ in, const PlanesVarlenGeom* __restrict__ g, uint8_t* __restrict__ planes,
                               uint64_t stride)
{
    if (g->n == 0) return;
    planes_split<W>(in, nullptr, g->m, planes, stride);
}

// The split of the delta encode: the planes of d = zigzag(in - base)
template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    delta_split_kernel(const uint8_t* __restrict__ in, const uint8_t* __restrict__ base, uint64_t m, uint8_t* __restrict__ planes,
                       uint64_t stride)
{
    planes_split<W, true>(in, base, m, planes, stride);
}

// The inverse, from the decode workspace into out: n from the record, and nothing unless every check passed.  DELTA
// (version 8): the planes hold d, and out = base + unzigzag(d), base 16-byte aligned; each thread reads exactly the base
// bytes it writes to out, so out == base (the delta applied in place) is correct, and neither pointer is __restrict__.
template <int W, bool DELTA>
__device__ __forceinline__ void planes_interleave(const uint8_t* __restrict__ planes, uint64_t stride, const uint8_t* base, uint8_t* out,
                                                  const PlanesWork* __restrict__ r)
{
    if (!r->go) return;
    const uint64_t m = r->n / W, groups = m / 16, step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (uint64_t g = tid; g < groups; g += step) {
        uint32_t x[4 * W], y[4 * W];
#pragma unroll
        for (int k = 0; k < W; k++) {
            const uint4 v = __ldcs(reinterpret_cast<const uint4*>(planes + k * stride + g * 16));
            y[4 * k] = v.x;
            y[4 * k + 1] = v.y;
            y[4 * k + 2] = v.z;
            y[4 * k + 3] = v.w;
        }
        planes_untranspose<W>(y, x);
        if (DELTA) {
            uint32_t b[4 * W];
            planes_load_group<W>(reinterpret_cast<const uint4*>(base) + g * W, b);
            delta_inverse<W>(x, b);
        }
        uint4* dst = reinterpret_cast<uint4*>(out) + g * W;
#pragma unroll
        for (int i = 0; i < W; i++) dst[i] = make_uint4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    }
    const uint64_t tail = groups * 16;
    if (DELTA) {
        if (tid < m - tail) {
            const uint64_t e = tail + tid;
            uint64_t d = 0, b = 0;
#pragma unroll
            for (int k = 0; k < W; k++) {
                d |= static_cast<uint64_t>(planes[k * stride + e]) << (8 * k);
                b |= static_cast<uint64_t>(base[e * W + k]) << (8 * k);
            }
            const uint64_t x = delta_unzigzag<W>(d, b);
#pragma unroll
            for (int k = 0; k < W; k++) out[e * W + k] = static_cast<uint8_t>(x >> (8 * k));
        }
    } else if (tid < (m - tail) * W) {
        const uint64_t e = tail + tid / W, k = tid % W;
        out[e * W + k] = planes[k * stride + e];
    }
}

template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    planes_interleave_kernel(const uint8_t* __restrict__ planes, uint64_t stride, uint8_t* __restrict__ out, const PlanesWork* __restrict__ r)
{
    planes_interleave<W, false>(planes, stride, nullptr, out, r);
}

template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    delta_interleave_kernel(const uint8_t* __restrict__ planes, uint64_t stride, const uint8_t* base, uint8_t* out,
                            const PlanesWork* __restrict__ r)
{
    planes_interleave<W, true>(planes, stride, base, out, r);
}

// Encode: plane p's verdict and place.  Its container is complete (header included) at src -- out + 64 + 16 units for
// plane 0, the staging area for the others -- exactly when the status word is clear, since version 6's header kernel
// writes only then.  units counts the 16-byte units between the header and plane 0: W table entries, and in version 9
// round16(8 T) / 16 more for the directory.  Entry p: the offset right after plane p - 1 (entry p - 1, written by the
// previous launch), the size from the plane's header.  Plane 0 is in place; the others are copied, 16 bytes per thread
// and step.
__global__ void __launch_bounds__(kPlanesThreads)
    planes_place_kernel(uint8_t* __restrict__ out, const uint8_t* __restrict__ src, uint32_t p, uint32_t units, uint64_t out_cap,
                        PlanesWork* __restrict__ r, uint32_t* status)
{
    const bool ok = *status == 0;
    const bool first = blockIdx.x == 0 && threadIdx.x == 0;
    if (first) r->plane_go[p] = 0;
    if (!ok) return;
    PlaneEntry* table = reinterpret_cast<PlaneEntry*>(out + sizeof(ContainerHeader));
    const ContainerHeader h = *reinterpret_cast<const ContainerHeader*>(src);
    const uint64_t size = container_bitmap_blob_offset(h.n_chunks) + h.blob_bytes;
    const uint64_t offset = p ? table[p - 1].offset + table[p - 1].size : sizeof(ContainerHeader) + sizeof(PlaneEntry) * units;
    if (offset > out_cap || size > out_cap - offset) {                // not reached: the host checked the bound
        if (first) atomicOr(status, kStatSpace);
        return;
    }
    if (first) {
        table[p] = PlaneEntry{offset, size};
        r->plane_go[p] = 1;
    }
    if (p == 0) return;
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(out + offset);
    const uint64_t step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < size / 16; i += step) d[i] = s[i];
}

// CRC-32 of the header (crc fields zero) and the table, staged in shared memory at s (bytes = 64 + 16 W, a multiple
// of 32): one warp, bytes / 32 per lane, each shifted past the bytes after it
__device__ __forceinline__ uint32_t planes_meta_crc(const uint8_t* s, uint32_t bytes)
{
    using namespace crc_detail;
    const uint32_t lane = threadIdx.x & 31, piece = bytes / 32;
    uint32_t c = raw_bytes_bitwise(s + lane * piece, piece);
    c = __reduce_xor_sync(0xffffffffu, crc32_shift(c, bytes - piece * (lane + 1)));
    return finish_warp(0, bytes, c);
}

// Encode: the version 7 header, when every plane was placed and the status word is still clear.  h arrives complete
// but for blob_bytes and meta_crc; s_v is the kernel's shared staging of header and table; dir_bytes the directory's
// (version 9; 0 otherwise), between the table and plane 0.
__device__ __forceinline__ void planes_finish(uint4* s_v, uint8_t* out, ContainerHeader h, uint64_t dir_bytes, const PlanesWork* __restrict__ r,
                                              const uint32_t* status)
{
    uint8_t* s = reinterpret_cast<uint8_t*>(s_v);
    const uint32_t lane = threadIdx.x, w = h.block_size;
    bool all = *status == 0;
    for (uint32_t p = 0; p < w; p++) all = all && r->plane_go[p];
    if (!all) return;
    const PlaneEntry* table = reinterpret_cast<const PlaneEntry*>(out + sizeof(ContainerHeader));
    const uint64_t end = container_planes_table_end(w, 0);
    h.blob_bytes = table[w - 1].offset + table[w - 1].size - end - dir_bytes;
    h.meta_crc = 0;
    h.blob_crc = 0;
    if (lane == 0) *reinterpret_cast<ContainerHeader*>(s) = h;
    if (lane < w) s_v[4 + lane] = reinterpret_cast<const uint4*>(table)[lane];
    __syncwarp();
    const uint32_t meta = planes_meta_crc(s, static_cast<uint32_t>(end));
    if (lane == 0) reinterpret_cast<ContainerHeader*>(s)->meta_crc = meta;
    __syncwarp();
    if (lane < 4) reinterpret_cast<uint4*>(out)[lane] = s_v[lane];
}

__global__ void __launch_bounds__(32)
    planes_finish_kernel(uint8_t* out, ContainerHeader h, const PlanesWork* __restrict__ r, const uint32_t* status)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    planes_finish(s_v, out, h, 0, r, status);
}

// The finish of the delta encode: version 8, reserved the base's CRC
__global__ void __launch_bounds__(32)
    delta_finish_kernel(uint8_t* out, ContainerHeader h, const DeltaWork* __restrict__ d, const PlanesWork* __restrict__ r, const uint32_t* status)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    h.version = kContainerVersionDelta;
    h.reserved = d->crc.crc;
    planes_finish(s_v, out, h, 0, r, status);
}

// The finish of the varlen encode: n from the record.  A bad length left the status word set, so nothing is written.
__global__ void __launch_bounds__(32)
    planes_finish_varlen_kernel(uint8_t* out, ContainerHeader h, const PlanesVarlenGeom* __restrict__ g, const PlanesWork* __restrict__ r,
                                const uint32_t* status)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    h.n_symbols = g->n;
    planes_finish(s_v, out, h, 0, r, status);
}

// The first kernel of the varlen encode, one thread: reads n = *d_n and writes n and m = n / w into *g when
// 1 <= n <= n_max and w divides n; otherwise n = 0 and m = UINT64_MAX, which every plane's version 6 varlen plan
// refuses as above its bound (kStatArg, the fixed call's RB200_E_ARG for n == 0 or n % w != 0), writing nothing.
__global__ void __launch_bounds__(32)
    planes_varlen_plan_kernel(const uint64_t* __restrict__ d_n, uint64_t n_max, uint32_t w, PlanesVarlenGeom* __restrict__ g)
{
    if (threadIdx.x) return;
    const uint64_t n = *d_n;
    const bool ok = n != 0 && n <= n_max && n % w == 0;
    *g = ok ? PlanesVarlenGeom{n, n / w} : PlanesVarlenGeom{0, UINT64_MAX};
}

// Decode: every rule of version 7 (VERSION 8 or 9: that version's, and for 9 a T of count) on the header, the table
// and the planes' headers, and meta_crc; the record is reset for the call.  One warp: lanes 0..3 stage the header,
// lanes 4.. the table, lane p < W checks plane p's header.
template <uint16_t VERSION>
__device__ __forceinline__ void planes_plan(uint4* s_v, const uint8_t* __restrict__ buf, uint64_t size, uint32_t w, uint32_t count,
                                            PlanesWork* __restrict__ r)
{
    uint8_t* s = reinterpret_cast<uint8_t*>(s_v);
    const uint32_t lane = threadIdx.x;
    ContainerHeader h = {};
    if (size >= sizeof(ContainerHeader)) h = *reinterpret_cast<const ContainerHeader*>(buf);   // a shorter buffer is not read
    bool ok = size >= sizeof(ContainerHeader) && container_planes_header_version_ok(h, size, VERSION) && h.block_size == w &&
              (VERSION != kContainerVersionTensors || h.n_blocks == count);
    const uint32_t meta_crc = h.meta_crc;
    if (ok) {                                                         // the table lies in size (header rule)
        h.meta_crc = 0;
        h.blob_crc = 0;
        if (lane == 0) *reinterpret_cast<ContainerHeader*>(s) = h;
        if (lane < w) s_v[4 + lane] = reinterpret_cast<const uint4*>(buf + sizeof(ContainerHeader))[lane];
        __syncwarp();
        const PlaneEntry* table = reinterpret_cast<const PlaneEntry*>(s + sizeof(ContainerHeader));
        ok = planes_meta_crc(s, static_cast<uint32_t>(container_planes_table_end(w, 0))) == meta_crc &&
             container_planes_table_ok(h, table, container_planes_dir_bytes(h, VERSION));
        // each plane's header lies in size once the table passes
        const bool plane = !ok || lane >= w ||
                           container_planes_plane_ok(h, *reinterpret_cast<const ContainerHeader*>(buf + table[lane].offset), table[lane].size);
        ok = __all_sync(0xffffffffu, plane) && ok;
    }
    if (lane < 8) {
        r->plane_go[lane] = 0;
        r->table[lane] = ok && lane < w ? reinterpret_cast<const PlaneEntry*>(s + sizeof(ContainerHeader))[lane] : PlaneEntry{0, 0};
    }
    if (lane == 0) {
        r->ok = ok;
        r->go = 0;
        r->n = ok ? h.n_symbols : 0;
    }
}

__global__ void __launch_bounds__(32)
    planes_plan_kernel(const uint8_t* __restrict__ buf, uint64_t size, uint32_t w, PlanesWork* __restrict__ r)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    planes_plan<kContainerVersionPlanes>(s_v, buf, size, w, 0, r);
}

__global__ void __launch_bounds__(32)
    delta_plan_kernel(const uint8_t* __restrict__ buf, uint64_t size, uint32_t w, PlanesWork* __restrict__ r)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    planes_plan<kContainerVersionDelta>(s_v, buf, size, w, 0, r);
}

// Decode: plane p's bytes into staging, when the record passed and the plane fits it; otherwise a zero header, which
// version 6's plan rejects.
__global__ void __launch_bounds__(kPlanesThreads)
    planes_fetch_kernel(const uint8_t* __restrict__ buf, uint8_t* __restrict__ stage, uint64_t stage_cap, uint32_t p,
                        const PlanesWork* __restrict__ r)
{
    const PlaneEntry e = r->table[p];
    const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (!r->ok || e.size > stage_cap) {
        if (tid < sizeof(ContainerHeader) / 16) reinterpret_cast<uint4*>(stage)[tid] = make_uint4(0, 0, 0, 0);
        return;
    }
    const uint4* s = reinterpret_cast<const uint4*>(buf + e.offset);
    uint4* d = reinterpret_cast<uint4*>(stage);
    const uint64_t step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = tid; i < e.size / 16; i += step) d[i] = s[i];
}

// Decode: plane p's version 6 verdict (its workspace's go) into the record
__global__ void __launch_bounds__(32) planes_record_kernel(uint32_t p, const ContainerAsyncWork* __restrict__ w6, PlanesWork* __restrict__ r)
{
    if (threadIdx.x == 0) r->plane_go[p] = w6->go != 0;
}

// Decode: the call's verdict.  The header and table rejected: kStatStream.  Otherwise n is written, then n > out_cap
// is kStatSpace, a plane that failed its checks kStatStream, and a call that passed everything sets go.
__device__ __forceinline__ void planes_verdict(uint32_t w, uint64_t out_cap, uint64_t* __restrict__ n_symbols, PlanesWork* __restrict__ r,
                                               uint32_t* status)
{
    if (!r->ok) {
        atomicOr(status, kStatStream);
        return;
    }
    if (n_symbols) *n_symbols = r->n;
    bool all = true;
    for (uint32_t p = 0; p < w; p++) all = all && r->plane_go[p];
    if (r->n > out_cap)
        atomicOr(status, kStatSpace);
    else if (!all)
        atomicOr(status, kStatStream);
    else
        r->go = 1;
}

__global__ void __launch_bounds__(32)
    planes_verdict_kernel(uint32_t w, uint64_t out_cap, uint64_t* __restrict__ n_symbols, PlanesWork* __restrict__ r, uint32_t* status)
{
    if (threadIdx.x) return;
    planes_verdict(w, out_cap, n_symbols, r, status);
}

// Decode, version 8: the verdict, then the length of base the CRC covers: n once every check passed (so n <= out_cap),
// otherwise 0, and the base is not read
__global__ void __launch_bounds__(32)
    delta_verdict_kernel(uint32_t w, uint64_t out_cap, uint64_t* __restrict__ n_symbols, PlanesWork* __restrict__ r, uint32_t* status,
                         DeltaWork* __restrict__ d)
{
    if (threadIdx.x) return;
    planes_verdict(w, out_cap, n_symbols, r, status);
    d->base_n = r->go ? r->n : 0;
}

// Decode, version 8: when every other check passed, the base's CRC against the header's reserved word (the header
// passed, so buf holds it); a different base clears go, so the interleave writes nothing, and flags kStatBase.
__global__ void __launch_bounds__(32)
    delta_check_kernel(const uint8_t* __restrict__ buf, const DeltaWork* __restrict__ d, PlanesWork* __restrict__ r, uint32_t* status)
{
    if (threadIdx.x || !r->go) return;
    if (d->crc.crc != reinterpret_cast<const ContainerHeader*>(buf)->reserved) {
        r->go = 0;
        atomicOr(status, kStatBase);
    }
}

// ---- version 9: a list of tensors

constexpr uint32_t kTensorsPlanThreads = 1024;   // the plan and check kernels: one CTA, 32 warps

// Thread t of a kTensorsPlanThreads CTA takes the entries [begin, end) of count: a run of ceil(count / threads)
__device__ __forceinline__ void tensors_run(uint32_t count, uint32_t& begin, uint32_t& end)
{
    const uint32_t k = (count + kTensorsPlanThreads - 1) / kTensorsPlanThreads;
    begin = min(threadIdx.x * k, count);
    end = min(begin + k, count);
}

// The CTA's exclusive scan of one value per thread (the sum of its run): returns the sum of the threads before this
// one, and *total the sum of all.  s_warp: 32 words of shared memory.
__device__ __forceinline__ uint64_t tensors_block_scan(uint64_t v, uint64_t* s_warp, uint64_t* total)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t t = s_warp[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t y = __shfl_up_sync(0xffffffffu, t, d);
            if (lane >= d) t += y;
        }
        s_warp[lane] = t;
    }
    __syncthreads();
    *total = s_warp[31];
    return (warp ? s_warp[warp - 1] : 0) + x - v;
}

// Encode, the first kernel: every entry of the list -- bytes a multiple of w and at most n_max (so the sum of the
// count entries cannot overflow), ptr nonzero and aligned to w unless bytes is 0 -- and the total, 1 .. n_max.  Writes
// the exclusive prefix of the element counts, prefix[0 .. count], and *g: {n, n / w}, or {0, UINT64_MAX} for a bad list
// (which every plane's version 6 varlen plan refuses as kStatArg, so nothing is written).  Only a good list's lengths
// go to the directory at dir, with its zero padding.
__global__ void __launch_bounds__(kTensorsPlanThreads)
    tensors_plan_kernel(const rb200_tensor_ref* __restrict__ refs, uint32_t count, uint32_t w, uint64_t n_max, uint64_t* __restrict__ prefix,
                        PlanesVarlenGeom* __restrict__ g, uint64_t* __restrict__ dir)
{
    __shared__ uint64_t s_warp[32];
    const uint32_t shift = __ffs(w) - 1;                               // w is 2, 4 or 8
    uint32_t begin, end;
    tensors_run(count, begin, end);
    bool ok = true;
    uint64_t sum = 0;                                                  // elements
    for (uint32_t i = begin; i < end; i++) {
        const rb200_tensor_ref t = refs[i];
        const bool fits = t.bytes <= n_max;
        ok = ok && fits && !(t.bytes & (w - 1)) && (t.bytes == 0 || (t.ptr && !(t.ptr & (w - 1))));
        sum += fits ? t.bytes >> shift : 0;
    }
    ok = __syncthreads_and(ok);
    uint64_t total;
    uint64_t e = tensors_block_scan(sum, s_warp, &total);
    ok = ok && total && total <= n_max >> shift;
    for (uint32_t i = begin; i < end; i++) {
        const uint64_t bytes = refs[i].bytes;
        prefix[i] = e;
        e += bytes <= n_max ? bytes >> shift : 0;
        if (ok) dir[i] = bytes;
    }
    if (threadIdx.x == 0) {
        prefix[count] = total;
        if (ok && count % 2) dir[count] = 0;
        *g = ok ? PlanesVarlenGeom{total << shift, total} : PlanesVarlenGeom{0, UINT64_MAX};
    }
}

// A thread's place in the list: tensor i holds the elements [lo, hi) of the concatenation, at ptr
struct TensorCursor {
    uint32_t i;
    uint64_t lo, hi, ptr;
};

// Moves c to the tensor that holds element e < prefix[count]; e never decreases along a thread's walk, so c stays while
// e < hi and otherwise a binary search over prefix[c.i .. count] finds the last tensor that starts at or before e, which
// is never one of zero length.
__device__ __forceinline__ void tensors_seek(const uint64_t* __restrict__ prefix, const rb200_tensor_ref* __restrict__ refs, uint32_t count,
                                             uint64_t e, TensorCursor& c)
{
    if (e < c.hi) return;
    uint32_t a = c.i, b = count;                                       // prefix[a] <= e < prefix[b]
    while (b - a > 1) {
        const uint32_t mid = (a + b) / 2;
        if (prefix[mid] <= e) a = mid;
        else b = mid;
    }
    c.i = a;
    c.lo = prefix[a];
    c.hi = prefix[a + 1];
    c.ptr = refs[a].ptr;
}

// Element j (0..15) of 16 in 4 W words, as planes_load_group leaves them
template <int W>
__device__ __forceinline__ void tensors_put(uint32_t (&x)[4 * W], int j, uint64_t v)
{
    if (W == 2) {
        if (j & 1) x[j >> 1] |= static_cast<uint32_t>(v) << 16;
        else x[j >> 1] = static_cast<uint32_t>(v);
    } else if (W == 4) {
        x[j] = static_cast<uint32_t>(v);
    } else {
        x[2 * j] = static_cast<uint32_t>(v);
        x[2 * j + 1] = static_cast<uint32_t>(v >> 32);
    }
}
template <int W>
__device__ __forceinline__ uint64_t tensors_get(const uint32_t (&x)[4 * W], int j)
{
    if (W == 2) return (x[j >> 1] >> (16 * (j & 1))) & 0xffffu;
    if (W == 4) return x[j];
    return static_cast<uint64_t>(x[2 * j + 1]) << 32 | x[2 * j];
}

// One element at a w-aligned address (the encode's list rule)
template <int W>
__device__ __forceinline__ uint64_t tensors_load(uint64_t addr)
{
    if (W == 2) return *reinterpret_cast<const uint16_t*>(addr);
    if (W == 4) return *reinterpret_cast<const uint32_t*>(addr);
    return *reinterpret_cast<const uint64_t*>(addr);
}
// One element at any address: the decode's outputs need no alignment
template <int W>
__device__ __forceinline__ void tensors_store(uint64_t addr, uint64_t v)
{
    if (addr % W) {
#pragma unroll
        for (int k = 0; k < W; k++) reinterpret_cast<uint8_t*>(addr)[k] = static_cast<uint8_t>(v >> (8 * k));
    } else if (W == 2) {
        *reinterpret_cast<uint16_t*>(addr) = static_cast<uint16_t>(v);
    } else if (W == 4) {
        *reinterpret_cast<uint32_t*>(addr) = static_cast<uint32_t>(v);
    } else {
        *reinterpret_cast<uint64_t*>(addr) = v;
    }
}

// The segmented split: the concatenation of the list's tensors (m elements, from the record) into W planes, as
// planes_split_kernel would split the concatenated bytes.  Groups of 16 elements; a group that lies in one tensor at a
// 16-byte-aligned address takes W 16-byte loads, any other (across tensors, or in an element-aligned view) one load
// per element.  The ragged end (fewer than 16 elements) an element per thread.  Nothing for a bad list.
template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    tensors_split_kernel(const rb200_tensor_ref* __restrict__ refs, const uint64_t* __restrict__ prefix, uint32_t count,
                         const PlanesVarlenGeom* __restrict__ geom, uint8_t* __restrict__ planes, uint64_t stride)
{
    if (geom->n == 0) return;
    const uint64_t m = geom->m, groups = m / 16, step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    TensorCursor c = {0, 0, 0, 0};
    for (uint64_t g = tid; g < groups; g += step) {
        const uint64_t e = g * 16;
        tensors_seek(prefix, refs, count, e, c);
        uint32_t x[4 * W], y[4 * W];
        const uint64_t src = c.ptr + (e - c.lo) * W;
        if (e + 16 <= c.hi && !(src & 15)) {
            planes_load_group<W>(reinterpret_cast<const uint4*>(src), x);
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++) {
                tensors_seek(prefix, refs, count, e + j, c);
                tensors_put<W>(x, j, tensors_load<W>(c.ptr + (e + j - c.lo) * W));
            }
        }
        planes_transpose<W>(x, y);
#pragma unroll
        for (int k = 0; k < W; k++)
            *reinterpret_cast<uint4*>(planes + k * stride + g * 16) = make_uint4(y[4 * k], y[4 * k + 1], y[4 * k + 2], y[4 * k + 3]);
    }
    const uint64_t tail = groups * 16;
    if (tid < m - tail) {
        const uint64_t e = tail + tid;
        tensors_seek(prefix, refs, count, e, c);
        const uint64_t v = tensors_load<W>(c.ptr + (e - c.lo) * W);
#pragma unroll
        for (int k = 0; k < W; k++) planes[k * stride + e] = static_cast<uint8_t>(v >> (8 * k));
    }
}

// Its inverse, from the decode workspace into the refs' outputs, only when every check passed: the groups' 16-byte
// stores where a group lies in one tensor at a 16-byte-aligned address, element stores otherwise.
template <int W>
__global__ void __launch_bounds__(kPlanesThreads)
    tensors_interleave_kernel(const uint8_t* __restrict__ planes, uint64_t stride, const rb200_tensor_ref* __restrict__ refs,
                              const uint64_t* __restrict__ prefix, uint32_t count, const PlanesWork* __restrict__ r)
{
    if (!r->go) return;
    const uint64_t m = r->n / W, groups = m / 16, step = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    const uint64_t tid = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    TensorCursor c = {0, 0, 0, 0};
    for (uint64_t g = tid; g < groups; g += step) {
        uint32_t x[4 * W], y[4 * W];
#pragma unroll
        for (int k = 0; k < W; k++) {
            const uint4 v = __ldcs(reinterpret_cast<const uint4*>(planes + k * stride + g * 16));
            y[4 * k] = v.x;
            y[4 * k + 1] = v.y;
            y[4 * k + 2] = v.z;
            y[4 * k + 3] = v.w;
        }
        planes_untranspose<W>(y, x);
        const uint64_t e = g * 16;
        tensors_seek(prefix, refs, count, e, c);
        const uint64_t dst = c.ptr + (e - c.lo) * W;
        if (e + 16 <= c.hi && !(dst & 15)) {
            uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
            for (int i = 0; i < W; i++) d[i] = make_uint4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < 16; j++) {
                tensors_seek(prefix, refs, count, e + j, c);
                tensors_store<W>(c.ptr + (e + j - c.lo) * W, tensors_get<W>(x, j));
            }
        }
    }
    const uint64_t tail = groups * 16;
    if (tid < m - tail) {
        const uint64_t e = tail + tid;
        uint64_t v = 0;
#pragma unroll
        for (int k = 0; k < W; k++) v |= static_cast<uint64_t>(planes[k * stride + e]) << (8 * k);
        tensors_seek(prefix, refs, count, e, c);
        tensors_store<W>(c.ptr + (e - c.lo) * W, v);
    }
}

// Encode, last: the version 9 header (h arrives with version 9 and n_blocks = T), with n from the record and reserved
// the directory's CRC.  A bad list left the status word set, so nothing is written.
__global__ void __launch_bounds__(32)
    tensors_finish_kernel(uint8_t* out, ContainerHeader h, uint64_t dir_bytes, const PlanesVarlenGeom* __restrict__ g,
                          const TensorsWork* __restrict__ t, const PlanesWork* __restrict__ r, const uint32_t* status)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    h.n_symbols = g->n;
    h.reserved = t->crc.crc;
    planes_finish(s_v, out, h, dir_bytes, r, status);
}

// Decode, first: the plan with version 9's rules and T == count, and the directory's length for its CRC (8 T once the
// header and table passed, so the directory lies in size; else 0)
__global__ void __launch_bounds__(32)
    tensors_open_kernel(const uint8_t* __restrict__ buf, uint64_t size, uint32_t w, uint32_t count, PlanesWork* __restrict__ r,
                        TensorsWork* __restrict__ t)
{
    __shared__ uint4 s_v[(sizeof(ContainerHeader) + 8 * sizeof(PlaneEntry)) / 16];
    planes_plan<kContainerVersionTensors>(s_v, buf, size, w, count, r);
    if (threadIdx.x == 0) t->dir_len = r->ok ? 8ull * count : 0;
}

// Decode, after the verdict, when every other check passed: the directory's CRC against the header's reserved word,
// its rules (container_tensors_dir_part_ok over every thread's run, the sum n, the zero padding) -- a failure is
// kStatStream -- then d_lengths and the directory's exclusive prefix in elements, prefix[0 .. count], and every length
// against its ref's capacity -- a failure is kStatSpace.  Either clears go, so the interleave writes nothing.
__global__ void __launch_bounds__(kTensorsPlanThreads)
    tensors_check_kernel(const uint8_t* __restrict__ buf, uint32_t w, uint32_t count, const rb200_tensor_ref* __restrict__ refs,
                         uint64_t* __restrict__ prefix, uint64_t* __restrict__ d_lengths, const TensorsWork* __restrict__ t,
                         PlanesWork* __restrict__ r, uint32_t* status)
{
    __shared__ uint64_t s_warp[32];
    if (!r->go) return;                  // every thread reads go before any clears it: the clears follow the barriers below
    const uint64_t* dir = reinterpret_cast<const uint64_t*>(buf + container_planes_table_end(w, 0));
    const uint64_t n = r->n;
    const uint32_t shift = __ffs(w) - 1;                               // w is 2, 4 or 8
    uint32_t begin, end;
    tensors_run(count, begin, end);
    uint64_t sum = 0;
    bool ok = container_tensors_dir_part_ok(dir, begin, end, w, n, &sum);
    if (threadIdx.x == 0)
        ok = ok && t->crc.crc == reinterpret_cast<const ContainerHeader*>(buf)->reserved && container_tensors_dir_pad_ok(dir, count);
    ok = __syncthreads_and(ok);
    uint64_t total;
    uint64_t e = tensors_block_scan(sum, s_warp, &total);
    if (!ok || total != n) {
        if (threadIdx.x == 0) {
            r->go = 0;
            atomicOr(status, kStatStream);
        }
        return;
    }
    bool fits = true;
    for (uint32_t i = begin; i < end; i++) {
        const uint64_t bytes = dir[i];
        if (d_lengths) d_lengths[i] = bytes;
        prefix[i] = e >> shift;
        e += bytes;
        fits = fits && bytes <= refs[i].bytes;
    }
    if (threadIdx.x == 0) prefix[count] = n >> shift;
    fits = __syncthreads_and(fits);
    if (!fits && threadIdx.x == 0) {
        r->go = 0;
        atomicOr(status, kStatSpace);
    }
}

}  // namespace rb200

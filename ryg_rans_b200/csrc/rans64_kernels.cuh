// rans64_kernels.cuh -- sm_90a kernels for the rans64.h coder as main64.cpp drives it:
// 64-bit state in [2^31, 2^63), 32-bit renormalisation units (never loops), cum2sym symbol lookup.
//
//   Rans64DecGet / cum2sym / Rans64DecAdvanceSymbolStep / Rans64DecRenorm   rans64.h:118-121, main64.cpp:202,
//                                                                           rans64.h:289-316
//   Rans64EncPutSymbol (reciprocal form) + Rans64EncFlush                    rans64.h:262-278, :96-103
//
// Same mapping as the other coders (one warp = one chunk = one 32-way stream, one ballot per step
// because a lane moves at most one u32 per step).  This is the "lets the GPU decode streams made by
// the reference's fastest CPU encoder" row of SURVEY 8(f); it runs on the chunk decoder and encoder every coder
// shares (decode_stream.cuh: stream window; encode_stream.cuh: symbol stage, output ring, flush), and is not
// tuned beyond that.  Its encoder is split-only: per-chunk slots, then the tile scan and compaction.
#pragma once
#include "decode_stream.cuh"
#include "device_utils.cuh"
#include "encode_stream.cuh"
#include "tables.h"

namespace rb200 {

constexpr uint64_t kRans64L = 1ull << 31;          // RANS64_L, rans64.h:59
constexpr uint32_t kRans64HeaderBytes = 256;       // 32 lanes x u64 (Rans64EncFlush x 32)
constexpr int kRans64Warps = 16;
constexpr uint32_t kRans64DecReplicas = 16;        // an LDS.64 is served 16 lanes at a time: one {start, freq} copy per lane of a half-warp
constexpr uint32_t kRans64DecSymBytes = 256 * kRans64DecReplicas * 8;      // 32 KiB

// The rans64 coder for decode_window_chunk.  tab = shared address of cum2sym[1 << sb]; syms_lane = this lane's replica of
// the 256 x {start, freq} table that follows it (16 replicas, entry s of replica r at (s * 16 + r) * 8: the 16 lanes of
// each LDS.64 phase hit 16 different 8-byte bank groups whatever their symbols are)
struct Rans64Decoder {
    using X = uint64_t;
    static constexpr uint32_t kHeaderBytes = kRans64HeaderBytes, kUnit = 4, kMaxBytes = 4;
    static constexpr X kL = kRans64L;                  // Rans64EncInit, rans64.h:65-68
    uint32_t tab;
    uint32_t syms_lane;
    uint32_t sb;

    // Rans64DecInit x 32 (rans64.h:107-115): lane k's state is the k-th u64
    template <class At>
    __device__ __forceinline__ X read_header(At at, uint32_t lane) const
    {
        return lds_u32(at(8 * lane)) | (static_cast<uint64_t>(lds_u32(at(8 * lane + 4))) << 32);
    }

    template <bool FULL>
    __device__ __forceinline__ void step(uint64_t& x, uint32_t& cursor, uint32_t ring, uint8_t* o, uint32_t lt, bool active) const
    {
        bool need = false;
        if (active) {
            const uint32_t cf = static_cast<uint32_t>(x) & ((1u << sb) - 1);               // rans64.h:120
            const uint32_t s = lds_u8_ro(tab + cf);                                        // main64.cpp:202
            const uint2 ds = lds_u64_ro(syms_lane + s * (kRans64DecReplicas * 8));         // Rans64DecSymbol {start, freq}
            x = static_cast<uint64_t>(ds.y) * (x >> sb) + cf - ds.x;                       // rans64.h:297
            *o = static_cast<uint8_t>(s);
            need = x < kRans64L;                                                           // :309
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, need);
        const uint32_t a = cursor + 4u * __popc(mask & lt);
        const uint32_t w = lds_u32(ring | (a & (kRingBytes - 1)));
        if (need) x = (x << 32) | w;                                                       // :310
        cursor += 4u * __popc(mask);
    }
};

__global__ void __launch_bounds__(kRans64Warps * 32, 2)
rans64_decode_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets, uint32_t sb,
                     const uint8_t* __restrict__ g_tab,   // cum2sym[1 << sb] + 256 x {start, freq}
                     uint8_t* __restrict__ out, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t* __restrict__ status)
{
    extern __shared__ __align__(1024) uint8_t s_r64[];        // [16 x 1 KiB rings][cum2sym][256 x 16 replicas x {start, freq}]
    uint4* s_tab = reinterpret_cast<uint4*>(s_r64 + kRans64Warps * kRingBytes);
    const uint32_t vecs = (1u << sb) / 16;
    for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) s_tab[i] = reinterpret_cast<const uint4*>(g_tab)[i];
    {
        const uint2* g_syms = reinterpret_cast<const uint2*>(g_tab + (1u << sb));
        uint2* s_syms = reinterpret_cast<uint2*>(s_r64 + kRans64Warps * kRingBytes + (1u << sb));
        for (uint32_t i = threadIdx.x; i < 256 * kRans64DecReplicas; i += blockDim.x) s_syms[i] = g_syms[i / kRans64DecReplicas];
    }
    __syncthreads();

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * kRans64Warps + warp;
    if (chunk >= n_chunks) return;
    const uint64_t first = static_cast<uint64_t>(chunk) * chunk_syms;
    const uint32_t m = static_cast<uint32_t>(min(static_cast<uint64_t>(chunk_syms), n - first));
    const uint32_t tab = smem_addr(s_tab);
    const Rans64Decoder coder = {tab, tab + (1u << sb) + (lane & (kRans64DecReplicas - 1)) * 8, sb};
    decode_window_chunk(coder, blob, blob_size, offsets, chunk, smem_addr(s_r64) + warp * kRingBytes, out + first, m, status);
}

// The rans64 coder for encode_stream (encode_stream.cuh); wpos is the ring position of the next u32 =
// 508 - 4 * words_emitted.  step = Rans64EncPutSymbol for 32 lanes (rans64.h:262-278).  tab_lane = this lane's replica
// of the 256-entry table {rcp_lo, rcp_hi, bias, cmpl_freq | rcp_shift << 20 | bad << 31}: one 16-byte Rans64EncSymbol
// image per symbol (freq is M - cmpl_freq), replicated 8x so that the 8 lanes of a quarter-warp hit 8 different 16-byte
// bank groups -- ONE conflict-free LDS.128 per step.  (Round 1 read the 32-byte image with two LDS.128 from an
// unreplicated table: ~28 wavefronts per step, shared-memory data pipe 99 % busy, 3.8 ms per GiB.)
struct Rans64Encoder {
    using X = uint64_t;
    static constexpr uint32_t kUnit = 4, kMaxEmit = 4, kBadBit = kEncBadSymbol;
    static constexpr X kInit = kRans64L;               // Rans64EncInit, rans64.h:65-68
    uint32_t tab;                                      // shared address of the 8x replicated uint4 table
    uint32_t sb;

    template <bool FULL>
    __device__ __forceinline__ void step(EncState<X>& st, uint32_t sym, uint32_t tab_lane, uint32_t ring, uint32_t gt, bool active) const
    {
        bool need = false;
        uint4 e = make_uint4(0, 0, 0, 0);
        if (active) {
            e = lds_u128_ro(tab_lane + sym * (kEncReplicas * 16));
            st.flags |= e.w;
            const uint32_t freq = (1u << sb) - (e.w & 0xfffffu);
            const uint64_t x_max = static_cast<uint64_t>(freq) << (63 - sb);               // ((L >> sb) << 32) * freq, :269
            need = st.x >= x_max;
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, need);
        if (need) {
            asm volatile("st.shared.u32 [%0], %1;" ::"r"(ring | ((st.wpos - 4u * __popc(mask & gt)) & (kEncRingBytes - 1))),
                         "r"(static_cast<uint32_t>(st.x))
                         : "memory");                                                      // :271-272
            st.x >>= 32;                                                                   // :273
        }
        st.wpos -= 4u * __popc(mask);
        if (active) {
            const uint64_t rcp = static_cast<uint64_t>(e.x) | (static_cast<uint64_t>(e.y) << 32);
            const uint64_t q = __umul64hi(st.x, rcp) >> ((e.w >> 20) & 63u);               // :276
            st.x = st.x + e.z + q * (e.w & 0xfffffu);                                      // :277
        }
    }
};

// GEOM (rb200_container_model_encode_varlen_async): n and the chunk count from the record, on a grid sized for n_max; a
// CTA past the real chunks exits before it stages the table.  GATED (rb200_container_model_encode_auto_async): runs only
// when the choice record names `group`, at the recorded scale_bits; otherwise it exits at entry.
template <bool GEOM = false, bool GATED = false>
__global__ void __launch_bounds__(kRans64Warps * 32, 2)
rans64_encode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t sb,
                     const uint4* __restrict__ g_enc,      // 256 x 2 x uint4
                     uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint32_t* __restrict__ sizes, uint32_t* __restrict__ status,
                     const VarlenGeom* __restrict__ geom, const CoderChoice* __restrict__ choice, uint32_t group)
{
    if (GATED) {
        if (choice->group != group) return;
        sb = choice->scale_bits;
    }
    if (GEOM) {
        n_chunks = geom->n_chunks;
        if (!geom->go || blockIdx.x * kRans64Warps >= n_chunks) return;
    }
    // [16 x 1 KiB stage + ring][32 KiB table, 8 replicas].  The instances name it differently: with one name for
    // GEOM and not, or for GATED and not, ptxas schedules the shipped instances differently.
    extern __shared__ __align__(1024) uint8_t s_r64e[];
    extern __shared__ __align__(1024) uint8_t s_r64v[];
    extern __shared__ __align__(1024) uint8_t s_r64g[];
    uint8_t* const s_enc = GATED ? s_r64g : (GEOM ? s_r64v : s_r64e);
    uint4* s_tab = reinterpret_cast<uint4*>(s_enc + kRans64Warps * kEncWarpSmem);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) {
        const uint4 a = g_enc[2 * (i / kEncReplicas)], b = g_enc[2 * (i / kEncReplicas) + 1];   // {rcp_lo, rcp_hi, freq, bias}, {cmpl, shift | bad, -, -}
        s_tab[i] = make_uint4(a.x, a.y, a.w, (b.x & 0xfffffu) | ((b.y & 63u) << 20) | (b.y & kEncBadSymbol));
    }
    __syncthreads();

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * kRans64Warps + warp;
    if (chunk >= n_chunks) return;
    if (GEOM) n = geom->n;
    const ChunkRange r = chunk_range(chunk, chunk_syms, n);
    encode_chunk_split(in + r.first, r.m, chunk, Rans64Encoder{smem_addr(s_tab), sb}, smem_addr(s_enc) + warp * kEncWarpSmem, scratch,
                       slot_bytes, sizes, status);
}
constexpr uint32_t kRans64EncSmemBytes = kRans64Warps * kEncWarpSmem + kEncTableBytes;     // dynamic shared memory of the encoder

inline void configure_rans64_kernels()
{
    cudaFuncSetAttribute(rans64_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRans64Warps * kRingBytes + kRans64DecSymBytes + (1u << 16));
    cudaFuncSetAttribute(rans64_decode_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    for (const void* k : {reinterpret_cast<const void*>(rans64_encode_kernel<false>), reinterpret_cast<const void*>(rans64_encode_kernel<true>),
                          reinterpret_cast<const void*>(rans64_encode_kernel<false, true>), reinterpret_cast<const void*>(rans64_encode_kernel<true, true>)}) {
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kRans64EncSmemBytes);
    }
}

inline void launch_rans64_decode(cudaStream_t stream, const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, uint32_t sb,
                                 const uint8_t* table, uint8_t* out, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t* status)
{
    const uint32_t grid = (n_chunks + kRans64Warps - 1) / kRans64Warps;
    rans64_decode_kernel<<<grid, kRans64Warps * 32, kRans64Warps * kRingBytes + kRans64DecSymBytes + (1u << sb), stream>>>(
        blob, blob_size, offsets, sb, table, out, n, chunk_syms, n_chunks, status);
}

}  // namespace rb200

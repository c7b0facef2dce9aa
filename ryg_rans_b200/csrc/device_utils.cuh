// device_utils.cuh -- small sm_90a device helpers shared by the rANS kernels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace rb200 {

// status bits the kernels OR into the context's device status word
constexpr uint32_t kStatStream = 1u;   // a chunk stream did not end where it must / bad directory
constexpr uint32_t kStatSymbol = 2u;   // encoder saw a symbol with model frequency 0
constexpr uint32_t kStatSpace  = 4u;   // compacted blob does not fit blob_cap
constexpr uint32_t kStatStall  = 8u;   // a bounded wait inside a kernel expired (a bug or a wedged GPU, not bad input)
constexpr uint32_t kStatModel  = 16u;  // the model built from the data is one rb200_model_create refuses
constexpr uint32_t kStatArg    = 32u;  // a length read from device memory is outside what the call was enqueued for
constexpr uint32_t kStatBase   = 64u;  // a delta container's base has another CRC than the one it was encoded against

constexpr uint32_t kHeaderBytes = 128; // 32 lanes x u32 final state (RansWordEncFlush / RansEncFlush x 32)

// The geometry of rb200_container_model_encode_varlen_async, which reads the input length from device memory: written
// by varlen_plan_kernel (model_kernels.cuh) from *d_n at every run, read at entry by every kernel after it (the GEOM
// instances of the C4 kernels), which all exit when go == 0.  The launch shapes are the host's, sized for n_max;
// everything that depends on n is here.
struct VarlenGeom {
    uint64_t n;            // symbols, 1 <= n <= n_max
    uint64_t dir_len;      // directory bytes, 8 (n_chunks + 1)
    uint64_t blob_off;     // offset of the blob in the container, round16(dir_off + dir_len)
    uint64_t blob_cap;     // out_cap - blob_off
    uint64_t blob_len;     // dir[n_chunks], copied after the encoder (the blob CRC's length)
    uint32_t n_chunks;
    uint32_t go;           // 1: *d_n passed the checks; 0: nothing after the plan runs (dir_len, blob_off, blob_len are 0)
    uint64_t dir_off;      // offset of the directory in the container: 1088 (version 1), 64 + 512 n_blocks (per-block)
};

// The geometry of rb200_container_blocks_model_encode_varlen_async, which reads the block count from device memory:
// written by blocks_varlen_plan_kernel (model_kernels.cuh) from *d_n_blocks at every run.  v is the VarlenGeom of the
// container's symbols and chunks (n = n_blocks x block_size), so the GEOM instances of C5 read it as they are; the
// meta CRC's length follows it.
struct BlocksVarlenGeom {
    VarlenGeom v;
    uint64_t meta_len;     // 512 n_blocks + v.dir_len: models and directory, the bytes the meta CRC's kernel covers
    uint32_t n_blocks;     // 1 <= n_blocks <= n_blocks_max; 0 when v.go == 0
    uint32_t reserved;
};

// The geometry of rb200_container_stored_encode_varlen_async (version 6), which reads the input length from device
// memory: written by stored_varlen_plan_kernel (model_kernels.cuh) from *d_n at every run.  v is the VarlenGeom of the
// container's symbols and chunks with v.blob_off past the stored-chunk bitmap (container_bitmap_blob_offset), so the
// GEOM instances of C5 read it as they are; the meta CRC's length follows it.
struct StoredVarlenGeom {
    VarlenGeom v;
    uint64_t meta_len;     // v.blob_off - 1088: directory, pad and bitmap, the bytes the meta CRC's kernel covers
};

// The choice of rb200_container_model_encode_auto_async: written by coder_choice_kernel (model_kernels.cuh) at every
// run, read by the CHOSEN / GATED instances after it.  The host launches one gated group of encode kernels per distinct
// encoder instance the candidate list needs; only the group named here runs, the others exit at entry.
constexpr uint32_t kMaxCandidates = 16;
struct CoderChoice {
    uint32_t coder, scale_bits;        // the chosen pair
    uint32_t index;                    // its place in the caller's list (the first one when none is feasible)
    uint32_t group;                    // the launch group that encodes
    uint64_t costs[kMaxCandidates];    // every candidate's cost, UINT64_MAX when infeasible
};

// The choice of rb200_container_blocks_model_encode_auto_async: the record the gated encode groups read (choice: pair,
// index, group and every candidate's cost) and the container version the header kernel writes, with the running sums
// of blocks_choice_kernel (model_kernels.cuh), which the host zeroes (one memset from `done` on) before every launch.
struct BlocksChoice {
    CoderChoice choice;
    uint32_t version;
    uint32_t done;                                // CTAs that have added their costs
    unsigned long long sums[kMaxCandidates];      // the costs so far
};

__device__ __forceinline__ uint32_t lanemask_lt()
{
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
__device__ __forceinline__ uint32_t lanemask_gt()
{
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_gt;" : "=r"(m));
    return m;
}

__device__ __forceinline__ uint64_t global_timer_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint32_t smem_addr(const void* p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// same value, but produced by a volatile asm so the compiler keeps it in a register instead of
// re-deriving it (S2UR SR_CgaCtaId + LEA) inside hot loops when registers are tight
__device__ __forceinline__ uint32_t smem_addr_pinned(const void* p)
{
    uint32_t a;
    asm volatile("{ .reg .u64 t; cvta.to.shared.u64 t, %1; cvt.u32.u64 %0, t; }" : "=r"(a) : "l"(p));
    return a;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr)
{
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
// read-only tables (written once before a __syncthreads): not volatile, so the
// compiler may schedule these freely
__device__ __forceinline__ uint32_t lds_u32_ro(uint32_t addr)
{
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8_ro(uint32_t addr)
{
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint2 lds_u64_ro(uint32_t addr)
{
    uint2 v;
    asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint4 lds_u128_ro(uint32_t addr)
{
    uint4 v;
    asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

__device__ __forceinline__ uint2 lds_u64(uint32_t addr)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint4 lds_u128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u128(uint32_t addr, uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts_u16(uint32_t addr, uint32_t v)
{
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(static_cast<uint16_t>(v)) : "memory");
}
__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v)
{
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// streaming 128-bit global load: read-only path, do not keep in L1
__device__ __forceinline__ uint4 ldg_stream_u128(const uint4* p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ void stg_stream_u128(uint4* p, uint4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}


// ---- L2 residency hints (createpolicy + .L2::cache_hint).  The fused encoders park every finished stream in a
// per-warp scratch slot until its final position is known; marking those lines evict_last and the one-pass streams
// (symbols in, blob out) evict_first keeps as much of the scratch as fits in L2 (50 MB on H100) instead of making an HBM round trip.
__device__ __forceinline__ uint64_t l2_policy_keep()
{
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_stream()
{
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void stg_hint_u128(uint4* p, uint4 v, uint64_t policy)
{
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w), "l"(policy)
                 : "memory");
}
// L2-coherent load (data this kernel wrote itself) with a residency hint
__device__ __forceinline__ uint4 ldg_cg_hint_u128(const uint4* p, uint64_t policy)
{
    uint4 v;
    asm volatile("ld.global.cg.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(policy)
                 : "memory");
    return v;
}
__device__ __forceinline__ uint4 ldg_stream_hint_u128(const uint4* p, uint64_t policy)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p), "l"(policy));
    return v;
}

}  // namespace rb200

// pairing.cu -- block_alias_tables and block_alias_remap (block_coder_kernels.cuh), the per-block alias table build of
// the rb200_blocks_alias_* kernels, run on the GPU for tests/test_alias_pairing_on_gpu.py.
//
// One CTA per model, at the blockDim the test picks (the kernels run 128 to 1024 threads): block_prefix of the row, then
// the shipped device functions on the shared arrays, the remap in dynamic shared memory pre-filled with a sentinel so
// that a slot the fill misses shows.  Every array goes back to global memory for the comparison with the host builder
// rb200_alias_tables_build.
#include "rans_b200.h"

#include "block_coder_kernels.cuh"

using namespace rb200;

namespace {

constexpr uint16_t kSentinel = 0xfffe;

__global__ void __launch_bounds__(1024)
    batch_alias_tables(const uint16_t* rows, uint32_t M, uint32_t* divider, uint32_t* slot_adjust, uint32_t* slot_freqs, uint8_t* sym_id,
                       uint16_t* remap, uint32_t* flags)
{
    extern __shared__ __align__(16) uint8_t s_dyn[];            // [AliasBuildSmem][remap: M x u16]
    __shared__ uint32_t s_cum[257];
    __shared__ uint32_t s_flag[1];
    AliasBuildSmem& a = *reinterpret_cast<AliasBuildSmem*>(s_dyn);
    uint16_t* s_remap = reinterpret_cast<uint16_t*>(s_dyn + sizeof(AliasBuildSmem));
    const uint32_t tid = threadIdx.x, m = blockIdx.x;
    for (uint32_t j = tid; j < M; j += blockDim.x) s_remap[j] = kSentinel;
    const bool summed = block_prefix(rows + m * 256, s_cum, &s_flag[0], M);
    const bool paired = summed && block_alias_tables(s_cum, M, a);
    if (paired) block_alias_remap(a, M, s_remap);
    __syncthreads();
    for (uint32_t i = tid; i < 512; i += blockDim.x) {
        if (i < 256) divider[m * 256 + i] = a.divider[i];
        slot_adjust[m * 512 + i] = a.slot_adjust[i];
        slot_freqs[m * 512 + i] = a.slot_freqs[i];
        sym_id[m * 512 + i] = a.sym_id[i];
    }
    for (uint32_t j = tid; j < M; j += blockDim.x) remap[static_cast<uint64_t>(m) * M + j] = s_remap[j];
    if (tid == 0) flags[m] = (summed ? 1u : 0u) | (paired ? 2u : 0u);
}

}  // namespace

// n_models rows of 256 u16 frequencies (device memory) summing to M = 1 << sb; outputs per model: divider[256],
// slot_adjust[512], slot_freqs[512], sym_id[512], remap[M], flags (1: sums to M, 2: paired).  Returns the CUDA error.
extern "C" int pd_alias_tables(const uint16_t* rows, uint32_t n_models, uint32_t sb, uint32_t threads, uint32_t* divider,
                               uint32_t* slot_adjust, uint32_t* slot_freqs, uint8_t* sym_id, uint16_t* remap, uint32_t* flags)
{
    const uint32_t M = 1u << sb, smem = sizeof(AliasBuildSmem) + 2 * M;
    cudaFuncSetAttribute(batch_alias_tables, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    batch_alias_tables<<<n_models, threads, smem>>>(rows, M, divider, slot_adjust, slot_freqs, sym_id, remap, flags);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return static_cast<int>(e);
}

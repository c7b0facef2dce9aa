// steps.cu -- the device build of steps.inc: one kernel per entry, one thread per work item.  Every hd_* launcher
// takes device addresses, enqueues on the default stream and returns cudaGetLastError().
#include <cuda_runtime.h>

#define HD_ENTRY(name, params, args)                                                                   \
    __global__ void k_##name(uint64_t n, HD_UNPAREN params)                                            \
    {                                                                                                  \
        const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;                            \
        if (i < n) body_##name(i, HD_UNPAREN args);                                                    \
    }                                                                                                  \
    extern "C" int hd_##name(uint64_t n, HD_UNPAREN params)                                            \
    {                                                                                                  \
        if (n) k_##name<<<(unsigned)((n + 255) / 256), 256>>>(n, HD_UNPAREN args);                     \
        return (int)cudaGetLastError();                                                                \
    }

#include "steps.inc"

// The word tables live in shared memory, as a caller's decode kernel would keep them: block b builds the table of
// model b with one thread per symbol.  hd_word_tables copies each table out (slots as the u32 view of RansWordSlot).
__device__ void word_table_in_shared(RansWordTables* tab, const uint32_t* freqs, const uint32_t* cum)
{
    uint32_t* words = (uint32_t*)tab;
    for (uint32_t k = threadIdx.x; k < sizeof(RansWordTables) / 4; k += blockDim.x) words[k] = 0;
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < RANS_WORD_NSYMS; s += blockDim.x) body_word_row(s, tab, freqs, cum);
    __syncthreads();
}

__global__ void k_word_tables(const uint32_t* freqs, const uint32_t* cum, uint32_t* slots, uint8_t* slot2sym)
{
    __shared__ RansWordTables tab;
    const uint32_t b = blockIdx.x;
    word_table_in_shared(&tab, freqs + 256 * b, cum + 257 * b);
    for (uint32_t k = threadIdx.x; k < RANS_WORD_M; k += blockDim.x) {
        slots[RANS_WORD_M * b + k] = tab.slots[k].u32;
        slot2sym[RANS_WORD_M * b + k] = tab.slot2sym[k];
    }
}

extern "C" int hd_word_tables(uint64_t n_models, const uint32_t* freqs, const uint32_t* cum, uint32_t* slots,
                              uint8_t* slot2sym)
{
    if (n_models) k_word_tables<<<(unsigned)n_models, RANS_WORD_NSYMS>>>(freqs, cum, slots, slot2sym);
    return (int)cudaGetLastError();
}

__global__ void k_dec_word(uint64_t n, uint32_t nl, const uint32_t* freqs, const uint32_t* cum, HD_DEC_PARAMS)
{
    __shared__ RansWordTables tab;
    word_table_in_shared(&tab, freqs, cum);
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) body_dec_word(t, nl, &tab, HD_DEC_ARGS);
}

extern "C" int hd_dec_word(uint64_t n, uint32_t nl, const uint32_t* freqs, const uint32_t* cum, HD_DEC_PARAMS)
{
    if (n) k_dec_word<<<(unsigned)((n + 127) / 128), 128>>>(n, nl, freqs, cum, HD_DEC_ARGS);
    return (int)cudaGetLastError();
}

// rans_word_sse41.h -- word-renormalising rANS (32-bit state, 16-bit words, scale_bits 12):
// scalar coder, the 4-lane SSE4.1 decoder, and (under nvcc) the same scalar functions as
// __host__ __device__.
//
// Names, types and signatures are the reference's (rygorous/ryg_rans rans_word_sse41.h;
// lines cited) so main_simd.cpp compiles against this header unchanged.  This is the coder
// the GPU kernels implement warp-wide (csrc/word_kernels.cuh): RansSimdDecRenorm's
// "movemask -> shuffle the next k words to the k lanes that need them" is the 4-lane
// version of the kernels' ballot + popc(mask & lanemask_lt).
//
// Interval: state in [2^16, 2^32), one 16-bit word in or out per step at most, so
// renormalisation never iterates (ref :31-35).  Model resolution is fixed at 12 bits and
// the alphabet at 8 bits (ref :37-40); the decode table has one entry per slot.
#ifndef RANS_WORD_SSE41_HEADER
#define RANS_WORD_SSE41_HEADER

#include <stdint.h>
#include "rans_hd.h"
#if !defined(__CUDA_ARCH__)
#include <smmintrin.h>
#define RANS_WORD_HAVE_SSE41 1
#endif

#define RANS_WORD_L (1u << 16)
#define RANS_WORD_SCALE_BITS 12
#define RANS_WORD_M (1u << RANS_WORD_SCALE_BITS)
#define RANS_WORD_NSYMS 256

typedef uint32_t RansWordEnc;
typedef uint32_t RansWordDec;

union RansWordSlot {                     // ref :50-56
    uint32_t u32;
    struct {
        uint16_t freq;
        uint16_t bias;
    };
};

struct RansWordTables {                  // ref :58-61
    RansWordSlot slots[RANS_WORD_M];
    uint8_t slot2sym[RANS_WORD_M];
};

// one table row per code slot owned by `sym`                                  (ref :64-72)
RANS_HD void RansWordTablesInitSymbol(RansWordTables* tab, uint8_t sym, uint32_t start, uint32_t freq)
{
    RansWordSlot* row = tab->slots + start;
    uint8_t* owner = tab->slot2sym + start;
    for (uint32_t k = 0; k != freq; ++k) {
        row[k].freq = (uint16_t)freq;
        row[k].bias = (uint16_t)k;
        owner[k] = sym;
    }
}

RANS_HD RansWordEnc RansWordEncInit() { return RANS_WORD_L; }                  // ref :75

// ref :81-93.  Threshold is ((L >> 12) << 16) * freq evaluated in 32 bits, as the reference does.
RANS_HD void RansWordEncPut(RansWordEnc* r, uint16_t** pptr, uint32_t start, uint32_t freq)
{
    uint32_t x = *r;
    const uint32_t limit = ((RANS_WORD_L >> RANS_WORD_SCALE_BITS) << 16) * freq;
    if (x >= limit) {
        *--*pptr = (uint16_t)x;
        x >>= 16;
    }
    const uint32_t q = x / freq;
    *r = (q << RANS_WORD_SCALE_BITS) + (x - q * freq) + start;
}

RANS_HD void RansWordEncFlush(RansWordEnc* r, uint16_t** pptr)                 // ref :96
{
    uint16_t* p = *pptr - 2;
    p[0] = (uint16_t)*r;
    p[1] = (uint16_t)(*r >> 16);
    *pptr = p;
}

RANS_HD void RansWordDecInit(RansWordDec* r, uint16_t** pptr)                  // ref :109
{
    const uint16_t* p = *pptr;
    *r = (uint32_t)p[0] | ((uint32_t)p[1] << 16);
    *pptr += 2;
}

RANS_HD uint8_t RansWordDecSym(RansWordDec* r, RansWordTables const* tab)      // ref :123
{
    const uint32_t x = *r;
    const uint32_t slot = x % RANS_WORD_M;
    const RansWordSlot e = tab->slots[slot];
    *r = (uint32_t)e.freq * (x >> RANS_WORD_SCALE_BITS) + e.bias;
    return tab->slot2sym[slot];
}

RANS_HD void RansWordDecRenorm(RansWordDec* r, uint16_t** pptr)                // ref :134
{
    if (*r < RANS_WORD_L) *r = (*r << 16) | *(*pptr)++;
}

#if defined(RANS_WORD_HAVE_SSE41)

typedef union {                          // ref :45-48
    __m128i simd;
    uint32_t lane[4];
} RansSimdDec;

static inline void RansSimdDecInit(RansSimdDec* r, uint16_t** pptr)            // ref :144
{
    r->simd = _mm_loadu_si128((const __m128i*)*pptr);
    *pptr += 8;
}

// four table look-ups + one vector multiply-add                               (ref :151-179)
static inline uint32_t RansSimdDecSym(RansSimdDec* r, RansWordTables const* tab)
{
    const __m128i x = r->simd;
    uint32_t slot[4];
    _mm_storeu_si128((__m128i*)slot, _mm_and_si128(x, _mm_set1_epi32(RANS_WORD_M - 1)));

    const __m128i fb = _mm_set_epi32((int)tab->slots[slot[3]].u32, (int)tab->slots[slot[2]].u32,
                                     (int)tab->slots[slot[1]].u32, (int)tab->slots[slot[0]].u32);
    const __m128i freq = _mm_and_si128(fb, _mm_set1_epi32(0xffff));
    const __m128i bias = _mm_srli_epi32(fb, 16);
    r->simd = _mm_add_epi32(_mm_mullo_epi32(_mm_srli_epi32(x, RANS_WORD_SCALE_BITS), freq), bias);

    return (uint32_t)tab->slot2sym[slot[0]] | ((uint32_t)tab->slot2sym[slot[1]] << 8)
         | ((uint32_t)tab->slot2sym[slot[2]] << 16) | ((uint32_t)tab->slot2sym[slot[3]] << 24);
}

namespace rans_detail {

// For every 4-bit "lane needs a word" mask: the pshufb control that drops the k-th pending
// word into the low half of the k-th needy lane (0x80 = write zero), and the word count.
struct SimdRefillPlan {
    alignas(16) int8_t control[16][16];
    uint8_t words[16];
    constexpr SimdRefillPlan() : control(), words()
    {
        for (int mask = 0; mask < 16; mask++) {
            int next = 0;
            for (int lane = 0; lane < 4; lane++) {
                const bool needy = (mask >> lane) & 1;
                control[mask][4 * lane + 0] = needy ? (int8_t)(2 * next) : (int8_t)-128;
                control[mask][4 * lane + 1] = needy ? (int8_t)(2 * next + 1) : (int8_t)-128;
                control[mask][4 * lane + 2] = (int8_t)-128;
                control[mask][4 * lane + 3] = (int8_t)-128;
                next += needy ? 1 : 0;
            }
            words[mask] = (uint8_t)next;
        }
    }
};

}  // namespace rans_detail

// ref :182-227.  Reads 8 bytes at *pptr regardless of how many words are consumed: callers
// pad the stream end (main_simd.cpp:146).
static inline void RansSimdDecRenorm(RansSimdDec* r, uint16_t** pptr)
{
    static constexpr rans_detail::SimdRefillPlan plan{};
    const __m128i x = r->simd;
    // unsigned x < L  <=>  the high 16 bits are all zero
    const __m128i needy = _mm_cmpeq_epi32(_mm_srli_epi32(x, 16), _mm_setzero_si128());
    const int mask = _mm_movemask_ps(_mm_castsi128_ps(needy));
    const __m128i pending = _mm_loadl_epi64((const __m128i*)*pptr);
    const __m128i routed = _mm_shuffle_epi8(pending, _mm_load_si128((const __m128i*)plan.control[mask]));
    const __m128i refilled = _mm_or_si128(_mm_slli_epi32(x, 16), routed);
    r->simd = _mm_blendv_epi8(x, refilled, needy);
    *pptr += plan.words[mask];
}

#endif  // RANS_WORD_HAVE_SSE41

#endif  // RANS_WORD_SSE41_HEADER

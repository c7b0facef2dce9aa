// rans_byte.h -- byte-renormalising rANS step functions, host + sm_90a device.
//
// Source-level API of the GPU rANS package.  Every name, type and signature below is
// the reference's (rygorous/ryg_rans rans_byte.h; line numbers cited per function) so
// that main.cpp / main_alias.cpp-style callers compile against this header unchanged
// (tests/test_dropin_drivers.py does exactly that), and the same functions are usable
// inside CUDA kernels.  The bodies are this repo's own: one generic core
// (rans_detail::ByteCoder) with the reference names as thin wrappers.
//
// Conventions kept from the reference (rans_byte.h:17-42): encode symbols in reverse,
// the encoder's byte pointer moves DOWN from the end of the caller's buffer, decoders
// read upwards, any number of coders may share one byte stream.
#ifndef RANS_BYTE_HEADER
#define RANS_BYTE_HEADER

#include <stdint.h>
#include "rans_hd.h"

#ifdef assert
#define RansAssert assert
#else
#define RansAssert(x)
#endif

// lower bound of the normalisation interval: state lives in [2^23, 2^31)   (ref :50)
#define RANS_BYTE_L (1u << 23)

typedef uint32_t RansState;                                                // ref :53

typedef struct {                                                           // ref :159-165
    uint32_t x_max;      // renormalise while x >= x_max
    uint32_t rcp_freq;   // fixed-point reciprocal of freq
    uint32_t bias;
    uint16_t cmpl_freq;  // (1 << scale_bits) - freq
    uint16_t rcp_shift;
} RansEncSymbol;

typedef struct {                                                           // ref :168-171
    uint16_t start;
    uint16_t freq;
} RansDecSymbol;

namespace rans_detail {

struct ByteCoder {
    // push bytes out (low byte first, to descending addresses) until x < limit
    static RANS_HDM uint32_t shrink(uint32_t x, uint8_t** pptr, uint32_t limit)
    {
        uint8_t* p = *pptr;
        while (x >= limit) {
            *--p = (uint8_t)x;
            x >>= 8;
        }
        *pptr = p;
        return x;
    }
    // pull bytes in until x >= L
    static RANS_HDM uint32_t grow(uint32_t x, uint8_t** pptr)
    {
        uint8_t* p = *pptr;
        while (x < RANS_BYTE_L) x = (x << 8) | *p++;
        *pptr = p;
        return x;
    }
    static RANS_HDM uint32_t limit_for(uint32_t freq, uint32_t scale_bits) { return ((RANS_BYTE_L >> scale_bits) << 8) * freq; }
    static RANS_HDM uint32_t pop(uint32_t x, uint32_t start, uint32_t freq, uint32_t scale_bits)
    {
        return freq * (x >> scale_bits) + (x & ((1u << scale_bits) - 1)) - start;
    }
    static RANS_HDM void store32(uint8_t* p, uint32_t v)
    {
        for (int i = 0; i < 4; i++) p[i] = (uint8_t)(v >> (8 * i));
    }
    static RANS_HDM uint32_t load32(const uint8_t* p)
    {
        uint32_t v = 0;
        for (int i = 3; i >= 0; i--) v = (v << 8) | p[i];
        return v;
    }
};

}  // namespace rans_detail

RANS_HD void RansEncInit(RansState* r) { *r = RANS_BYTE_L; }                                       // ref :56

RANS_HD RansState RansEncRenorm(RansState x, uint8_t** pptr, uint32_t freq, uint32_t scale_bits)   // ref :62
{
    return rans_detail::ByteCoder::shrink(x, pptr, rans_detail::ByteCoder::limit_for(freq, scale_bits));
}

RANS_HD void RansEncPut(RansState* r, uint8_t** pptr, uint32_t start, uint32_t freq, uint32_t scale_bits)   // ref :83
{
    const RansState x = RansEncRenorm(*r, pptr, freq, scale_bits);
    *r = ((x / freq) << scale_bits) + (x % freq) + start;
}

RANS_HD void RansEncFlush(RansState* r, uint8_t** pptr)                                            // ref :93
{
    *pptr -= 4;
    rans_detail::ByteCoder::store32(*pptr, *r);
}

RANS_HD void RansDecInit(RansState* r, uint8_t** pptr)                                             // ref :109
{
    *r = rans_detail::ByteCoder::load32(*pptr);
    *pptr += 4;
}

RANS_HD uint32_t RansDecGet(RansState* r, uint32_t scale_bits) { return *r & ((1u << scale_bits) - 1); }   // ref :125

RANS_HD void RansDecAdvance(RansState* r, uint8_t** pptr, uint32_t start, uint32_t freq, uint32_t scale_bits)   // ref :133
{
    *r = rans_detail::ByteCoder::grow(rans_detail::ByteCoder::pop(*r, start, freq, scale_bits), pptr);
}

// Precompute the division-free encoder parameters for one symbol (ref :174-243).
// For freq >= 2: rcp = ceil(2^(31+k) / freq) with k = ceil(log2 freq) is an exact
// reciprocal for every 31-bit x (Alverson), so q = mulhi(x, rcp) >> (k - 1) == x / freq
// and x' = x + bias + q * (M - freq) == (x / freq) * M + x % freq + start.
// For freq == 1 the reciprocal would be 2^32; rcp = 2^32 - 1 gives q = x - 1 instead and
// the missing M - 1 is folded into bias.
RANS_HD void RansEncSymbolInit(RansEncSymbol* s, uint32_t start, uint32_t freq, uint32_t scale_bits)
{
    RansAssert(scale_bits <= 16);
    RansAssert(start <= (1u << scale_bits));
    RansAssert(freq <= (1u << scale_bits) - start);
    const uint32_t M = 1u << scale_bits;
    s->x_max = rans_detail::ByteCoder::limit_for(freq, scale_bits);
    s->cmpl_freq = (uint16_t)(M - freq);
    if (freq >= 2) {
        uint32_t k = 0;
        while ((1u << k) < freq) k++;
        s->rcp_freq = (uint32_t)(((1ull << (k + 31)) + freq - 1) / freq);
        s->rcp_shift = (uint16_t)(k - 1);
        s->bias = start;
    } else {
        s->rcp_freq = 0xffffffffu;
        s->rcp_shift = 0;
        s->bias = start + M - 1;
    }
}

RANS_HD void RansDecSymbolInit(RansDecSymbol* s, uint32_t start, uint32_t freq)                    // ref :246
{
    RansAssert(start <= (1 << 16));
    RansAssert(freq <= (1 << 16) - start);
    s->start = (uint16_t)start;
    s->freq = (uint16_t)freq;
}

RANS_HD void RansEncPutSymbol(RansState* r, uint8_t** pptr, RansEncSymbol const* sym)              // ref :258
{
    RansAssert(sym->x_max != 0);
    const uint32_t x = rans_detail::ByteCoder::shrink(*r, pptr, sym->x_max);
#if defined(__CUDA_ARCH__)
    const uint32_t q = __umulhi(x, sym->rcp_freq) >> sym->rcp_shift;
#else
    const uint32_t q = (uint32_t)(((uint64_t)x * sym->rcp_freq) >> 32) >> sym->rcp_shift;
#endif
    *r = x + sym->bias + q * sym->cmpl_freq;
}

RANS_HD void RansDecAdvanceSymbol(RansState* r, uint8_t** pptr, RansDecSymbol const* sym, uint32_t scale_bits)   // ref :283
{
    RansDecAdvance(r, pptr, sym->start, sym->freq, scale_bits);
}

RANS_HD void RansDecAdvanceStep(RansState* r, uint32_t start, uint32_t freq, uint32_t scale_bits)  // ref :291
{
    *r = rans_detail::ByteCoder::pop(*r, start, freq, scale_bits);
}

RANS_HD void RansDecAdvanceSymbolStep(RansState* r, RansDecSymbol const* sym, uint32_t scale_bits) // ref :301
{
    RansDecAdvanceStep(r, sym->start, sym->freq, scale_bits);
}

RANS_HD void RansDecRenorm(RansState* r, uint8_t** pptr)                                           // ref :307
{
    *r = rans_detail::ByteCoder::grow(*r, pptr);
}

#endif  // RANS_BYTE_HEADER

// rans_word_avx2.h -- 32-lane AVX2 decoder for the chunk streams the GPU encoder produces.
//
// SURVEY 8f.4: "host SIMD decoders for CPU-side consumption of GPU streams" -- the 16-way AVX2 decoder
// the reference's README mentions (README:120-122) but never shipped, taken to the interleave width the
// GPU uses.  A chunk stream of the bulk API (include/rans_b200.h) is exactly the reference's N-way word
// coder stream with N = 32 (rans_word_sse41.h semantics, scale_bits 12): this header decodes one with
// four __m256i of states, eight lanes each, and is bit-compatible with driving RansWordDecSym /
// RansWordDecRenorm (or the reference's own) for 32 lanes in order.
//
// This is a source-level header for HOST callers that receive a container and have no GPU.  It is NOT
// part of librans_b200.so and no rb200_* call ever routes through it: the GPU path has no CPU fallback.
//
//   RansWord32Tables tab;  RansWord32TablesInit(&tab, &word_tables);    // or Reset + InitSymbol per symbol
//   RansWord32DecodeChunk(stream, stream_bytes, &tab, out, m);          // m symbols of one chunk
//
// Streams need 16 readable bytes behind their end (the same kind of padding RansSimdDecRenorm asks for,
// main_simd.cpp:146); inside a container every stream but the last is followed by the next one, and a buffer
// holding rb200_container_pack output can simply be over-allocated by 16 bytes.
// (A two-__m512i variant with vpexpandd refills was measured at the same speed -- the gathers dominate -- and
// is not shipped.)
#ifndef RANS_WORD_AVX2_HEADER
#define RANS_WORD_AVX2_HEADER

#include <stdint.h>
#include <string.h>
#include <immintrin.h>
#include "rans_word_sse41.h"

#if !defined(__AVX2__)
#error "rans_word_avx2.h needs AVX2 (compile with -mavx2)"
#endif

#define RANS_WORD32_LANES 32

// One u32 per code slot: freq << 20 | bias << 8 | symbol -- RansWordSlot{freq,bias} (rans_word_sse41.h:50-56)
// and slot2sym fused, so that a decode step is ONE gather.  freq 4096 (a one-symbol model) does not fit
// 12 bits and is stored as 0; `wide` tells the step to map 0 back to 4096.
struct RansWord32Tables {
    uint32_t entry[RANS_WORD_M];
    int wide;
};

static inline void RansWord32TablesReset(RansWord32Tables* tab) { memset(tab, 0, sizeof *tab); }

// after RansWord32TablesReset: one call per symbol with freq > 0, like RansWordTablesInitSymbol (rans_word_sse41.h:64-72)
static inline void RansWord32TablesInitSymbol(RansWord32Tables* tab, uint8_t sym, uint32_t start, uint32_t freq)
{
    for (uint32_t k = 0; k != freq; ++k) tab->entry[start + k] = ((freq & 0xfffu) << 20) | (k << 8) | sym;
    if (freq == RANS_WORD_M) tab->wide = 1;
}

static inline void RansWord32TablesInit(RansWord32Tables* tab, RansWordTables const* src)
{
    tab->wide = 0;
    for (uint32_t s = 0; s != RANS_WORD_M; ++s) {
        const uint32_t freq = src->slots[s].freq, bias = src->slots[s].bias;
        tab->entry[s] = ((freq & 0xfffu) << 20) | (bias << 8) | src->slot2sym[s];
        if (freq == RANS_WORD_M) tab->wide = 1;
    }
}

typedef struct {
    __m256i v[4];              // lanes 0-7, 8-15, 16-23, 24-31
} RansWord32Dec;

// the flushed header: lane k's state is the little-endian u32 at byte 4k (main_simd.cpp:298-299 with N = 32)
static inline void RansWord32DecInit(RansWord32Dec* r, uint16_t** pptr)
{
    for (int g = 0; g < 4; g++) r->v[g] = _mm256_loadu_si256((const __m256i*)(*pptr + 16 * g));
    *pptr += 2 * RANS_WORD32_LANES;
}

namespace rans_detail {

// For every 8-bit "lane needs a word" mask: the vpermd control that routes the k-th pending word to the
// k-th needy lane, and the number of words consumed (the AVX2 form of RansSimdDecRenorm's pshufb table).
struct Avx2RefillPlan {
    alignas(32) uint32_t route[256][8];
    uint8_t words[256];
    Avx2RefillPlan()
    {
        for (int mask = 0; mask < 256; mask++) {
            uint32_t next = 0;
            for (int lane = 0; lane < 8; lane++) {
                route[mask][lane] = next;            // lanes that do not refill ignore what they are handed
                next += (mask >> lane) & 1;
            }
            words[mask] = (uint8_t)next;
        }
    }
};

inline const Avx2RefillPlan& avx2_refill_plan()
{
    static const Avx2RefillPlan plan;
    return plan;
}

// RansWordDecSym for eight lanes: one gather, returns the eight symbols in the low bytes of the dwords
static inline __m256i word32_step(__m256i* x, const RansWord32Tables* tab)
{
    const __m256i slot = _mm256_and_si256(*x, _mm256_set1_epi32(RANS_WORD_M - 1));
    const __m256i e = _mm256_i32gather_epi32((const int*)tab->entry, slot, 4);
    __m256i freq = _mm256_srli_epi32(e, 20);
    if (tab->wide) freq = _mm256_blendv_epi8(freq, _mm256_set1_epi32(RANS_WORD_M), _mm256_cmpeq_epi32(freq, _mm256_setzero_si256()));
    const __m256i bias = _mm256_and_si256(_mm256_srli_epi32(e, 8), _mm256_set1_epi32(0xfff));
    *x = _mm256_add_epi32(_mm256_mullo_epi32(_mm256_srli_epi32(*x, RANS_WORD_SCALE_BITS), freq), bias);
    return _mm256_and_si256(e, _mm256_set1_epi32(0xff));
}

// RansWordDecRenorm for eight lanes, restricted to the lanes set in `active` (all ones except in the ragged
// last step of a chunk).  Reads 16 bytes at *pptr whatever it consumes.
static inline void word32_renorm(__m256i* x, uint16_t** pptr, __m256i active, const Avx2RefillPlan& plan)
{
    const __m256i needy = _mm256_and_si256(active, _mm256_cmpeq_epi32(_mm256_srli_epi32(*x, 16), _mm256_setzero_si256()));
    const int mask = _mm256_movemask_ps(_mm256_castsi256_ps(needy));
    const __m256i pending = _mm256_cvtepu16_epi32(_mm_loadu_si128((const __m128i*)*pptr));
    const __m256i routed = _mm256_permutevar8x32_epi32(pending, _mm256_load_si256((const __m256i*)plan.route[mask]));
    const __m256i refilled = _mm256_or_si256(_mm256_slli_epi32(*x, 16), routed);
    *x = _mm256_blendv_epi8(*x, refilled, needy);
    *pptr += plan.words[mask];
}

// eight dword symbols -> eight bytes
static inline void word32_store8(uint8_t* out, __m256i sym)
{
    const __m256i packed = _mm256_shuffle_epi8(sym, _mm256_setr_epi8(0, 4, 8, 12, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1,
                                                                     0, 4, 8, 12, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1));
    const uint32_t lo = (uint32_t)_mm256_extract_epi32(packed, 0), hi = (uint32_t)_mm256_extract_epi32(packed, 4);
    memcpy(out, &lo, 4);
    memcpy(out + 4, &hi, 4);
}

}  // namespace rans_detail

// One full step: 32 symbols to out[0..32), then the 32 lanes renormalise in lane order.
static inline void RansWord32DecStep(RansWord32Dec* r, uint16_t** pptr, RansWord32Tables const* tab, uint8_t* out)
{
    const rans_detail::Avx2RefillPlan& plan = rans_detail::avx2_refill_plan();
    const __m256i all = _mm256_set1_epi32(-1);
    __m256i sym[4];
    for (int g = 0; g < 4; g++) sym[g] = rans_detail::word32_step(&r->v[g], tab);      // four independent gathers in flight
    for (int g = 0; g < 4; g++) {
        rans_detail::word32_store8(out + 8 * g, sym[g]);
        rans_detail::word32_renorm(&r->v[g], pptr, all, plan);
    }
}

// Decode the m symbols of one chunk.  Returns 0 when the stream is consumed exactly and every lane is back
// at the initial state (what the GPU decoder checks too), -1 otherwise.
static inline int RansWord32DecodeChunk(const uint8_t* stream, size_t stream_bytes, RansWord32Tables const* tab, uint8_t* out, size_t m)
{
    if (stream_bytes < 4 * RANS_WORD32_LANES || (stream_bytes & 1)) return -1;
    uint16_t* ptr = (uint16_t*)stream;
    uint16_t* const end = (uint16_t*)(stream + stream_bytes);
    RansWord32Dec r;
    RansWord32DecInit(&r, &ptr);
    const size_t steps = m / RANS_WORD32_LANES, rem = m % RANS_WORD32_LANES;
    const rans_detail::Avx2RefillPlan& plan = rans_detail::avx2_refill_plan();
    const __m256i all = _mm256_set1_epi32(-1);
    for (size_t s = 0; s < steps; s++) {
        __m256i sym[4];
        for (int g = 0; g < 4; g++) sym[g] = rans_detail::word32_step(&r.v[g], tab);
        for (int g = 0; g < 4; g++) {
            if (ptr > end) return -1;                   // a corrupt stream cannot run away: reads stay below end + 16
            rans_detail::word32_store8(out + RANS_WORD32_LANES * s + 8 * g, sym[g]);
            rans_detail::word32_renorm(&r.v[g], &ptr, all, plan);
        }
    }
    if (rem) {                                          // ragged last step: only lanes < rem decode and renormalise
        uint8_t tail[RANS_WORD32_LANES];
        for (int g = 0; g < 4; g++) {
            if (ptr > end) return -1;
            const __m256i lane = _mm256_add_epi32(_mm256_setr_epi32(0, 1, 2, 3, 4, 5, 6, 7), _mm256_set1_epi32(8 * g));
            const __m256i active = _mm256_cmpgt_epi32(_mm256_set1_epi32((int)rem), lane);
            __m256i x = r.v[g];
            const __m256i sym = rans_detail::word32_step(&x, tab);
            r.v[g] = _mm256_blendv_epi8(r.v[g], x, active);
            rans_detail::word32_store8(tail + 8 * g, sym);
            rans_detail::word32_renorm(&r.v[g], &ptr, active, plan);
        }
        memcpy(out + RANS_WORD32_LANES * steps, tail, rem);
    }
    if (ptr != end) return -1;
    const __m256i L = _mm256_set1_epi32((int)RANS_WORD_L);
    int ok = 1;
    for (int g = 0; g < 4; g++) ok &= _mm256_movemask_epi8(_mm256_cmpeq_epi32(r.v[g], L)) == -1;
    return ok ? 0 : -1;
}

// All chunks of a blob + directory as produced by rb200_encode / found by rb200_container_open.  Chunks are
// independent: callers that want threads split the range [0, n_chunks) themselves.  `blob` needs 16 readable bytes
// behind its end.  Returns 0, or -(1 + index of the first chunk that failed).
static inline long RansWord32DecodeChunks(const uint8_t* blob, const uint64_t* offsets, size_t first_chunk, size_t last_chunk,
                                          uint32_t chunk_syms, size_t n, RansWord32Tables const* tab, uint8_t* out)
{
    for (size_t c = first_chunk; c < last_chunk; c++) {
        const uint64_t lo = offsets[c], end = offsets[c + 1] & ~(uint64_t)15;
        const size_t first = c * (size_t)chunk_syms;
        const size_t m = n - first < chunk_syms ? n - first : chunk_syms;
        if (end < lo) return -(long)(1 + c);
        if (RansWord32DecodeChunk(blob + lo, (size_t)(end - lo), tab, out + first, m)) return -(long)(1 + c);
    }
    return 0;
}

#endif  // RANS_WORD_AVX2_HEADER

/*
 * rans_oracle.c -- CPU restatement of the ryg_rans hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This file is the parity oracle for the GPU kernels.  It is plain C99, single
 * threaded, and restates the reference algorithms in a deliberately simple
 * "array of lane states + one shared cursor" form, generalised from the
 * reference drivers' fixed N (1, 2, 8) to an arbitrary lane count N.
 * Nothing in the product path (ryg_rans_b200/, include/) may link or call it;
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg do.
 *
 * Parity status: PINNED.  tests/test_oracle.py checks every function below
 *   (a) against oracle/_ref (the reference's own headers + driver code compiled
 *       from /root/reference, see oracle/ref_harness_*.cpp) byte for byte, and
 *   (b) against the reference's known-answer compressed sizes for book1
 *       (README:48,62,82,96,110 -> 435113/435117/435116/435120/435626), and
 *   (c) against the committed golden fixtures in tests/golden/ (made by
 *       tests/golden/make_golden.py from oracle/_ref).
 *
 * Each function cites the reference file:line it follows.
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK            0
#define ORC_E_ARG        -1
#define ORC_E_MODEL      -2
#define ORC_E_SPACE      -3
#define ORC_E_STREAM     -4

/* ------------------------------------------------------------------------ */
/* Order-0 model: SymbolStats (main.cpp:49-129; identical copies in          */
/* main64.cpp:49-129, main_simd.cpp:49-129, main_alias.cpp:47-144)           */
/* ------------------------------------------------------------------------ */

/* main.cpp:59-66  count_freqs */
void orc_count_freqs(const uint8_t *in, size_t n, uint32_t freqs[256])
{
    memset(freqs, 0, 256 * sizeof(uint32_t));
    for (size_t i = 0; i < n; i++)
        freqs[in[i]] += 1;
}

/* main.cpp:68-73 calc_cum_freqs + main.cpp:75-129 normalize_freqs.
 * freqs[] in: raw counts; out: normalised.  cum[] out: 257 entries.
 * The reference asserts; the oracle returns an error code instead. */
int orc_normalize_freqs(uint32_t freqs[256], uint32_t cum[257], uint32_t target_total)
{
    if (target_total < 256)                      /* main.cpp:77 */
        return ORC_E_ARG;

    uint32_t run = 0;                            /* main.cpp:68-73 */
    for (int s = 0; s < 256; s++) {
        cum[s] = run;
        run += freqs[s];
    }
    cum[256] = run;
    const uint32_t total = run;                  /* main.cpp:80 */
    if (total == 0)
        return ORC_E_MODEL;                      /* reference would divide by 0 */

    for (int s = 1; s <= 256; s++)               /* main.cpp:83-84 */
        cum[s] = (uint32_t)(((uint64_t)target_total * cum[s]) / total);

    /* main.cpp:90-116: a symbol that occurs but was rounded to width 0 takes
     * one slot from the narrowest symbol that still has width > 1 (first such
     * symbol wins ties), and every boundary between them moves by one. */
    for (int s = 0; s < 256; s++) {
        if (freqs[s] == 0 || cum[s + 1] != cum[s])
            continue;
        uint32_t narrowest = UINT32_MAX;
        int donor = -1;
        for (int t = 0; t < 256; t++) {
            uint32_t w = cum[t + 1] - cum[t];
            if (w > 1 && w < narrowest) {
                narrowest = w;
                donor = t;
            }
        }
        if (donor < 0)
            return ORC_E_MODEL;                  /* main.cpp:104 */
        if (donor < s) {
            for (int t = donor + 1; t <= s; t++) /* main.cpp:107-109 */
                cum[t] -= 1;
        } else {
            for (int t = s + 1; t <= donor; t++) /* main.cpp:110-113 */
                cum[t] += 1;
        }
    }

    if (cum[0] != 0 || cum[256] != target_total) /* main.cpp:119 */
        return ORC_E_MODEL;
    for (int s = 0; s < 256; s++) {              /* main.cpp:120-128 */
        uint32_t w = cum[s + 1] - cum[s];
        if ((freqs[s] == 0) != (w == 0))
            return ORC_E_MODEL;
        freqs[s] = w;
    }
    return ORC_OK;
}

/* main.cpp:145-148: brute-force cumulative-frequency -> symbol table. */
void orc_build_cum2sym(const uint32_t cum[257], uint8_t *cum2sym)
{
    for (int s = 0; s < 256; s++)
        for (uint32_t i = cum[s]; i < cum[s + 1]; i++)
            cum2sym[i] = (uint8_t)s;
}

/* rans_word_sse41.h:64-72 RansWordTablesInitSymbol, applied to all 256 symbols
 * (main_simd.cpp:141-143).  slots[i] = freq | bias<<16 (little-endian view of
 * the RansWordSlot union, rans_word_sse41.h:50-56). */
void orc_word_tables(const uint32_t freqs[256], const uint32_t cum[257],
                     uint32_t slots[4096], uint8_t slot2sym[4096])
{
    for (int s = 0; s < 256; s++) {
        for (uint32_t i = 0; i < freqs[s]; i++) {
            uint32_t slot = cum[s] + i;
            slot2sym[slot] = (uint8_t)s;
            slots[slot] = (freqs[s] & 0xffffu) | (i << 16);
        }
    }
}

/* ------------------------------------------------------------------------ */
/* Word coder: 32-bit state, 16-bit renorm, L = 1<<16, scale_bits = 12       */
/* (rans_word_sse41.h:35-37)                                                 */
/* ------------------------------------------------------------------------ */

#define WORD_L      (1u << 16)
#define WORD_SB     12u
#define WORD_M      (1u << WORD_SB)

/* N-way interleaved encode.  Interleave policy = main_simd.cpp:287-300 with
 * 8 replaced by nlanes: symbol i goes to lane i % nlanes, symbols are walked
 * last to first, the stream grows downwards from the end of the buffer, and the
 * lanes are flushed nlanes-1 .. 0.  Per-symbol step = RansWordEncPut
 * (rans_word_sse41.h:81-93); flush = RansWordEncFlush (:96-106).
 * Returns the stream size in bytes; the stream is left at out[0..size). */
long orc_word_encode(const uint8_t *in, size_t n,
                     const uint32_t freqs[256], const uint32_t cum[257],
                     uint32_t nlanes, uint8_t *out, size_t cap)
{
    if (nlanes == 0)
        return ORC_E_ARG;
    size_t max_words = n + 2 * (size_t)nlanes;
    uint16_t *buf = (uint16_t *)malloc(max_words * sizeof(uint16_t));
    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    if (!buf || !x) { free(buf); free(x); return ORC_E_SPACE; }
    for (uint32_t k = 0; k < nlanes; k++)
        x[k] = WORD_L;                                   /* :75-78 */

    uint16_t *cur = buf + max_words;
    for (size_t i = n; i-- > 0;) {
        uint32_t s = in[i];
        uint32_t f = freqs[s];
        if (f == 0) { free(buf); free(x); return ORC_E_MODEL; }
        uint32_t v = x[i % nlanes];
        if (v >= ((WORD_L >> WORD_SB) << 16) * f) {      /* :85 */
            *--cur = (uint16_t)v;                        /* :86-87 */
            v >>= 16;                                    /* :88 */
        }
        x[i % nlanes] = ((v / f) << WORD_SB) + (v % f) + cum[s]; /* :92 */
    }
    for (uint32_t k = nlanes; k-- > 0;) {                /* main_simd.cpp:298-299 */
        cur -= 2;                                        /* :101-103 */
        cur[0] = (uint16_t)(x[k] & 0xffffu);
        cur[1] = (uint16_t)(x[k] >> 16);
    }
    size_t bytes = (size_t)((buf + max_words) - cur) * 2;
    long rv;
    if (bytes > cap) {
        rv = ORC_E_SPACE;
    } else {
        memcpy(out, cur, bytes);
        rv = (long)bytes;
    }
    free(buf);
    free(x);
    return rv;
}

/* N-way interleaved decode (main_simd.cpp:313-332 generalised): states are
 * read lane 0 first (RansWordDecInit, rans_word_sse41.h:109-120), then groups
 * of nlanes symbols are decoded (RansWordDecSym :123-131) and renormalised in
 * lane order (RansWordDecRenorm :134-141).  The reference's tail loop omits
 * the renorm; that is equivalent because the state of a lane after its last
 * symbol is exactly L (its encoder initial state) and so never refills.
 * Returns bytes consumed, or a negative error if the stream is too short. */
long orc_word_decode(const uint8_t *stream, size_t size,
                     const uint32_t freqs[256], const uint32_t cum[257],
                     uint32_t nlanes, uint8_t *out, size_t n)
{
    if (nlanes == 0 || (size & 1) || size < 4 * (size_t)nlanes)
        return ORC_E_ARG;
    static uint32_t slots[4096];
    static uint8_t slot2sym[4096];
    orc_word_tables(freqs, cum, slots, slot2sym);

    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    if (!x) return ORC_E_SPACE;
    const uint8_t *p = stream;
    const uint8_t *end = stream + size;
    for (uint32_t k = 0; k < nlanes; k++) {
        x[k] = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
        p += 4;
    }
    for (size_t i = 0; i < n; i++) {
        uint32_t v = x[i % nlanes];
        uint32_t slot = v & (WORD_M - 1);                           /* :126 */
        out[i] = slot2sym[slot];                                    /* :130 */
        v = (slots[slot] & 0xffffu) * (v >> WORD_SB) + (slots[slot] >> 16); /* :129 */
        if (v < WORD_L) {                                           /* :137 */
            if (p + 2 > end) { free(x); return ORC_E_STREAM; }
            v = (v << 16) | (uint32_t)p[0] | ((uint32_t)p[1] << 8); /* :138 */
            p += 2;
        }
        x[i % nlanes] = v;
    }
    free(x);
    return (long)(p - stream);
}

/* ------------------------------------------------------------------------ */
/* Byte coder: 31-bit state, byte renorm, L = 1<<23 (rans_byte.h:50)         */
/* ------------------------------------------------------------------------ */

#define BYTE_L (1u << 23)

typedef struct {
    uint32_t x_max, rcp_freq, bias;
    uint16_t cmpl_freq, rcp_shift;
} orc_enc_symbol;                               /* rans_byte.h:159-165 */

/* rans_byte.h:174-243 RansEncSymbolInit */
static void orc_enc_symbol_init(orc_enc_symbol *e, uint32_t start, uint32_t freq, uint32_t sb)
{
    e->x_max = ((BYTE_L >> sb) << 8) * freq;                 /* :197 */
    e->cmpl_freq = (uint16_t)((1u << sb) - freq);            /* :198 */
    if (freq < 2) {                                          /* :199-228 */
        e->rcp_freq = ~0u;
        e->rcp_shift = 0;
        e->bias = start + (1u << sb) - 1;
    } else {                                                 /* :229-242 */
        uint32_t shift = 0;
        while (freq > (1u << shift))
            shift++;
        e->rcp_freq = (uint32_t)(((1ull << (shift + 31)) + freq - 1) / freq);
        e->rcp_shift = (uint16_t)(shift - 1);
        e->bias = start;
    }
}

/* N-way byte-coder encode with the division-free step RansEncPutSymbol
 * (rans_byte.h:258-280), interleave policy of main.cpp:226-246 generalised
 * (for N=2 that driver special-cases the odd tail; "lane = i % N, walk
 * backwards, flush N-1..0" produces the identical order). */
long orc_byte_encode(const uint8_t *in, size_t n,
                     const uint32_t freqs[256], const uint32_t cum[257],
                     uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t cap)
{
    if (nlanes == 0 || scale_bits > 16 || scale_bits < 8)
        return ORC_E_ARG;
    orc_enc_symbol es[256];
    for (int s = 0; s < 256; s++)
        orc_enc_symbol_init(&es[s], cum[s], freqs[s], scale_bits);

    size_t max_bytes = 2 * n + 4 * (size_t)nlanes + 16;
    uint8_t *buf = (uint8_t *)malloc(max_bytes);
    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    if (!buf || !x) { free(buf); free(x); return ORC_E_SPACE; }
    for (uint32_t k = 0; k < nlanes; k++)
        x[k] = BYTE_L;                                       /* :56-59 */
    uint8_t *cur = buf + max_bytes;
    for (size_t i = n; i-- > 0;) {
        const orc_enc_symbol *e = &es[in[i]];
        if (e->x_max == 0) { free(buf); free(x); return ORC_E_MODEL; } /* :260 */
        uint32_t v = x[i % nlanes];
        while (v >= e->x_max) {                              /* :265-272 */
            *--cur = (uint8_t)(v & 0xff);
            v >>= 8;
        }
        uint32_t q = (uint32_t)(((uint64_t)v * e->rcp_freq) >> 32) >> e->rcp_shift; /* :278 */
        x[i % nlanes] = v + e->bias + q * e->cmpl_freq;      /* :279 */
    }
    for (uint32_t k = nlanes; k-- > 0;) {                    /* :93-105 */
        cur -= 4;
        cur[0] = (uint8_t)(x[k] >> 0);
        cur[1] = (uint8_t)(x[k] >> 8);
        cur[2] = (uint8_t)(x[k] >> 16);
        cur[3] = (uint8_t)(x[k] >> 24);
    }
    size_t bytes = (size_t)((buf + max_bytes) - cur);
    long rv = ORC_E_SPACE;
    if (bytes <= cap) { memcpy(out, cur, bytes); rv = (long)bytes; }
    free(buf); free(x);
    return rv;
}

/* N-way byte-coder decode: RansDecGet (rans_byte.h:125-128) -> cum2sym
 * (main.cpp:200) -> RansDecAdvanceSymbolStep (:291-304) -> RansDecRenorm
 * (:307-318), lanes in order (main.cpp:259-280 generalised). */
long orc_byte_decode(const uint8_t *stream, size_t size,
                     const uint32_t freqs[256], const uint32_t cum[257],
                     uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t n)
{
    if (nlanes == 0 || scale_bits > 16 || scale_bits < 8 || size < 4 * (size_t)nlanes)
        return ORC_E_ARG;
    uint8_t *cum2sym = (uint8_t *)malloc((size_t)1 << scale_bits);
    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    if (!cum2sym || !x) { free(cum2sym); free(x); return ORC_E_SPACE; }
    orc_build_cum2sym(cum, cum2sym);
    const uint32_t mask = (1u << scale_bits) - 1;
    const uint8_t *p = stream, *end = stream + size;
    for (uint32_t k = 0; k < nlanes; k++) {                  /* :109-122 */
        x[k] = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
        p += 4;
    }
    long rv = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t v = x[i % nlanes];
        uint32_t s = cum2sym[v & mask];
        out[i] = (uint8_t)s;
        v = freqs[s] * (v >> scale_bits) + (v & mask) - cum[s];  /* :297 */
        while (v < BYTE_L) {                                     /* :311-315 */
            if (p >= end) { rv = ORC_E_STREAM; goto done; }
            v = (v << 8) | *p++;
        }
        x[i % nlanes] = v;
    }
    rv = (long)(p - stream);
done:
    free(cum2sym); free(x);
    return rv;
}

/* ------------------------------------------------------------------------ */
/* Alias-table model + coder (main_alias.cpp:47-267)                         */
/* ------------------------------------------------------------------------ */

typedef struct {
    uint32_t divider[256];        /* main_alias.cpp:56 */
    uint32_t slot_adjust[512];    /* :57 */
    uint32_t slot_freqs[512];     /* :58 */
    uint8_t  sym_id[512];         /* :59 */
} orc_alias_tables;

/* main_alias.cpp:147-237 make_alias_table.  remap must hold sum entries
 * (sum = cum[256]).  Returns 0 or an error where the reference asserts. */
int orc_alias_build(const uint32_t freqs[256], const uint32_t cum[257],
                    orc_alias_tables *t, uint32_t *remap)
{
    const uint32_t sum = cum[256];
    if (sum == 0 || (sum % 256) != 0)                   /* :151 */
        return ORC_E_MODEL;
    const uint32_t tgt = sum / 256;                     /* :155 */

    uint32_t left[256];                                 /* :159-165 */
    for (int i = 0; i < 256; i++) {
        left[i] = freqs[i];
        t->divider[i] = tgt;
        t->sym_id[2 * i] = (uint8_t)i;
        t->sym_id[2 * i + 1] = (uint8_t)i;
    }

    /* Vose sweep, :170-204.  "big" walks symbols that still hold >= tgt slots,
     * "small" walks symbols holding < tgt; each small bucket is topped up from
     * the current big one.  A big symbol that drops below tgt and lies behind
     * the small cursor is revisited immediately. */
    int big = 0, small = 0;
    while (big < 256 && left[big] < tgt) big++;         /* :172-173 */
    while (small < 256 && left[small] >= tgt) small++;  /* :174-175 */
    int peek = small + 1;                               /* :179 */
    while (big < 256 && small < 256) {                  /* :183 */
        t->sym_id[2 * small] = (uint8_t)big;            /* :185 */
        t->divider[small] = left[small];                /* :186 */
        left[big] -= tgt - t->divider[small];           /* :189 */
        if (left[big] >= tgt || peek <= big) {          /* :192 */
            small = peek;
            while (small < 256 && left[small] >= tgt) small++;
            peek = small + 1;
        } else {
            small = big;                                /* :199 */
        }
        while (big < 256 && left[big] < tgt) big++;     /* :202-203 */
    }

    /* slot distribution, :207-232 */
    uint32_t placed[256];
    memset(placed, 0, sizeof placed);
    for (int i = 0; i < 256; i++) {
        int j = t->sym_id[2 * i];
        uint32_t h0 = t->divider[i];
        uint32_t h1 = tgt - h0;
        uint32_t b0 = placed[i];
        uint32_t b1 = placed[j];
        uint32_t c0 = cum[i] + b0;
        uint32_t c1 = cum[j] + b1;
        t->divider[i] = (uint32_t)i * tgt + h0;                    /* :219 */
        t->slot_freqs[2 * i + 1] = freqs[i];                       /* :221 */
        t->slot_freqs[2 * i] = freqs[j];                           /* :222 */
        t->slot_adjust[2 * i + 1] = (uint32_t)i * tgt - b0;        /* :223 */
        t->slot_adjust[2 * i] = (uint32_t)i * tgt - (b1 - h0);     /* :224 */
        for (uint32_t k = 0; k < h0; k++)                          /* :225-226 */
            remap[c0 + k] = k + (uint32_t)i * tgt;
        for (uint32_t k = 0; k < h1; k++)                          /* :227-228 */
            remap[c1 + k] = (k + h0) + (uint32_t)i * tgt;
        placed[i] += h0;                                           /* :230-231 */
        placed[j] += h1;
    }
    for (int i = 0; i < 256; i++)                                  /* :235-236 */
        if (placed[i] != freqs[i])
            return ORC_E_MODEL;
    return ORC_OK;
}

/* N-way alias encode: RansEncPutAlias (main_alias.cpp:241-250) =
 * RansEncRenorm (rans_byte.h:62-74) + true divide + alias_remap gather;
 * interleave as main_alias.cpp:353-373 generalised. */
long orc_alias_encode(const uint8_t *in, size_t n,
                      const uint32_t freqs[256], const uint32_t cum[257],
                      uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t cap)
{
    if (nlanes == 0 || scale_bits > 16 || scale_bits < 8 || cum[256] != (1u << scale_bits))
        return ORC_E_ARG;
    orc_alias_tables *t = (orc_alias_tables *)malloc(sizeof *t);
    uint32_t *remap = (uint32_t *)malloc(((size_t)1 << scale_bits) * sizeof(uint32_t));
    size_t max_bytes = 2 * n + 4 * (size_t)nlanes + 16;
    uint8_t *buf = (uint8_t *)malloc(max_bytes);
    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    long rv = ORC_E_SPACE;
    if (!t || !remap || !buf || !x) goto done;
    if (orc_alias_build(freqs, cum, t, remap) != ORC_OK) { rv = ORC_E_MODEL; goto done; }
    for (uint32_t k = 0; k < nlanes; k++)
        x[k] = BYTE_L;
    uint8_t *cur = buf + max_bytes;
    for (size_t i = n; i-- > 0;) {
        uint32_t s = in[i];
        uint32_t f = freqs[s];
        if (f == 0) { rv = ORC_E_MODEL; goto done; }
        uint32_t v = x[i % nlanes];
        uint32_t x_max = ((BYTE_L >> scale_bits) << 8) * f;     /* rans_byte.h:64 */
        while (v >= x_max) {                                    /* :65-72 */
            *--cur = (uint8_t)(v & 0xff);
            v >>= 8;
        }
        x[i % nlanes] = ((v / f) << scale_bits) + remap[(v % f) + cum[s]]; /* main_alias.cpp:249 */
    }
    for (uint32_t k = nlanes; k-- > 0;) {
        cur -= 4;
        cur[0] = (uint8_t)(x[k] >> 0);
        cur[1] = (uint8_t)(x[k] >> 8);
        cur[2] = (uint8_t)(x[k] >> 16);
        cur[3] = (uint8_t)(x[k] >> 24);
    }
    {
        size_t bytes = (size_t)((buf + max_bytes) - cur);
        if (bytes <= cap) { memcpy(out, cur, bytes); rv = (long)bytes; }
    }
done:
    free(t); free(remap); free(buf); free(x);
    return rv;
}

/* N-way alias decode: RansDecGetAlias (main_alias.cpp:252-267) followed by
 * RansDecRenorm (rans_byte.h:307-318), lanes in order (:386-405 generalised). */
long orc_alias_decode(const uint8_t *stream, size_t size,
                      const uint32_t freqs[256], const uint32_t cum[257],
                      uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t n)
{
    if (nlanes == 0 || scale_bits > 16 || scale_bits < 8 || size < 4 * (size_t)nlanes
        || cum[256] != (1u << scale_bits))
        return ORC_E_ARG;
    orc_alias_tables *t = (orc_alias_tables *)malloc(sizeof *t);
    uint32_t *remap = (uint32_t *)malloc(((size_t)1 << scale_bits) * sizeof(uint32_t));
    uint32_t *x = (uint32_t *)malloc(nlanes * sizeof(uint32_t));
    long rv = ORC_E_SPACE;
    if (!t || !remap || !x) goto done;
    if (orc_alias_build(freqs, cum, t, remap) != ORC_OK) { rv = ORC_E_MODEL; goto done; }
    {
        const uint32_t mask = (1u << scale_bits) - 1;
        const uint8_t *p = stream, *end = stream + size;
        for (uint32_t k = 0; k < nlanes; k++) {
            x[k] = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
            p += 4;
        }
        for (size_t i = 0; i < n; i++) {
            uint32_t v = x[i % nlanes];
            uint32_t xm = v & mask;                                 /* :258 */
            uint32_t bucket = xm >> (scale_bits - 8);               /* :259 */
            uint32_t b2 = 2 * bucket + (xm < t->divider[bucket]);   /* :260-262 */
            v = t->slot_freqs[b2] * (v >> scale_bits) + xm - t->slot_adjust[b2]; /* :265 */
            out[i] = t->sym_id[b2];                                 /* :266 */
            while (v < BYTE_L) {
                if (p >= end) { rv = ORC_E_STREAM; goto done; }
                v = (v << 8) | *p++;
            }
            x[i % nlanes] = v;
        }
        rv = (long)(p - stream);
    }
done:
    free(t); free(remap); free(x);
    return rv;
}

/* ------------------------------------------------------------------------ */
/* rans64: 63-bit state, 32-bit renorm, L = 1<<31 (rans64.h:59)              */
/* ------------------------------------------------------------------------ */

#define R64_L (1ull << 31)

/* N-way rans64 encode.  Step = Rans64EncPut (rans64.h:77-93); the reference
 * driver uses the reciprocal form Rans64EncPutSymbol (:262-278), which is
 * constructed to give the identical quotient (:239-241), so the oracle uses the
 * plain divide.  Flush :96-103.  Interleave main64.cpp:228-248 generalised.
 * Words are written native-endian like the reference (README:12). */
long orc_rans64_encode(const uint8_t *in, size_t n,
                       const uint32_t freqs[256], const uint32_t cum[257],
                       uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t cap)
{
    if (nlanes == 0 || scale_bits > 31)
        return ORC_E_ARG;
    size_t max_words = n + 2 * (size_t)nlanes + 4;
    uint32_t *buf = (uint32_t *)malloc(max_words * sizeof(uint32_t));
    uint64_t *x = (uint64_t *)malloc(nlanes * sizeof(uint64_t));
    if (!buf || !x) { free(buf); free(x); return ORC_E_SPACE; }
    for (uint32_t k = 0; k < nlanes; k++)
        x[k] = R64_L;                                            /* :65-68 */
    uint32_t *cur = buf + max_words;
    for (size_t i = n; i-- > 0;) {
        uint32_t s = in[i];
        uint32_t f = freqs[s];
        if (f == 0) { free(buf); free(x); return ORC_E_MODEL; }  /* :79 */
        uint64_t v = x[i % nlanes];
        uint64_t x_max = ((R64_L >> scale_bits) << 32) * f;      /* :83 */
        if (v >= x_max) {                                        /* :84-89 */
            *--cur = (uint32_t)v;
            v >>= 32;
        }
        x[i % nlanes] = ((v / f) << scale_bits) + (v % f) + cum[s]; /* :92 */
    }
    for (uint32_t k = nlanes; k-- > 0;) {                        /* :96-103 */
        cur -= 2;
        cur[0] = (uint32_t)(x[k] >> 0);
        cur[1] = (uint32_t)(x[k] >> 32);
    }
    size_t bytes = (size_t)((buf + max_words) - cur) * 4;
    long rv = ORC_E_SPACE;
    if (bytes <= cap) { memcpy(out, cur, bytes); rv = (long)bytes; }
    free(buf); free(x);
    return rv;
}

/* N-way rans64 decode: Rans64DecInit (:107-115), Rans64DecGet (:118-121),
 * cum2sym (main64.cpp:202), Rans64DecAdvanceSymbolStep (:289-302),
 * Rans64DecRenorm (:305-316); lanes in order (main64.cpp:261-282). */
long orc_rans64_decode(const uint8_t *stream, size_t size,
                       const uint32_t freqs[256], const uint32_t cum[257],
                       uint32_t scale_bits, uint32_t nlanes, uint8_t *out, size_t n)
{
    if (nlanes == 0 || scale_bits > 24 || (size & 3) || size < 8 * (size_t)nlanes)
        return ORC_E_ARG;
    uint8_t *cum2sym = (uint8_t *)malloc((size_t)1 << scale_bits);
    uint64_t *x = (uint64_t *)malloc(nlanes * sizeof(uint64_t));
    if (!cum2sym || !x) { free(cum2sym); free(x); return ORC_E_SPACE; }
    orc_build_cum2sym(cum, cum2sym);
    const uint64_t mask = (1ull << scale_bits) - 1;
    const uint8_t *p = stream, *end = stream + size;
    for (uint32_t k = 0; k < nlanes; k++) {
        uint32_t lo, hi;
        memcpy(&lo, p, 4); memcpy(&hi, p + 4, 4);
        x[k] = (uint64_t)lo | ((uint64_t)hi << 32);
        p += 8;
    }
    long rv = 0;
    for (size_t i = 0; i < n; i++) {
        uint64_t v = x[i % nlanes];
        uint32_t s = cum2sym[v & mask];
        out[i] = (uint8_t)s;
        v = freqs[s] * (v >> scale_bits) + (v & mask) - cum[s];  /* :297 */
        if (v < R64_L) {                                         /* :309-313 */
            if (p + 4 > end) { rv = ORC_E_STREAM; goto done; }
            uint32_t w;
            memcpy(&w, p, 4);
            v = (v << 32) | w;
            p += 4;
        }
        x[i % nlanes] = v;
    }
    rv = (long)(p - stream);
done:
    free(cum2sym); free(x);
    return rv;
}

/* ------------------------------------------------------------------------ */
/* Chunked container used by the GPU path (DESIGN.md section 3, mirrors the    */
/* statement in include/rans_b200.h): the symbol buffer is cut into chunks of */
/* chunk_syms symbols; every chunk is an independent nlanes-way stream exactly */
/* as produced by the *_encode functions above.  Streams are END-aligned:      */
/* stream c occupies blob[offsets[c] .. E_c) with E_c = E_{c-1} +              */
/* round_up(size_c, align), E_{-1} = 0; the gap in front of it is zero;        */
/* offsets[n_chunks] = E_last.  coder: 0 = word (scale 12), 1 = byte/cum2sym,  */
/* 2 = alias, 3 = rans64.                                                      */
/* ------------------------------------------------------------------------ */

static long one_encode(int coder, const uint8_t *in, size_t n, const uint32_t *freqs,
                       const uint32_t *cum, uint32_t sb, uint32_t nl, uint8_t *out, size_t cap)
{
    switch (coder) {
    case 0: return orc_word_encode(in, n, freqs, cum, nl, out, cap);
    case 1: return orc_byte_encode(in, n, freqs, cum, sb, nl, out, cap);
    case 2: return orc_alias_encode(in, n, freqs, cum, sb, nl, out, cap);
    case 3: return orc_rans64_encode(in, n, freqs, cum, sb, nl, out, cap);
    }
    return ORC_E_ARG;
}

static long one_decode(int coder, const uint8_t *st, size_t size, const uint32_t *freqs,
                       const uint32_t *cum, uint32_t sb, uint32_t nl, uint8_t *out, size_t n)
{
    switch (coder) {
    case 0: return orc_word_decode(st, size, freqs, cum, nl, out, n);
    case 1: return orc_byte_decode(st, size, freqs, cum, sb, nl, out, n);
    case 2: return orc_alias_decode(st, size, freqs, cum, sb, nl, out, n);
    case 3: return orc_rans64_decode(st, size, freqs, cum, sb, nl, out, n);
    }
    return ORC_E_ARG;
}

long orc_chunked_encode(int coder, const uint8_t *in, size_t n,
                        const uint32_t freqs[256], const uint32_t cum[257],
                        uint32_t scale_bits, uint32_t nlanes, size_t chunk_syms, size_t align,
                        uint8_t *blob, size_t cap, uint64_t *offsets)
{
    if (chunk_syms == 0 || align == 0)
        return ORC_E_ARG;
    size_t n_chunks = (n + chunk_syms - 1) / chunk_syms;
    size_t tmp_cap = 2 * chunk_syms + 16 * (size_t)nlanes + 256;
    uint8_t *tmp = (uint8_t *)malloc(tmp_cap);
    if (!tmp) return ORC_E_SPACE;
    size_t end_prev = 0;
    long rv = 0;
    for (size_t c = 0; c < n_chunks; c++) {
        size_t lo = c * chunk_syms;
        size_t m = (n - lo < chunk_syms) ? n - lo : chunk_syms;
        long r = one_encode(coder, in + lo, m, freqs, cum, scale_bits, nlanes, tmp, tmp_cap);
        if (r < 0) { rv = r; goto done; }
        size_t padded = ((size_t)r + align - 1) / align * align;
        size_t end = end_prev + padded;
        if (end > cap) { rv = ORC_E_SPACE; goto done; }
        offsets[c] = end - (size_t)r;
        memset(blob + end_prev, 0, padded - (size_t)r);
        memcpy(blob + offsets[c], tmp, (size_t)r);
        end_prev = end;
    }
    offsets[n_chunks] = end_prev;
    rv = (long)end_prev;
done:
    free(tmp);
    return rv;
}

long orc_chunked_decode(int coder, const uint8_t *blob, size_t blob_size, const uint64_t *offsets,
                        const uint32_t freqs[256], const uint32_t cum[257],
                        uint32_t scale_bits, uint32_t nlanes, size_t chunk_syms, size_t align,
                        uint8_t *out, size_t n)
{
    if (chunk_syms == 0 || align == 0)
        return ORC_E_ARG;
    size_t n_chunks = (n + chunk_syms - 1) / chunk_syms;
    for (size_t c = 0; c < n_chunks; c++) {
        size_t lo = c * chunk_syms;
        size_t m = (n - lo < chunk_syms) ? n - lo : chunk_syms;
        uint64_t end = offsets[c + 1] / align * align;
        if (end > blob_size || offsets[c] > end) return ORC_E_STREAM;
        long r = one_decode(coder, blob + offsets[c], (size_t)(end - offsets[c]),
                            freqs, cum, scale_bits, nlanes, out + lo, m);
        if (r < 0) return r;
        if ((uint64_t)r != end - offsets[c]) return ORC_E_STREAM;   /* must end exactly at E_c */
    }
    return (long)n;
}

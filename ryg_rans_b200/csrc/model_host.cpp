// model_host.cpp -- host-side order-0 model construction for the GPU rANS coder.
//
// Model construction is setup, not hot path, but it decides every table entry and
// therefore every bit of the stream, so it has to reproduce the reference's
// SymbolStats exactly (SURVEY H7):
//   count_freqs / calc_cum_freqs / normalize_freqs   main.cpp:59-129
//   RansWordTablesInitSymbol                         rans_word_sse41.h:64-72
//   make_alias_table                                 main_alias.cpp:147-237
// The reference asserts on bad input; this library returns RB200_E_MODEL.
#include "rans_b200.h"
#include "tables.h"

#include <algorithm>
#include <cstring>
#include <vector>

extern "C" int rb200_count_freqs(const uint8_t* in, size_t n, uint32_t freqs[256])
{
    if (!freqs || (!in && n)) return RB200_E_ARG;
    // four interleaved sub-histograms: same result as main.cpp:59-66, fewer
    // store-to-load stalls on runs of equal bytes
    uint32_t h[4][256];
    std::memset(h, 0, sizeof h);
    size_t i = 0;
    for (; i + 4 <= n; i += 4) {
        h[0][in[i]]++; h[1][in[i + 1]]++; h[2][in[i + 2]]++; h[3][in[i + 3]]++;
    }
    for (; i < n; i++) h[0][in[i]]++;
    for (int s = 0; s < 256; s++) freqs[s] = h[0][s] + h[1][s] + h[2][s] + h[3][s];
    return RB200_OK;
}

extern "C" int rb200_normalize_freqs(uint32_t freqs[256], uint32_t cum[257], uint32_t target_total)
{
    if (!freqs || !cum) return RB200_E_ARG;
    if (target_total < 256) return RB200_E_ARG;                   // main.cpp:77

    // prefix sums of the raw counts (main.cpp:68-73)
    cum[0] = 0;
    for (int s = 0; s < 256; s++) cum[s + 1] = cum[s] + freqs[s];
    const uint32_t raw_total = cum[256];
    if (raw_total == 0) return RB200_E_MODEL;

    // rescale the boundaries, 64-bit intermediate (main.cpp:83-84)
    for (int s = 1; s <= 256; s++)
        cum[s] = static_cast<uint32_t>((static_cast<uint64_t>(target_total) * cum[s]) / raw_total);

    // give every occurring-but-squashed symbol one slot, taken from the symbol with
    // the smallest width > 1 (lowest index on ties); boundaries in between shift by
    // one (main.cpp:90-116).  Order dependent, so done in symbol order.
    for (int s = 0; s < 256; s++) {
        if (!freqs[s] || cum[s + 1] > cum[s]) continue;
        int victim = -1;
        uint32_t victim_width = 0xffffffffu;
        for (int t = 0; t < 256; t++) {
            const uint32_t width = cum[t + 1] - cum[t];
            if (width > 1 && width < victim_width) { victim = t; victim_width = width; }
        }
        if (victim < 0) return RB200_E_MODEL;                     // main.cpp:104
        if (victim < s) for (int t = victim + 1; t <= s; t++) cum[t]--;
        else            for (int t = s + 1; t <= victim; t++) cum[t]++;
    }

    if (cum[0] != 0 || cum[256] != target_total) return RB200_E_MODEL;   // main.cpp:119
    for (int s = 0; s < 256; s++) {
        const uint32_t width = cum[s + 1] - cum[s];
        if ((freqs[s] != 0) != (width != 0)) return RB200_E_MODEL;       // main.cpp:120-124
        freqs[s] = width;                                                // main.cpp:127
    }
    return RB200_OK;
}

extern "C" int rb200_word_tables_build(const uint32_t freqs[256], const uint32_t cum[257],
                                       uint32_t slots[4096], uint8_t slot2sym[4096])
{
    if (!freqs || !cum || !slots || !slot2sym) return RB200_E_ARG;
    if (cum[0] != 0 || cum[256] != 4096) return RB200_E_MODEL;
    for (int s = 0; s < 256; s++) {
        if (cum[s + 1] - cum[s] != freqs[s] || cum[s] > 4096 || freqs[s] > 4096 - cum[s]) return RB200_E_MODEL;
        for (uint32_t k = 0; k < freqs[s]; k++) {                 // rans_word_sse41.h:66-71
            slots[cum[s] + k] = (freqs[s] & 0xffffu) | (k << 16);
            slot2sym[cum[s] + k] = static_cast<uint8_t>(s);
        }
    }
    return RB200_OK;
}

extern "C" int rb200_alias_tables_build(const uint32_t freqs[256], const uint32_t cum[257],
                                        uint32_t divider[256], uint32_t slot_adjust[512],
                                        uint32_t slot_freqs[512], uint8_t sym_id[512], uint32_t* alias_remap)
{
    if (!freqs || !cum || !divider || !slot_adjust || !slot_freqs || !sym_id || !alias_remap) return RB200_E_ARG;
    const uint32_t total = cum[256];
    if (total == 0 || total % 256u != 0) return RB200_E_MODEL;    // main_alias.cpp:151-152
    const uint32_t bucket = total / 256u;                         // :155
    uint32_t rest[256], given[256];
    const bool ok = rb200::alias_tables_core(freqs, bucket, divider, slot_adjust, slot_freqs, sym_id, rest, given);

    // alias_remap (main_alias.cpp:225-228): bucket s gives its own part to symbol s and the rest to its partner, each
    // after what earlier buckets gave that symbol -- the bases slot_adjust was formed from (:223-224)
    for (int s = 0; s < 256; s++) {
        const uint32_t lo = static_cast<uint32_t>(s) * bucket;
        const uint32_t own = divider[s] - lo, lent = bucket - own;
        const int other = sym_id[2 * s];
        const uint32_t own_base = lo - slot_adjust[2 * s + 1], other_base = lo + own - slot_adjust[2 * s];
        uint32_t* dst_own = alias_remap + cum[s] + own_base;
        for (uint32_t k = 0; k < own; k++) dst_own[k] = lo + k;
        uint32_t* dst_other = alias_remap + cum[other] + other_base;
        for (uint32_t k = 0; k < lent; k++) dst_other[k] = lo + own + k;
    }
    return ok ? RB200_OK : RB200_E_MODEL;
}

// ---------------------------------------------------------------------------
// Device table images (formats documented in tables.h)
// ---------------------------------------------------------------------------

namespace rb200 {

static uint32_t ceil_log2(uint32_t v)
{
    uint32_t s = 0;
    while ((1u << s) < v) s++;
    return s;
}

int build_word_device_tables(const uint32_t freqs[256], WordDeviceTables& t)
{
    uint32_t cum[257];
    cum[0] = 0;
    for (int s = 0; s < 256; s++) {
        if (freqs[s] > 4096) return RB200_E_MODEL;
        cum[s + 1] = cum[s] + freqs[s];
    }
    if (cum[256] != 4096) return RB200_E_MODEL;
    t.wide = 0;
    t.enc32_ok = 1;
    for (int s = 0; s < 256; s++) {
        const uint32_t f = freqs[s];
        if (f == 4096) t.wide = 1;
        for (uint32_t k = 0; k < f; k++)                               // decode: one u32 per slot
            t.dec[cum[s] + k] = word_dec_entry(static_cast<uint32_t>(s), f, k);
        // encode: exact x / f for any 32-bit x by the round-up reciprocal
        //   M = ceil(2^(32+sh) / f) = 2^32 + magic,  q = (x + mulhi(x, magic)) >> sh
        if (f == 0) {
            t.enc[s] = {0u, kEncBadSymbol};
            t.enc32[s] = {0u, kEncBadSymbol};
        } else {
            const uint32_t sh = ceil_log2(f);
            const unsigned __int128 one = 1;
            const unsigned __int128 M = ((one << (32 + sh)) + f - 1) / f;
            const uint32_t magic = static_cast<uint32_t>(M - (one << 32));
            t.enc[s] = {magic, f | (cum[s] << 13) | (sh << 25)};
            // 32-bit reciprocal, exact on x < f << 20 (see tables.h)
            if (f == 1) {
                t.enc32[s] = {0xffffffffu, f | (cum[s] << 13)};
            } else {
                const uint32_t s32 = sh - 1;
                const uint64_t pow = 1ull << (32 + s32);
                const uint64_t M32 = (pow + f - 1) / f;                    // < 2^32 because 2^s32 < f
                const uint64_t err = M32 * f - pow;                        // < f
                const uint64_t xmax = (static_cast<uint64_t>(f) << 20) - 1;
                if (M32 >> 32 || xmax * err >= pow) t.enc32_ok = 0;
                t.enc32[s] = {static_cast<uint32_t>(M32), f | (cum[s] << 13) | (s32 << 25)};
            }
        }
    }
    return RB200_OK;
}

int build_alias_device_tables(const uint32_t freqs[256], uint32_t scale_bits, AliasDeviceTables& t)
{
    if (scale_bits < 8 || scale_bits > 16) return RB200_E_ARG;
    uint32_t cum[257];
    cum[0] = 0;
    for (int s = 0; s < 256; s++) {
        if (freqs[s] > (1u << scale_bits)) return RB200_E_MODEL;
        cum[s + 1] = cum[s] + freqs[s];
    }
    if (cum[256] != (1u << scale_bits)) return RB200_E_MODEL;
    uint32_t divider[256], slot_adjust[512], slot_freqs[512];
    uint8_t sym_id[512];
    std::vector<uint32_t> remap(cum[256]);
    int rc = rb200_alias_tables_build(freqs, cum, divider, slot_adjust, slot_freqs, sym_id, remap.data());
    if (rc != RB200_OK) return rc;
    t.scale_bits = scale_bits;
    for (uint32_t b = 0; b < 256; b++) t.dec[b] = alias_dec_entry(b, divider, slot_adjust, slot_freqs, sym_id);
    t.remap.resize(cum[256]);
    for (uint32_t i = 0; i < cum[256]; i++) t.remap[i] = static_cast<uint16_t>(remap[i]);
    for (int s = 0; s < 256; s++) {
        const uint32_t f = freqs[s];
        if (f == 0) {
            t.enc[s] = {0u, 0u, 0u, kEncBadSymbol};
        } else {
            // same round-up reciprocal as the word coder: exact for every 32-bit x
            const uint32_t sh = ceil_log2(f);
            const unsigned __int128 one = 1;
            const unsigned __int128 M = ((one << (32 + sh)) + f - 1) / f;
            t.enc[s] = {static_cast<uint32_t>(M - (one << 32)), f, cum[s], sh};
        }
    }
    return RB200_OK;
}

int build_byte_device_tables(const uint32_t freqs[256], uint32_t scale_bits, ByteDeviceTables& t)
{
    if (scale_bits < 8 || scale_bits > 16) return RB200_E_ARG;
    const uint32_t M = 1u << scale_bits;
    uint32_t cum[257];
    cum[0] = 0;
    for (int s = 0; s < 256; s++) {
        if (freqs[s] >= 65536u || freqs[s] > M) return RB200_E_MODEL;   // RansDecSymbol.freq is 16 bits wide
        cum[s + 1] = cum[s] + freqs[s];
    }
    if (cum[256] != M) return RB200_E_MODEL;
    t.scale_bits = scale_bits;
    t.dec.assign(M + 1024, 0);
    uint32_t* dsyms = reinterpret_cast<uint32_t*>(t.dec.data() + M);
    for (int s = 0; s < 256; s++) {
        std::memset(t.dec.data() + cum[s], s, freqs[s]);                // cum2sym, main.cpp:145-148
        dsyms[s] = byte_dec_symbol(cum[s], freqs[s]);                   // RansDecSymbolInit, rans_byte.h:246-252
        const uint32_t f = freqs[s];
        const uint32_t x_max = ((1u << 23 >> scale_bits) << 8) * (f ? f : 1);    // rans_byte.h:197
        if (f == 0) {           // never valid to encode (rans_byte.h:260): act like freq 1, flag it
            t.enc[s] = {x_max, 0xffffffffu, M - 1, ((M - 1) & 0xffffu) | kEncBadSymbol};
        } else if (f == 1) {    // rans_byte.h:199-228
            t.enc[s] = {x_max, 0xffffffffu, cum[s] + M - 1, (M - 1) & 0xffffu};
        } else {                // rans_byte.h:229-242
            const uint32_t sh = ceil_log2(f);
            const uint32_t rcp = static_cast<uint32_t>(((1ull << (sh + 31)) + f - 1) / f);
            t.enc[s] = {x_max, rcp, cum[s], ((M - f) & 0xffffu) | ((sh - 1) << 16)};
        }
    }
    return RB200_OK;
}

int build_rans64_device_tables(const uint32_t freqs[256], uint32_t scale_bits, Rans64DeviceTables& t)
{
    if (scale_bits < 8 || scale_bits > 16) return RB200_E_ARG;
    const uint32_t M = 1u << scale_bits;
    uint32_t cum[257];
    cum[0] = 0;
    for (int s = 0; s < 256; s++) {
        if (freqs[s] > M) return RB200_E_MODEL;
        cum[s + 1] = cum[s] + freqs[s];
    }
    if (cum[256] != M) return RB200_E_MODEL;
    t.scale_bits = scale_bits;
    t.dec.assign(M + 2048, 0);
    uint32_t* dsyms = reinterpret_cast<uint32_t*>(t.dec.data() + M);
    for (int s = 0; s < 256; s++) {
        std::memset(t.dec.data() + cum[s], s, freqs[s]);                // cum2sym, main64.cpp:145-148
        dsyms[2 * s] = cum[s];                                          // Rans64DecSymbolInit, rans64.h:250-256
        dsyms[2 * s + 1] = freqs[s];
        const uint32_t f = freqs[s];
        uint64_t rcp;
        uint32_t shift, bias, flag = 0;
        if (f < 2) {                                                    // rans64.h:199-228 (freq 0: same, flagged)
            rcp = ~0ull;
            shift = 0;
            bias = (f ? cum[s] : 0) + M - 1;
            if (f == 0) flag = kEncBadSymbol;
        } else {                                                        // rans64.h:229-246
            const uint32_t k = ceil_log2(f);
            const unsigned __int128 one = 1;
            rcp = static_cast<uint64_t>(((one << (k + 63)) + f - 1) / f);
            shift = k - 1;
            bias = cum[s];
        }
        const uint32_t fe = f ? f : 1;
        const uint32_t e[8] = {static_cast<uint32_t>(rcp), static_cast<uint32_t>(rcp >> 32), fe, bias, M - fe, shift | flag, 0, 0};
        std::memcpy(t.enc[s], e, sizeof e);
    }
    return RB200_OK;
}

}  // namespace rb200

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
        // encode: exact x / f by the round-up reciprocal, 33-bit (any x) and 32-bit (x < f << 20) forms (tables.h)
        t.enc[s] = word_enc_entry(f, cum[s]);
        t.enc32[s] = word_enc32_entry(f, cum[s], &t.enc32_ok);
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
    for (int s = 0; s < 256; s++) t.enc[s] = alias_enc_entry(freqs[s], cum[s]);
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
        t.enc[s] = byte_enc_entry(freqs[s], cum[s], scale_bits);
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
        rans64_enc_entry(freqs[s], cum[s], scale_bits, t.enc[s]);
    }
    return RB200_OK;
}

}  // namespace rb200

// tables.h -- host images of the device-side coding tables (internal).
#pragma once
#include <cstdint>
#include <vector>

#include "hd.h"

namespace rb200 {

// marks a symbol the model gives frequency 0; the encoder flags RB200_E_SYMBOL
constexpr uint32_t kEncBadSymbol = 0x80000000u;

// The per-entry formulas of the decode tables below.  The host builders (model_host.cpp) and the device build of
// rb200_container_decode_async (container_decode.cuh) both call them, so both produce the same bytes.
// word: slot k of symbol s with frequency f (4096 is stored as 0, see WordDeviceTables)
RB200_HD inline uint32_t word_dec_entry(uint32_t s, uint32_t f, uint32_t k) { return ((f & 0xfffu) << 20) | (k << 8) | s; }
// byte: symbol s's RansDecSymbol {start, freq} (freq < 65536)
RB200_HD inline uint32_t byte_dec_symbol(uint32_t start, uint32_t f) { return start | (f << 16); }

// The per-entry formulas of the encode tables below, shared the same way by the host builders and the device model
// build of rb200_container_model_encode_async (model_kernels.cuh).  f <= 65536 and cum <= 65536 throughout.
RB200_HD inline uint32_t ceil_log2(uint32_t v)
{
    uint32_t s = 0;
    while ((1u << s) < v) s++;
    return s;
}
// ceil(2^(32 + sh) / f), sh = ceil_log2(f): the round-up reciprocal of the word and alias encoders, in [2^32, 2^33)
// (2^(32 + sh) <= 2^48, so 64 bits hold it exactly)
RB200_HD inline uint64_t rcp33(uint32_t f, uint32_t sh) { return ((1ull << (32 + sh)) + f - 1) / f; }

// ---- word coder (rans_word_sse41.h semantics, scale_bits 12)
//
// decode: one u32 per slot, 16 KiB: (freq & 0xfff) << 20 | bias << 8 | symbol.
//   It fuses RansWordSlot{freq,bias} and slot2sym (rans_word_sse41.h:50-61) so the
//   decode step is ONE shared-memory gather.  freq == 4096 (single-symbol model)
//   does not fit 12 bits; `wide` selects a kernel variant that maps 0 -> 4096.
// encode: per symbol {magic, freq | start << 13 | shift << 25}: exact division
//   q = (x + mulhi(x, magic)) >> shift for any 32-bit x (round-up reciprocal),
//   replacing the hardware divide of RansWordEncPut (rans_word_sse41.h:92).
//   `enc32` is the same table with a 32-bit reciprocal: the encoder only divides states x < freq << 20
//   (RansWordEncPut renormalises first), and on that range q = mulhi(x, M32) >> s32 with
//   M32 = ceil(2^(32+s32) / freq), s32 = ceil(log2 freq) - 1 is exact for every freq <= 2963 and most above
//   (checked per symbol: (freq * 2^20 - 1) * (M32 * freq - 2^(32+s32)) < 2^(32+s32)); three instructions
//   fewer per symbol.  freq 1 uses M32 = 2^32 - 1, which yields x - 1; the kernel adds the missing
//   1 * (4096 - 1) to `start`.  `enc32_ok` says every symbol of the model passed the check.
struct WordEncEntry { uint32_t magic, packed; };

// symbol s of frequency f starting at cum: its `enc` entry (33-bit reciprocal: exact for any 32-bit x)
RB200_HD inline WordEncEntry word_enc_entry(uint32_t f, uint32_t cum)
{
    if (f == 0) return {0u, kEncBadSymbol};
    const uint32_t sh = ceil_log2(f);
    return {static_cast<uint32_t>(rcp33(f, sh)), f | (cum << 13) | (sh << 25)};     // magic = M - 2^32
}
// its `enc32` entry (32-bit reciprocal, exact on x < f << 20); clears *exact when the check fails for f
RB200_HD inline WordEncEntry word_enc32_entry(uint32_t f, uint32_t cum, int* exact)
{
    if (f == 0) return {0u, kEncBadSymbol};
    if (f == 1) return {0xffffffffu, f | (cum << 13)};
    const uint32_t s32 = ceil_log2(f) - 1;
    const uint64_t pow = 1ull << (32 + s32);
    const uint64_t M32 = (pow + f - 1) / f;                    // < 2^32 because 2^s32 < f
    const uint64_t err = M32 * f - pow;                        // < f
    const uint64_t xmax = (static_cast<uint64_t>(f) << 20) - 1;
    if (M32 >> 32 || xmax * err >= pow) *exact = 0;
    return {static_cast<uint32_t>(M32), f | (cum << 13) | (s32 << 25)};
}

struct WordDeviceTables {
    uint32_t dec[4096];
    WordEncEntry enc[256];
    WordEncEntry enc32[256];
    int wide;
    int enc32_ok;
};
int build_word_device_tables(const uint32_t freqs[256], WordDeviceTables& t);

// ---- alias coder (main_alias.cpp semantics over the rans_byte.h state machine)
//
// decode: ONE 16-byte entry per bucket (main_alias.cpp:55-59 fused from four gathers to one):
//   w0 = divider[b]
//   w1 = slot_freqs[2b]   << 8 | sym_id[2b]           (taken when xm >= divider; slot_freqs <= 65536: 25 bits)
//   w2 = slot_freqs[2b+1] << 8 | sym_id[2b+1]         (taken when xm <  divider)
//   (the symbol in the low byte is what STG.U8 stores; the frequency is one shift away)
//   w3 = (slot_adjust[2b] & 0xffff) | (slot_adjust[2b+1] & 0xffff) << 16
//   xm - slot_adjust is the position inside the symbol's range, < freq <= 65536, so 16 bits of
//   the adjust are enough: bias = (xm - adjust16) & 0xffff.
// encode: per symbol {magic, freq, cum, shift} (same exact-division scheme) and
//   alias_remap as u16 (values < 65536; SURVEY H8) = 128 KiB at scale_bits 16.
struct AliasDecEntry { uint32_t divider, alt0, alt1, adjust; };
struct AliasEncEntry { uint32_t magic, freq, cum, shift; };

// alias: symbol s's encode entry (the word coder's round-up reciprocal: exact for every 32-bit x)
RB200_HD inline AliasEncEntry alias_enc_entry(uint32_t f, uint32_t cum)
{
    if (f == 0) return {0u, 0u, 0u, kEncBadSymbol};
    const uint32_t sh = ceil_log2(f);
    return {static_cast<uint32_t>(rcp33(f, sh)), f, cum, sh};
}

// bucket b's decode entry from the arrays of alias_tables_core
RB200_HD inline AliasDecEntry alias_dec_entry(uint32_t b, const uint32_t* divider, const uint32_t* slot_adjust, const uint32_t* slot_freqs,
                                              const uint8_t* sym_id)
{
    return {divider[b], (slot_freqs[2 * b] << 8) | sym_id[2 * b], (slot_freqs[2 * b + 1] << 8) | sym_id[2 * b + 1],
            (slot_adjust[2 * b] & 0xffffu) | (slot_adjust[2 * b + 1] << 16)};
}

// make_alias_table (main_alias.cpp:147-237) up to what decode needs: divider[256], slot_adjust[512], slot_freqs[512] and
// sym_id[512] for frequencies that sum to 256 * bucket.  alias_remap, which only the encoder needs, follows from these
// (rb200_alias_tables_build).  rest and given are 256 words of scratch each.  False if the pairing does not hand out
// exactly every symbol's frequency (main_alias.cpp:235-236).  Sequential by nature: one thread runs it.
RB200_HD inline bool alias_tables_core(const uint32_t* freqs, uint32_t bucket, uint32_t* divider, uint32_t* slot_adjust,
                                       uint32_t* slot_freqs, uint8_t* sym_id, uint32_t* rest, uint32_t* given)
{
    // Phase 1 (main_alias.cpp:159-204): pair every under-full symbol with an over-full donor.  rest[] is what each
    // symbol still has to hand out.
    for (int s = 0; s < 256; s++) {
        rest[s] = freqs[s];
        divider[s] = bucket;
        sym_id[2 * s] = sym_id[2 * s + 1] = static_cast<uint8_t>(s);
        given[s] = 0;
    }
    int donor = 0, taker = 0;
    while (donor < 256 && rest[donor] < bucket) donor++;          // :172-173
    while (taker < 256 && rest[taker] >= bucket) taker++;         // :174-175
    int resume = taker + 1;                                       // :179
    while (donor < 256 && taker < 256) {                          // :183
        sym_id[2 * taker] = static_cast<uint8_t>(donor);          // :185
        divider[taker] = rest[taker];                             // :186
        rest[donor] -= bucket - divider[taker];                   // :189
        if (rest[donor] >= bucket || resume <= donor) {           // :192
            taker = resume;
            while (taker < 256 && rest[taker] >= bucket) taker++;
            resume = taker + 1;
        } else {
            taker = donor;                                        // :199 (donor became a taker behind us)
        }
        while (donor < 256 && rest[donor] < bucket) donor++;      // :202-203
    }

    // Phase 2 (main_alias.cpp:207-232): hand out code slots bucket by bucket.
    for (int s = 0; s < 256; s++) {
        const int other = sym_id[2 * s];
        const uint32_t own = divider[s], lent = bucket - own;
        const uint32_t own_base = given[s], other_base = given[other];
        const uint32_t lo = static_cast<uint32_t>(s) * bucket;
        divider[s] = lo + own;                                    // :219
        slot_freqs[2 * s + 1] = freqs[s];                         // :221
        slot_freqs[2 * s] = freqs[other];                         // :222
        slot_adjust[2 * s + 1] = lo - own_base;                   // :223
        slot_adjust[2 * s] = lo - (other_base - own);             // :224
        given[s] += own;                                          // :230-231
        given[other] += lent;
    }
    for (int s = 0; s < 256; s++)
        if (given[s] != freqs[s]) return false;                   // :235-236
    return true;
}
struct AliasDeviceTables {
    uint32_t scale_bits;
    AliasDecEntry dec[256];
    AliasEncEntry enc[256];
    std::vector<uint16_t> remap;
};
int build_alias_device_tables(const uint32_t freqs[256], uint32_t scale_bits, AliasDeviceTables& t);

// ---- byte coder with cum2sym (main.cpp semantics over rans_byte.h), scale_bits 8..16
//
// decode: cum2sym[1 << scale_bits] (main.cpp:145-148) followed by 256 x u32 {start | freq << 16}
//   (= RansDecSymbol, rans_byte.h:168-171; like the reference's u16 field, freq must be < 65536).
// encode: RansEncSymbol images (rans_byte.h:159-165, built as RansEncSymbolInit :174-243 does)
//   stored in AliasEncEntry's four words: {x_max, rcp_freq, bias, cmpl_freq | rcp_shift << 16}.
struct ByteDeviceTables {
    uint32_t scale_bits;
    std::vector<uint8_t> dec;          // (1 << scale_bits) + 1024 bytes
    AliasEncEntry enc[256];
};
int build_byte_device_tables(const uint32_t freqs[256], uint32_t scale_bits, ByteDeviceTables& t);

// symbol s's RansEncSymbol image (RansEncSymbolInit, rans_byte.h:174-243)
RB200_HD inline AliasEncEntry byte_enc_entry(uint32_t f, uint32_t cum, uint32_t scale_bits)
{
    const uint32_t M = 1u << scale_bits;
    const uint32_t x_max = ((1u << 23 >> scale_bits) << 8) * (f ? f : 1);      // rans_byte.h:197
    if (f == 0) return {x_max, 0xffffffffu, M - 1, ((M - 1) & 0xffffu) | kEncBadSymbol};   // never valid to encode (:260): freq 1, flagged
    if (f == 1) return {x_max, 0xffffffffu, cum + M - 1, (M - 1) & 0xffffu};              // :199-228
    const uint32_t sh = ceil_log2(f);                                                      // :229-242
    const uint32_t rcp = static_cast<uint32_t>(((1ull << (sh + 31)) + f - 1) / f);
    return {x_max, rcp, cum, ((M - f) & 0xffffu) | ((sh - 1) << 16)};
}

// ---- rans64 (main64.cpp semantics over rans64.h), scale_bits 8..16
//
// decode: cum2sym[1 << scale_bits] followed by 256 x {u32 start, u32 freq} (= Rans64DecSymbol, rans64.h:151-154)
// encode: 256 x 32 B: {rcp_lo, rcp_hi, freq, bias}, {cmpl_freq, rcp_shift, 0, 0} (= Rans64EncSymbol, rans64.h:142-148,
//   built as Rans64EncSymbolInit :167-247 does); bit 31 of rcp_shift marks a symbol outside the model.
struct Rans64DeviceTables {
    uint32_t scale_bits;
    std::vector<uint8_t> dec;          // (1 << scale_bits) + 2048 bytes
    uint32_t enc[256][8];
};
int build_rans64_device_tables(const uint32_t freqs[256], uint32_t scale_bits, Rans64DeviceTables& t);

// ceil(2^(k + 63) / f) for 2 <= f <= 2^16, k = ceil_log2(f): in [2^63, 2^64).  Long division in base 2^32 of
// 2^(k - 1) * 2^64 (the top digit is below f), so that 64-bit arithmetic gives the exact quotient.
RB200_HD inline uint64_t rcp64(uint32_t f, uint32_t k)
{
    const uint64_t t1 = (1ull << (k - 1)) << 32;              // < f * 2^32
    const uint64_t q1 = t1 / f, t0 = (t1 % f) << 32;
    const uint64_t q0 = t0 / f;
    return ((q1 << 32) | q0) + (t0 % f != 0);
}
// symbol s's Rans64EncSymbol image, 8 words (Rans64EncSymbolInit, rans64.h:167-247)
RB200_HD inline void rans64_enc_entry(uint32_t f, uint32_t cum, uint32_t scale_bits, uint32_t e[8])
{
    const uint32_t M = 1u << scale_bits;
    uint64_t rcp;
    uint32_t shift, bias, flag = 0;
    if (f < 2) {                                                // rans64.h:199-228 (freq 0: same, flagged)
        rcp = ~0ull;
        shift = 0;
        bias = (f ? cum : 0) + M - 1;
        if (f == 0) flag = kEncBadSymbol;
    } else {                                                    // rans64.h:229-246
        const uint32_t k = ceil_log2(f);
        rcp = rcp64(f, k);
        shift = k - 1;
        bias = cum;
    }
    const uint32_t fe = f ? f : 1;
    e[0] = static_cast<uint32_t>(rcp);
    e[1] = static_cast<uint32_t>(rcp >> 32);
    e[2] = fe;
    e[3] = bias;
    e[4] = M - fe;
    e[5] = shift | flag;
    e[6] = 0;
    e[7] = 0;
}

}  // namespace rb200

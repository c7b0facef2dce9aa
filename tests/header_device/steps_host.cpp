// steps_host.cpp -- the host twin of steps.cu: the same entries of steps.inc as a host loop over the item index,
// plus RansAliasTablesInit (host-only set-up code) for the alias models.
#include <string.h>

#define HD_ENTRY(name, params, args)                                                                   \
    extern "C" int hd_##name(uint64_t n, HD_UNPAREN params)                                            \
    {                                                                                                  \
        for (uint64_t i = 0; i < n; i++) body_##name(i, HD_UNPAREN args);                              \
        return 0;                                                                                      \
    }

#include "steps.inc"

static void word_table(RansWordTables* tab, const uint32_t* freqs, const uint32_t* cum)
{
    memset(tab, 0, sizeof *tab);
    for (uint32_t s = 0; s < RANS_WORD_NSYMS; s++) body_word_row(s, tab, freqs, cum);
}

extern "C" int hd_word_tables(uint64_t n_models, const uint32_t* freqs, const uint32_t* cum, uint32_t* slots,
                              uint8_t* slot2sym)
{
    static RansWordTables tab;
    for (uint64_t b = 0; b < n_models; b++) {
        word_table(&tab, freqs + 256 * b, cum + 257 * b);
        for (uint32_t k = 0; k < RANS_WORD_M; k++) {
            slots[RANS_WORD_M * b + k] = tab.slots[k].u32;
            slot2sym[RANS_WORD_M * b + k] = tab.slot2sym[k];
        }
    }
    return 0;
}

extern "C" int hd_dec_word(uint64_t n, uint32_t nl, const uint32_t* freqs, const uint32_t* cum, HD_DEC_PARAMS)
{
    static RansWordTables tab;
    word_table(&tab, freqs, cum);
    for (uint64_t t = 0; t < n; t++) body_dec_word(t, nl, &tab, HD_DEC_ARGS);
    return 0;
}

// The alias tables of one model, built by RansAliasTablesInit with alias_remap = remap (cum[256] entries).
extern "C" int hd_alias_init(const uint32_t* freqs, const uint32_t* cum, RansAliasTables* t, uint32_t* remap)
{
    memset(t, 0, sizeof *t);
    memcpy(t->freqs, freqs, sizeof t->freqs);
    memcpy(t->cum_freqs, cum, sizeof t->cum_freqs);
    t->alias_remap = remap;
    return RansAliasTablesInit(t);
}

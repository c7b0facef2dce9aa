// Differential test of include/rans_alias.h against the reference's own alias code, which lives in its driver
// (main_alias.cpp: SymbolStats::make_alias_table, RansEncPutAlias, RansDecGetAlias).  REFDIR is replaced by the
// reference checkout's path at build time (oracle/Makefile); the driver is #included where it lies (its main renamed), nothing is copied.
// system headers first, outside the namespaces: their include guards then make the driver's own #includes no-ops
#include <stdio.h>
#include <stdarg.h>
#include <stdlib.h>
#include <stdint.h>
#include <string.h>
#include <assert.h>
#include <time.h>
#ifndef __STDC_FORMAT_MACROS
#define __STDC_FORMAT_MACROS
#endif
#include <inttypes.h>
#include <x86intrin.h>

#include <new>
#include <random>
#include <vector>

namespace ref {
#define main ref_driver_main_alias
#include "REFDIR/main_alias.cpp"
#undef main
}
#undef RANS_BYTE_HEADER
#undef RansAssert
#undef RANS_BYTE_L
namespace ours {
#include "rans_alias.h"
}

static int run(uint64_t seed, uint32_t scale_bits, size_t n)
{
    std::mt19937_64 rng(seed);
    std::vector<uint8_t> in(n);
    for (size_t i = 0; i < n; i++) {
        const uint64_t r = rng();
        in[i] = (uint8_t)((r & 0xff) & ((r >> 8) & 0xff) & (seed % 3 ? 0xff : (r >> 16) & 0xff));      // skewed
    }
    ref::SymbolStats st;
    st.count_freqs(in.data(), n);
    st.normalize_freqs(1u << scale_bits);
    st.make_alias_table();

    // 1. the tables
    ours::RansAliasTables t;
    memcpy(t.freqs, st.freqs, sizeof t.freqs);
    memcpy(t.cum_freqs, st.cum_freqs, sizeof t.cum_freqs);
    std::vector<uint32_t> remap(st.cum_freqs[256]);
    t.alias_remap = remap.data();
    if (ours::RansAliasTablesInit(&t) != 0) { printf("RansAliasTablesInit failed\n"); return 1; }
    if (memcmp(t.divider, st.divider, sizeof t.divider) || memcmp(t.slot_adjust, st.slot_adjust, sizeof t.slot_adjust) ||
        memcmp(t.slot_freqs, st.slot_freqs, sizeof t.slot_freqs) || memcmp(t.sym_id, st.sym_id, sizeof t.sym_id) ||
        memcmp(remap.data(), st.alias_remap, remap.size() * sizeof(uint32_t))) {
        printf("alias tables differ (seed %llu, scale_bits %u)\n", (unsigned long long)seed, scale_bits);
        return 1;
    }

    // 2. the two step functions, on the reference's SymbolStats and on our tables: streams and states must be identical
    const size_t cap = 2 * n + 64;
    std::vector<uint8_t> a(cap), b(cap), c(cap);
    uint8_t *pa = a.data() + cap, *pb = b.data() + cap, *pc = c.data() + cap;
    ref::RansState ra; ref::RansEncInit(&ra);
    ours::RansState rb, rc; ours::RansEncInit(&rb); ours::RansEncInit(&rc);
    for (size_t i = n; i-- > 0;) {
        ref::RansEncPutAlias(&ra, &pa, &st, in[i], scale_bits);
        ours::RansEncPutAlias(&rb, &pb, &st, in[i], scale_bits);          // our function on the driver's own struct
        ours::RansEncPutAlias(&rc, &pc, &t, in[i], scale_bits);           // and on RansAliasTables
        if (ra != rb || ra != rc) { printf("encoder state differs at %zu\n", i); return 1; }
    }
    ref::RansEncFlush(&ra, &pa); ours::RansEncFlush(&rb, &pb); ours::RansEncFlush(&rc, &pc);
    const size_t len = a.data() + cap - pa;
    if ((size_t)(b.data() + cap - pb) != len || (size_t)(c.data() + cap - pc) != len || memcmp(pa, pb, len) || memcmp(pa, pc, len)) {
        printf("streams differ\n");
        return 1;
    }
    uint8_t *qa = pa, *qb = pb;
    ref::RansState da; ref::RansDecInit(&da, &qa);
    ours::RansState db; ours::RansDecInit(&db, &qb);
    for (size_t i = 0; i < n; i++) {
        const uint32_t sa = ref::RansDecGetAlias(&da, &st, scale_bits);
        const uint32_t sb = ours::RansDecGetAlias(&db, &t, scale_bits);
        ref::RansDecRenorm(&da, &qa); ours::RansDecRenorm(&db, &qb);
        if (sa != sb || sa != in[i] || da != db || (qa - pa) != (qb - pb)) { printf("decoder differs at %zu\n", i); return 1; }
    }
    printf("rans_alias.h ok: seed %llu scale_bits %u: %zu symbols, %zu stream bytes identical\n", (unsigned long long)seed, scale_bits, n, len);
    return 0;
}

int main()
{
    int bad = 0;
    for (uint64_t seed = 1; seed <= 4; seed++)
        for (uint32_t sb : {8u, 11u, 14u, 16u}) bad += run(seed, sb, 20000 + 997 * seed);
    return bad;
}

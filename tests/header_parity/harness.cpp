// Function-level differential test of include/rans_byte.h, rans64.h, rans_word_sse41.h against the reference's headers.
// REFDIR is replaced by the reference checkout's path at build time (oracle/Makefile); nothing of the
// reference is copied here -- its headers are #included where they lie, inside namespace ref.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <assert.h>
#include <smmintrin.h>
#include "REFDIR/platform.h"
#include <algorithm>
#include <random>
#include <vector>

namespace ref {
#include "REFDIR/rans_byte.h"
#include "REFDIR/rans64.h"
#include "REFDIR/rans_word_sse41.h"
#include "body.inc"
}
#undef RANS_BYTE_HEADER
#undef RANS64_HEADER
#undef RANS_WORD_SSE41_HEADER
#undef RansAssert
#undef Rans64Assert
#undef RANS_BYTE_L
#undef RANS64_L
#undef RANS_WORD_L
#undef RANS_WORD_SCALE_BITS
#undef RANS_WORD_M
#undef RANS_WORD_NSYMS
namespace ours {
#include "rans_byte.h"
#include "rans64.h"
#include "rans_word_sse41.h"
#include "body.inc"
}

template <class A, class B> static int cmp(const char* what, const A& a, const B& b)
{
    if (!a.round_trips || !b.round_trips) { printf("%s: a decode did not reproduce its input (ref %d, ours %d)\n", what, (int)a.round_trips, (int)b.round_trips); return 1; }
    if (a.bytes != b.bytes || a.vals != b.vals) {
        size_t i = 0;
        while (i < a.vals.size() && i < b.vals.size() && a.vals[i] == b.vals[i]) i++;
        printf("%s DIFFERS: %zu/%zu values, %zu/%zu bytes, first value mismatch at %zu\n", what, a.vals.size(), b.vals.size(),
               a.bytes.size(), b.bytes.size(), i);
        for (size_t k = (i > 8 ? i - 8 : 0); k < i + 6 && k < a.vals.size(); k++) printf("  [%zu] ref=%llx ours=%llx\n", k, (unsigned long long)a.vals[k], (unsigned long long)b.vals[k]);
        printf("  bytes equal: %d\n", (int)(a.bytes == b.bytes));
        return 1;
    }
    printf("%s ok: %zu values, %zu stream bytes identical\n", what, a.vals.size(), a.bytes.size());
    return 0;
}

int main()
{
    int bad = 0;
    for (uint64_t seed = 1; seed <= 3; seed++) {
        { ref::Out a; ours::Out b; ref::run_byte(seed, a); ours::run_byte(seed, b); bad += cmp("rans_byte.h", a, b); }
        { ref::Out a; ours::Out b; ref::run_64(seed, a); ours::run_64(seed, b); bad += cmp("rans64.h", a, b); }
        { ref::Out a; ours::Out b; ref::run_word(seed, a); ours::run_word(seed, b); bad += cmp("rans_word_sse41.h", a, b); }
    }
    return bad;
}

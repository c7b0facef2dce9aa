// alias_kernels.cuh -- sm_90a kernels for the alias-table coder (main_alias.cpp semantics):
// rans_byte.h state machine (31-bit state, byte renormalisation, L = 1 << 23) with the
// alias-method symbol lookup of main_alias.cpp:252-267 (decode) and the slot remap of
// main_alias.cpp:241-250 (encode).
//
// Same mapping as the word coder: one warp = one chunk = one 32-way stream.  The byte
// coder moves 0, 1 or 2 bytes per lane per step (scale_bits <= 16: after a decode step
// x >= 2^(23-scale_bits) >= 2^7, and 2^7 << 16 = L; before an encode step x < 2^31 and
// x_max >= 2^15), so the warp-wide renormalisation needs two ballots: "at least one
// byte" and "two bytes".  Within a step lane k's bytes sit before lane k+1's, most
// significant first (RansDecRenorm, rans_byte.h:307-318, called lane by lane at
// main_alias.cpp:396-397).
#pragma once
#include "decode_stream.cuh"
#include "device_utils.cuh"
#include "tables.h"
#include "word_kernels.cuh"   // funnel_shr_wrap; encode_stream and placement for the encoder

namespace rb200 {

constexpr uint32_t kByteL = 1u << 23;   // RANS_BYTE_L, rans_byte.h:50
constexpr int kAliasDecWarps = 16;
constexpr uint32_t kAliasDecReplicas = 8;    // quarter-warp lanes hit 8 different 16-byte bank groups

// ---------------------------------------------------------------------------
// K8: the rans_byte cum2sym decoder (main.cpp) on the stream window of decode_stream.cuh.
// ---------------------------------------------------------------------------
// The byte coder for decode_window_chunk: RansDecGet -> cum2sym -> RansDecAdvanceSymbolStep (rans_byte.h:125-128,
// main.cpp:200, rans_byte.h:291-304), then RansDecRenorm (rans_byte.h:307-318).  tab = shared address of cum2sym[1 << sb],
// followed by the 256 x {start | freq << 16} table.
// SB: scale_bits as a compile-time constant (16, 14, 12: masks and shift counts become immediates), 0 = use `sb_rt`.
template <uint32_t SB>
struct ByteDecoder {
    using X = uint32_t;
    static constexpr uint32_t kHeaderBytes = rb200::kHeaderBytes, kUnit = 1, kMaxBytes = 2;
    static constexpr X kL = kByteL;                    // RansEncInit, rans_byte.h:56-59
    uint32_t tab;
    uint32_t sb_rt;

    // RansDecInit x 32 (rans_byte.h:109-122): lane k's state is the k-th little-endian u32
    template <class At>
    __device__ __forceinline__ X read_header(At at, uint32_t lane) const
    {
        uint32_t x = 0;
#pragma unroll
        for (int b = 3; b >= 0; b--) x = (x << 8) | lds_u8(at(4 * lane + b));
        return x;
    }

    template <bool FULL>
    __device__ __forceinline__ void step(uint32_t& x, uint32_t& cursor, uint32_t ring, uint8_t* o, uint32_t lt, bool active) const
    {
        const uint32_t sb = SB ? SB : sb_rt;
        bool n1 = false, n2 = false;
        if (active) {
            const uint32_t xm = x & ((1u << sb) - 1);                          // rans_byte.h:127
            const uint32_t s = lds_u8_ro(tab + xm);                            // cum2sym, main.cpp:200
            const uint32_t ds = lds_u32_ro(tab + (1u << sb) + 4u * s);         // RansDecSymbol {start, freq}
            x = (ds >> 16) * (x >> sb) + xm - (ds & 0xffffu);                  // rans_byte.h:297
            *o = static_cast<uint8_t>(s);
            n1 = x < kByteL;
            n2 = x < (kByteL >> 8);
        }
        renorm<FULL>(x, cursor, ring, lt, n1, n2);
    }

    // RansDecRenorm (rans_byte.h:307-318) for the warp on the stream window: 0, 1 or 2 bytes per lane, lane k's bytes
    // before lane k+1's, most significant first; n1 / n2: this lane takes at least one / two bytes (false when inactive)
    template <bool FULL>
    static __device__ __forceinline__ void renorm(uint32_t& x, uint32_t& cursor, uint32_t ring, uint32_t lt, bool n1, bool n2)
    {
        if (FULL) {
            // RansDecRenorm for the warp as one PTX sequence: two predicates feed the votes, the two ranked byte
            // loads and the state updates (the C++ below costs six more instructions and a branch per step)
            asm volatile(
                "{\n\t"
                ".reg .pred p1, p2;\n\t"
                ".reg .b32 m, r, a, b;\n\t"
                "setp.lt.u32 p1, %0, %2;\n\t"
                "setp.lt.u32 p2, %0, %3;\n\t"
                "vote.sync.ballot.b32 m, p1, 0xffffffff;\n\t"
                "and.b32 r, m, %4;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, %1, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "vote.sync.ballot.b32 m, p2, 0xffffffff;\n\t"
                "and.b32 r, m, %4;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, a, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "add.u32 b, a, 1;\n\t"
                "and.b32 a, a, %5;\n\t"
                "and.b32 b, b, %5;\n\t"
                "or.b32 a, a, %6;\n\t"
                "or.b32 b, b, %6;\n\t"
                "@p1 ld.shared.u8 a, [a];\n\t"
                "@p2 ld.shared.u8 b, [b];\n\t"
                "@p1 mad.lo.u32 %0, %0, 256, a;\n\t"
                "@p2 mad.lo.u32 %0, %0, 256, b;\n\t"
                "}"
                : "+r"(x), "+r"(cursor)
                : "n"(kByteL), "n"(kByteL >> 8), "r"(lt), "n"(kRingBytes - 1), "r"(ring)
                : "memory");
            return;
        }
        const uint32_t m1 = __ballot_sync(0xffffffffu, n1);
        const uint32_t m2 = __ballot_sync(0xffffffffu, n2);
        uint32_t a = cursor + __popc(m1 & lt);
        if (m2) a += __popc(m2 & lt);                                          // warp-uniform: two-byte refills are the rarer case
        const uint32_t b0 = lds_u8(ring | (a & (kRingBytes - 1)));
        if (n1) x = (x << 8) | b0;                                             // rans_byte.h:313
        cursor += __popc(m1);
        if (m2) {
            const uint32_t b1 = lds_u8(ring | ((a + 1) & (kRingBytes - 1)));
            if (n2) x = (x << 8) | b1;
            cursor += __popc(m2);
        }
}
};

// g_tab = cum2sym[1 << sb] followed by 256 x u32 {start | freq << 16}
template <uint32_t SB>
__global__ void __launch_bounds__(kAliasDecWarps * 32, 4)
byte_decode_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets, uint32_t sb_rt,
                   const void* __restrict__ g_tab, uint8_t* __restrict__ out, uint64_t n, uint32_t chunk_syms,
                   uint32_t n_chunks, uint32_t* __restrict__ status)
{
    const uint32_t sb = SB ? SB : sb_rt;
    extern __shared__ __align__(1024) uint8_t s_adec[];       // [16 x 1 KiB rings][table]
    uint4* s_tab = reinterpret_cast<uint4*>(s_adec + kAliasDecWarps * kRingBytes);
    const uint32_t vecs = ((1u << sb) + 1024) / 16;
    for (uint32_t i = threadIdx.x; i < vecs; i += blockDim.x) s_tab[i] = static_cast<const uint4*>(g_tab)[i];
    __syncthreads();

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * kAliasDecWarps + warp;
    if (chunk >= n_chunks) return;
    const uint64_t first = static_cast<uint64_t>(chunk) * chunk_syms;
    const uint32_t m = static_cast<uint32_t>(min(static_cast<uint64_t>(chunk_syms), n - first));
    decode_window_chunk(ByteDecoder<SB>{smem_addr_pinned(s_tab), sb}, blob, blob_size, offsets, chunk, smem_addr(s_adec) + warp * kRingBytes,
                        out + first, m, status);
}

// ---------------------------------------------------------------------------
// K3p: the alias decoder on the persistent window of decode_stream.cuh -- 2 CTAs of 20 warps per SM stay resident and
// pull chunk ids from the context's atomic counter; the 32 KiB replicated bucket table is built once per CTA; the
// per-warp stream window is the cp.async ring with a mirror behind it, wrapped once per 8 steps, so the two ranked byte
// reads of RansDecRenorm need no address masking (round 1's kernel spent 5 of its ~20 ALU-pipe instructions per step
// on that, and the ALU pipe is what bound it: 85 % busy).  Experiments and ablations: tools/decode_lab.cu --coder alias.
// ---------------------------------------------------------------------------
using AliasDecShip = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, 0, false, 256 * kAliasDecReplicas * 16>;

// Experiment switches of tools/decode_lab.cu --coder alias (the shipped kernel has all of them off).  The word decoder's
// ablation bits kAblNoSymbolStore / kAblNoRingRead / kAblNoRefill apply as they do there; two more are specific to this step:
constexpr int kAblAliasOneByte = 16;   // ABLATION: renormalise by at most one byte (no second vote / rank / load / merge)
// LEAN (not an ablation, bit-exact): the bucket entry is repacked when the CTA stages the table, so that the step needs
// two selects and no byte permute, and compares the bucket-local bits of x at the TOP of a word:
//   w0 = (own_count - 1) << (40 - SB) | own adjust,  w1 = own slot_freqs << 8 | sym,  w2 = other's,  w3 = other's adjust
// "own" <=> x << (40 - SB) <= w0 (the low bits of w0 cannot change the outcome: the left side has zeros there); an empty
// own part (own_count 0 wraps to all ones: always taken) carries the other slot's data.  Needs a compile-time SB > 8.
template <uint32_t SB>
__device__ __forceinline__ uint4 alias_lean_entry(const AliasDecEntry& e, uint32_t bucket)
{
    constexpr uint32_t LB = SB - 8, K = 32 - LB;
    const uint32_t own_count = e.divider - (bucket << LB);                     // 0 .. 1 << LB (model_host.cpp: divider = lo + own)
    const bool none = own_count == 0;
    const uint32_t adj_own = none ? (e.adjust & 0xffffu) : (e.adjust >> 16);
    return make_uint4(((own_count - 1u) << K) | adj_own, none ? e.alt0 : e.alt1, e.alt0, e.adjust & 0xffffu);
}

// The alias coder for decode_persistent: RansDecGetAlias (main_alias.cpp:252-267), then RansDecRenorm
// (rans_byte.h:307-318).  tab_lane = this lane's replica of the 256 x 16 B bucket table.
template <uint32_t SB, int LEAN = 0>
struct AliasDecoder {
    using X = uint32_t;
    static constexpr uint32_t kHeaderBytes = rb200::kHeaderBytes, kUnit = 1, kMaxBytes = 2;
    static constexpr X kL = kByteL;
    uint32_t tab_lane;
    uint32_t sb_rt;

    template <class At>
    __device__ __forceinline__ X read_header(At at, uint32_t lane) const
    {
        return ByteDecoder<SB>{0, 0}.read_header(at, lane);
    }

    // window step (decode_window_chunk): the lookup of step_p, then ByteDecoder's window renormalisation
    template <bool FULL>
    __device__ __forceinline__ void step(uint32_t& x, uint32_t& cursor, uint32_t ring, uint8_t* o, uint32_t lt, bool active) const
    {
        bool n1 = false, n2 = false;
        if (active) {
            get<true>(x, o);
            n1 = x < kByteL;
            n2 = x < (kByteL >> 8);
        }
        ByteDecoder<SB>::template renorm<FULL>(x, cursor, ring, lt, n1, n2);
    }

    // RansDecGetAlias (main_alias.cpp:252-267): the next state and, when STORE, the symbol
    template <bool STORE>
    __device__ __forceinline__ void get(uint32_t& x, uint8_t* o) const
    {
        const uint32_t sb = SB ? SB : sb_rt;
        if (LEAN && SB > 8) {
            constexpr uint32_t LB = SB > 8 ? SB - 8 : 1;
            // bucket id: byte 1 of x by one PRMT at scale_bits 16, otherwise masked in place and scaled by the IMAD
            const uint32_t addr = LB == 8 ? mad_u32(__byte_perm(x, 0u, 0x4441u), kAliasDecReplicas * 16, tab_lane)
                                          : mad_u32(x & (0xffu << LB), (kAliasDecReplicas * 16) >> (LB & 7), tab_lane);
            const uint4 e = lds_u128_ro(addr);
            const bool own = mad_u32(x, 1u << (32 - LB), 0u) <= e.x;           // main_alias.cpp:261 on the bucket-local bits
            const uint32_t fs = own ? e.y : e.z;
            const uint32_t adj = own ? e.x : e.w;
            x = mad_u32(fs >> 8, x >> SB, (x - adj) & ((1u << SB) - 1));       // :265
            if (STORE) *o = static_cast<uint8_t>(fs);                          // :266
        } else {
            const uint32_t xm = x & ((1u << sb) - 1);                              // main_alias.cpp:258
            const uint32_t bucket = xm >> (sb - 8);                                // :259
            const uint4 e = lds_u128_ro(mad_u32(bucket, kAliasDecReplicas * 16, tab_lane));
            const bool own = xm < e.x;                                             // :261 (bucket2 = 2 * bucket + 1)
            const uint32_t fs = own ? e.z : e.y;                                   // slot_freqs << 8 | sym_id
            const uint32_t adj = __byte_perm(e.w, 0u, own ? 0x4432u : 0x4410u);    // the taken half of the packed adjusts
            x = mad_u32(fs >> 8, x >> sb, (xm - adj) & 0xffffu);                   // :265
            if (STORE) *o = static_cast<uint8_t>(fs);                              // :266
        }
    }

    template <class P>
    __device__ __forceinline__ void step_p(uint32_t& x, uint32_t& cur, uint8_t* o, uint32_t lt, uint32_t lane, int j, bool active) const
    {
        if (active) get<!(P::kAblate & kAblNoSymbolStore)>(x, o);
        // RansDecRenorm (rans_byte.h:307-318) for the warp: 0, 1 or 2 bytes per lane, lane k's bytes before lane k+1's,
        // most significant first.  Two predicates feed the votes, the ranked byte loads and the merges.
        const uint32_t xr = active ? x : kByteL;
        uint32_t xo = x;
        if (P::kAblate & kAblAliasOneByte) {
            asm volatile(
                "{\n\t"
                ".reg .pred p1;\n\t"
                ".reg .b32 m, r, a, b0;\n\t"
                "setp.lt.u32 p1, %2, %4;\n\t"
                "vote.sync.ballot.b32 m, p1, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, %1, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "ld.shared.u8 b0, [a];\n\t"
                "@p1 mad.lo.u32 %0, %0, 256, b0;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt), "n"(kByteL));
        } else if (P::kAblate & kAblNoRingRead) {
            asm volatile(
                "{\n\t"
                ".reg .pred p1, p2;\n\t"
                ".reg .b32 m, r, a, b0;\n\t"
                "setp.lt.u32 p1, %2, %4;\n\t"
                "setp.lt.u32 p2, %2, %5;\n\t"
                "vote.sync.ballot.b32 m, p1, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, %1, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "vote.sync.ballot.b32 m, p2, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, a, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "and.b32 b0, a, 255;\n\t"
                "@p1 mad.lo.u32 %0, %0, 256, b0;\n\t"
                "@p2 mad.lo.u32 %0, %0, 256, b0;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt), "n"(kByteL), "n"(kByteL >> 8));
        } else {
            asm volatile(
                "{\n\t"
                ".reg .pred p1, p2;\n\t"
                ".reg .b32 m, r, a, b0, b1;\n\t"
                "setp.lt.u32 p1, %2, %4;\n\t"
                "setp.lt.u32 p2, %2, %5;\n\t"
                "vote.sync.ballot.b32 m, p1, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, %1, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "vote.sync.ballot.b32 m, p2, 0xffffffff;\n\t"
                "and.b32 r, m, %3;\n\t"
                "popc.b32 r, r;\n\t"
                "add.u32 a, a, r;\n\t"
                "popc.b32 m, m;\n\t"
                "add.u32 %1, %1, m;\n\t"
                "ld.shared.u8 b0, [a];\n\t"              // unpredicated: ring + mirror make both reads safe for every lane
                "ld.shared.u8 b1, [a+1];\n\t"
                "@p1 mad.lo.u32 %0, %0, 256, b0;\n\t"
                "@p2 mad.lo.u32 %0, %0, 256, b1;\n\t"
                "}"
                : "+r"(xo), "+r"(cur)
                : "r"(xr), "r"(lt), "n"(kByteL), "n"(kByteL >> 8));
        }
        x = xo;
    }
};

// P, LEAN: the shipped configuration unless tools/decode_lab.cu instantiates an experiment
template <uint32_t SB, class P = AliasDecShip, int LEAN = 0>
__global__ void __launch_bounds__(P::kWarps * 32, P::kMinBlocks)
alias_decode_persist_kernel(const uint8_t* __restrict__ blob, uint64_t blob_size, const uint64_t* __restrict__ offsets, uint32_t sb_rt,
                            const AliasDecEntry* __restrict__ g_dec, uint8_t* __restrict__ out, uint64_t n, uint32_t chunk_syms,
                            uint32_t n_chunks, DecodeWork* __restrict__ work, uint32_t* __restrict__ status)
{
    static_assert(P::kRefill == kRefillCpAsync, "the ring's mbarriers are not initialised here: cp.async refill only");
    extern __shared__ __align__(1024) uint8_t s_adec[];       // [32 KiB table][16 B][kWarps x (ring, mirror)]
    uint4* s_tab = reinterpret_cast<uint4*>(s_adec);
    for (uint32_t i = threadIdx.x; i < 256 * kAliasDecReplicas; i += blockDim.x) {
        const AliasDecEntry e = g_dec[i / kAliasDecReplicas];
        if (LEAN && SB > 8) s_tab[i] = alias_lean_entry<(SB > 8 ? SB : 9)>(e, i / kAliasDecReplicas);
        else s_tab[i] = make_uint4(e.divider, e.alt0, e.alt1, e.adjust);
    }
    __syncthreads();

    const uint32_t base = smem_addr_pinned(s_adec);
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
    const uint32_t lane = threadIdx.x & 31;
    const AliasDecoder<SB, LEAN> coder = {base + (lane & (kAliasDecReplicas - 1)) * 16, sb_rt};
    decode_persistent<P>(coder, base + P::kWarpsOff + warp * P::kWarpStride, blob, blob_size, offsets, out, n, chunk_syms, n_chunks,
                         work, lane, status);
}

// ---------------------------------------------------------------------------
// K4: 32-way alias encode.  RansEncPutAlias (main_alias.cpp:241-250) = RansEncRenorm
// (rans_byte.h:62-74) + divide + alias_remap gather.
//
// Persistent kernel, one 32-warp CTA per SM, because the encoder's slot permutation
// alias_remap (u16, 2 << scale_bits bytes = 128 KiB at scale_bits 16; SURVEY H8) lives in
// shared memory next to the 8x replicated per-symbol table ({magic, freq, cum, shift}, one
// conflict-free LDS.128 per step) and the per-warp 512 B symbol stage + 512 B output ring
// of the shared chunk encoder (encode_stream.cuh).
// ---------------------------------------------------------------------------
constexpr int kAliasEncWarps = 32;
constexpr uint32_t kAliasEncFixedSmem = kAliasEncWarps * kEncWarpSmem + kEncTableBytes;   // 64 KiB + remap
constexpr uint32_t kAliasFusedSlots = 2;        // scratch slots per worker warp in fused mode (a SlotQueue, placement.cuh)

__device__ __forceinline__ uint32_t lds_u16_ro(uint32_t addr)
{
    uint16_t v;
    asm("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}

// The byte-renormalising coders for encode_stream (encode_stream.cuh); wpos is the ring position of the next byte =
// 511 - bytes_emitted.  step = one encode step for the whole warp:
//   ALIAS:  RansEncPutAlias (main_alias.cpp:241-250); table {magic, freq, cum, shift}
//   !ALIAS: RansEncPutSymbol (rans_byte.h:258-280);   table {x_max, rcp_freq, bias, cmpl_freq | rcp_shift << 16}
//           = RansEncSymbol (rans_byte.h:159-165), bit 31 of the last word marks a symbol outside the model
template <bool ALIAS, uint32_t SB>
struct AliasEncoder {
    using X = uint32_t;
    static constexpr uint32_t kUnit = 1, kMaxEmit = 2, kBadBit = kEncBadSymbol;
    static constexpr X kInit = kByteL;                 // RansEncInit, rans_byte.h:56-59
    uint32_t tab;                                      // shared address of the 8x replicated uint4 table
    uint32_t remap;                                    // ALIAS: shared address of alias_remap (u16)
    uint32_t sb_rt;                                    // scale_bits when SB == 0

    template <bool FULL>
    __device__ __forceinline__ void step(EncState<X>& st, uint32_t sym, uint32_t tab_lane, uint32_t ring, uint32_t gt, bool active) const
    {
        const uint32_t sb = SB ? SB : sb_rt;
        bool n1 = false, n2 = false;
        uint4 e = make_uint4(0, 1, 0, 0);
        uint32_t x_max = 0;
        if (active) {
            e = lds_u128_ro(tab_lane + sym * (kEncReplicas * 16));
            st.flags |= e.w;
            x_max = ALIAS ? e.y << (31 - sb) : e.x;                   // ((L >> sb) << 8) * freq, rans_byte.h:64 / :197
        }
        if (FULL) {
            // the renormalisation below as one PTX sequence: two predicates feed the votes, the ranked stores and
            // the shifts (the compiler otherwise re-evaluates the comparisons and branches around the stores)
            asm volatile(
                "{\n\t"
                ".reg .pred p1, p2;\n\t"
                ".reg .b32 m1, m2, r1, r2, a, b, xs;\n\t"
                "shr.u32 xs, %0, 8;\n\t"
                "setp.ge.u32 p1, %0, %2;\n\t"
                "setp.ge.u32 p2, xs, %2;\n\t"
                "vote.sync.ballot.b32 m1, p1, 0xffffffff;\n\t"
                "vote.sync.ballot.b32 m2, p2, 0xffffffff;\n\t"
                "and.b32 r1, m1, %3;\n\t"
                "and.b32 r2, m2, %3;\n\t"
                "popc.b32 r1, r1;\n\t"
                "popc.b32 r2, r2;\n\t"
                "sub.u32 a, %1, r1;\n\t"
                "sub.u32 a, a, r2;\n\t"
                "sub.u32 b, a, 1;\n\t"
                "and.b32 a, a, %4;\n\t"
                "and.b32 b, b, %4;\n\t"
                "or.b32 a, a, %5;\n\t"
                "or.b32 b, b, %5;\n\t"
                "@p1 st.shared.u8 [a], %0;\n\t"
                "@p2 st.shared.u8 [b], xs;\n\t"
                "@p1 mov.b32 %0, xs;\n\t"
                "@p2 shr.u32 %0, %0, 8;\n\t"
                "popc.b32 m1, m1;\n\t"
                "popc.b32 m2, m2;\n\t"
                "sub.u32 %1, %1, m1;\n\t"
                "sub.u32 %1, %1, m2;\n\t"
                "}"
                : "+r"(st.x), "+r"(st.wpos)
                : "r"(x_max), "r"(gt), "n"(kEncRingBytes - 1), "r"(ring)
                : "memory");
        } else {
            if (active) {
                n1 = st.x >= x_max;                                   // :65 / :265
                n2 = (st.x >> 8) >= x_max;                            // second trip of the do/while, :67-70
            }
            const uint32_t m1 = __ballot_sync(0xffffffffu, n1);
            const uint32_t m2 = __ballot_sync(0xffffffffu, n2);
            if (n1) {
                // lanes are visited 31..0 (main_alias.cpp:365-370 generalised); each writes downwards
                const uint32_t pos = st.wpos - __popc(m1 & gt) - __popc(m2 & gt);
                sts_u8(ring | (pos & (kEncRingBytes - 1)), st.x);                          // :68
                if (n2) sts_u8(ring | ((pos - 1) & (kEncRingBytes - 1)), st.x >> 8);
                st.x >>= n2 ? 16 : 8;                                                      // :69
            }
            st.wpos -= __popc(m1) + __popc(m2);
        }
        if (active) {
            if (ALIAS) {
                // exact x / freq with the 33-bit round-up reciprocal 2^32 + magic, as in the word encoder; here
                // x < 2^31 (rans_byte.h:26-28), so x + mulhi(x, magic) < 2^32 and there is no carry to fold in
                const uint32_t q = funnel_shr_wrap(st.x + __umulhi(st.x, e.x), 0u, e.w);
                const uint32_t r = st.x - q * e.y;                                     // x % freq
                st.x = (q << sb) + lds_u16_ro(remap + 2u * (r + e.z));                 // main_alias.cpp:249
            } else {
                const uint32_t q = __umulhi(st.x, e.y) >> ((e.w >> 16) & 31u);         // rans_byte.h:278
                st.x = st.x + e.z + q * (e.w & 0xffffu);                               // :279
            }
        }
    }
};

// !ALIAS: g_enc holds RansEncSymbol images {x_max, rcp_freq, bias, cmpl | shift << 16}, g_remap is unused
// Two modes (like the word encoder):
//   look == nullptr: chunks strided over the persistent CTAs, each into its own worst-case slot of `scratch`,
//                    sizes[] written for the tile scan + compaction that follow;
//   look != nullptr: fused -- chunk ids from an atomic counter, kAliasFusedSlots scratch slots per warp, warp 0 of
//                    CTA 0 is the scanner (placement.cuh).
template <bool ALIAS, uint32_t SB>
__device__ __forceinline__ void alias_encode(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t sb_rt,
                                             const AliasEncEntry* __restrict__ g_enc, const uint16_t* __restrict__ g_remap,
                                             uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint32_t* __restrict__ sizes,
                                             uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob,
                                             uint64_t blob_cap, uint64_t* __restrict__ offsets, uint32_t* __restrict__ status)
{
    const uint32_t sb = SB ? SB : sb_rt;
    extern __shared__ __align__(1024) uint8_t s_alias[];      // [32 x 1.0 KiB stage+ring][32 KiB table][remap]
    uint4* s_tab = reinterpret_cast<uint4*>(s_alias + kAliasEncWarps * kEncWarpSmem);
    uint4* s_remap = reinterpret_cast<uint4*>(s_alias + kAliasEncFixedSmem);
    for (uint32_t i = threadIdx.x; i < 256 * kEncReplicas; i += blockDim.x) {
        const AliasEncEntry e = g_enc[i / kEncReplicas];
        // a symbol the model does not contain: keep the step well defined (freq 1), flag it
        if (ALIAS) s_tab[i] = (e.shift & kEncBadSymbol) ? make_uint4(0, 1, 0, kEncBadSymbol) : make_uint4(e.magic, e.freq, e.cum, e.shift);
        else       s_tab[i] = make_uint4(e.magic, e.freq, e.cum, e.shift);          // the host already made bad entries safe
    }
    if (ALIAS) {
        const uint32_t remap_vecs = (2u << sb) / 16;
        for (uint32_t i = threadIdx.x; i < remap_vecs; i += blockDim.x) s_remap[i] = reinterpret_cast<const uint4*>(g_remap)[i];
    }
    __syncthreads();

    const uint32_t warp = threadIdx.x >> 5;
    const uint32_t base = smem_addr(s_alias);
    const uint32_t wsm = base + warp * kEncWarpSmem;
    const AliasEncoder<ALIAS, SB> coder = {base + kAliasEncWarps * kEncWarpSmem, base + kAliasEncFixedSmem, sb};
    if (!look) {
        for (uint32_t chunk = blockIdx.x * kAliasEncWarps + warp; chunk < n_chunks; chunk += gridDim.x * kAliasEncWarps) {
            const ChunkRange r = chunk_range(chunk, chunk_syms, n);
            encode_chunk_split(in + r.first, r.m, chunk, coder, wsm, scratch, slot_bytes, sizes, status);
        }
        return;
    }
    encode_chunks_fused<kAliasFusedSlots, kAliasEncWarps, false>(in, n, chunk_syms, coder, wsm, scratch, slot_bytes,
                                                                 PlaceOut{look, n_chunks, blob, blob_cap, offsets, status}, counter);
}

// GEOM (rb200_container_model_encode_varlen_async): n, the chunk count, the blob's place in the container `blob` and
// its capacity from the record, on the grid the host sized for n_max.  In split mode a CTA past the real chunks exits
// before it stages its tables; in fused mode every CTA runs (CTA 0 holds the scanner, the others find no chunk and leave).
// GATED (rb200_container_model_encode_auto_async): runs only when the choice record names `group`, and then at the
// recorded scale_bits; otherwise it exits at entry, before it touches shared memory, the counter, look[] or scratch.
template <bool ALIAS, uint32_t SB, bool GEOM = false, bool GATED = false>
__global__ void __launch_bounds__(kAliasEncWarps * 32, 1)
alias_encode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t sb_rt,
                    const AliasEncEntry* __restrict__ g_enc, const uint16_t* __restrict__ g_remap,
                    uint8_t* __restrict__ scratch, uint32_t slot_bytes, uint32_t* __restrict__ sizes,
                    uint64_t* __restrict__ look, uint32_t* __restrict__ counter, uint8_t* __restrict__ blob, uint64_t blob_cap,
                    uint64_t* __restrict__ offsets, uint32_t* __restrict__ status, const VarlenGeom* __restrict__ geom,
                    const CoderChoice* __restrict__ choice, uint32_t group)
{
    if (GATED) {
        if (choice->group != group) return;
        sb_rt = choice->scale_bits;
    }
    if (GEOM) {
        n_chunks = geom->n_chunks;
        if (!geom->go || (!look && blockIdx.x * kAliasEncWarps >= n_chunks)) return;
        n = geom->n;
        blob += geom->blob_off;
        blob_cap = geom->blob_cap;
    }
    alias_encode<ALIAS, SB>(in, n, chunk_syms, n_chunks, sb_rt, g_enc, g_remap, scratch, slot_bytes, sizes, look, counter, blob, blob_cap,
                            offsets, status);
}

// dynamic shared memory of the alias (remap != nullptr) or byte encoder at scale_bits sb
inline uint32_t alias_encode_smem(bool alias, uint32_t sb) { return kAliasEncFixedSmem + (alias ? (2u << sb) : 0u); }

// scale_bits the kernels are specialised for (main_alias.cpp:276 uses 16, main.cpp:136 / main64.cpp:136 use 14, the word
// coder's 12); every other value runs the generic instantiation (SB = 0).  Each is configured for scale_bits 16, the
// most shared memory any of them is launched with.
template <bool ALIAS, uint32_t SB>
inline void configure_alias_encode()
{
    for (const void* k : {reinterpret_cast<const void*>(alias_encode_kernel<ALIAS, SB>), reinterpret_cast<const void*>(alias_encode_kernel<ALIAS, SB, true>),
                          reinterpret_cast<const void*>(alias_encode_kernel<ALIAS, SB, false, true>),
                          reinterpret_cast<const void*>(alias_encode_kernel<ALIAS, SB, true, true>)}) {
        cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, alias_encode_smem(ALIAS, 16));
    }
}
template <uint32_t SB>
inline void configure_byte_decode()
{
    cudaFuncSetAttribute(byte_decode_kernel<SB>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(byte_decode_kernel<SB>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAliasDecWarps * kRingBytes + 1024 + (1u << 16));
}
// Build switch: 1 ships the repacked ("lean") bucket entry of AliasDecoder for the compile-time scale_bits
// (A/B: tools/decode_lab.cu --coder alias); a runtime scale_bits always takes the plain entry.
#ifndef RB200_ALIAS_LEAN
#define RB200_ALIAS_LEAN 1
#endif
constexpr int kAliasLean = RB200_ALIAS_LEAN;
template <uint32_t SB>
inline void configure_alias_persist()
{
    auto k = alias_decode_persist_kernel<SB, AliasDecShip, kAliasLean>;
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, AliasDecShip::kSmemBytes);
}
inline void configure_alias_kernels()
{
    configure_alias_persist<0>(); configure_alias_persist<16>(); configure_alias_persist<14>(); configure_alias_persist<12>();
    configure_byte_decode<0>(); configure_byte_decode<16>(); configure_byte_decode<14>(); configure_byte_decode<12>();
    configure_alias_encode<true, 0>(); configure_alias_encode<true, 16>(); configure_alias_encode<true, 14>(); configure_alias_encode<true, 12>();
    configure_alias_encode<false, 0>(); configure_alias_encode<false, 16>(); configure_alias_encode<false, 14>(); configure_alias_encode<false, 12>();
}

#define RB200_ALIAS_SB_DISPATCH(sb, CALL) \
    switch (sb) {                        \
    case 16: { constexpr uint32_t SB = 16; CALL; } break; \
    case 14: { constexpr uint32_t SB = 14; CALL; } break; \
    case 12: { constexpr uint32_t SB = 12; CALL; } break; \
    default: { constexpr uint32_t SB = 0; CALL; } break;  \
    }

// remap == nullptr selects the rans_byte cum2sym coder.  look == nullptr: split mode (sizes[] out, one slot per
// chunk); otherwise fused mode (kAliasFusedSlots slots per worker warp; look/counter zeroed by the caller).
// grid <= one CTA per SM (the kernel is persistent), smem = alias_encode_smem(remap != nullptr, sb).  geom set: the
// GEOM instance, with n, n_chunks and the grid those of n_max and blob the container.  choice set: the GATED instance of
// sb's SB, run when the record names `group` (smem then covers the largest scale_bits of the group).
inline void launch_alias_encode(cudaStream_t stream, uint32_t grid, uint32_t smem, const uint8_t* d_in, uint64_t n, uint32_t chunk_syms,
                                uint32_t n_chunks, uint32_t sb, const AliasEncEntry* enc, const uint16_t* remap, uint8_t* scratch,
                                uint32_t slot, uint32_t* sizes, uint64_t* look, uint32_t* counter, uint8_t* blob, uint64_t blob_cap,
                                uint64_t* offsets, uint32_t* status, const VarlenGeom* geom, const CoderChoice* choice = nullptr,
                                uint32_t group = 0)
{
    auto kernel = alias_encode_kernel<false, 0>;
    if (choice) {
        if (remap) {
            RB200_ALIAS_SB_DISPATCH(sb, (kernel = geom ? alias_encode_kernel<true, SB, true, true> : alias_encode_kernel<true, SB, false, true>))
        } else {
            RB200_ALIAS_SB_DISPATCH(sb, (kernel = geom ? alias_encode_kernel<false, SB, true, true> : alias_encode_kernel<false, SB, false, true>))
        }
    } else if (remap) {
        RB200_ALIAS_SB_DISPATCH(sb, (kernel = geom ? alias_encode_kernel<true, SB, true> : alias_encode_kernel<true, SB>))
    } else {
        RB200_ALIAS_SB_DISPATCH(sb, (kernel = geom ? alias_encode_kernel<false, SB, true> : alias_encode_kernel<false, SB>))
    }
    kernel<<<grid, kAliasEncWarps * 32, smem, stream>>>(d_in, n, chunk_syms, n_chunks, sb, enc, remap, scratch, slot, sizes, look, counter,
                                                        blob, blob_cap, offsets, status, geom, choice, group);
}

// the persistent kernel: sms x 2 CTAs of 20 warps, chunk ids from the context's work counter
inline void launch_alias_decode(cudaStream_t stream, const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, uint32_t sb,
                                const AliasDecEntry* dec, uint8_t* out, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks,
                                uint32_t* status, DecodeWork* work, uint32_t sms)
{
    using P = AliasDecShip;
    const uint32_t want = (n_chunks + P::kWarps - 1) / P::kWarps, full = sms * P::kMinBlocks;
    const uint32_t grid = want < full ? want : full;
    RB200_ALIAS_SB_DISPATCH(sb, (alias_decode_persist_kernel<SB, P, kAliasLean><<<grid, P::kWarps * 32, P::kSmemBytes, stream>>>(
        blob, blob_size, offsets, sb, dec, out, n, chunk_syms, n_chunks, work, status)))
}

// rans_byte cum2sym decode: table = cum2sym[1 << sb] followed by 256 x u32 {start | freq << 16}
inline void launch_byte_decode(cudaStream_t stream, const uint8_t* blob, uint64_t blob_size, const uint64_t* offsets, uint32_t sb,
                               const uint8_t* table, uint8_t* out, uint64_t n, uint32_t chunk_syms, uint32_t n_chunks, uint32_t* status)
{
    const uint32_t grid = (n_chunks + kAliasDecWarps - 1) / kAliasDecWarps;
    RB200_ALIAS_SB_DISPATCH(sb, (byte_decode_kernel<SB><<<grid, kAliasDecWarps * 32, kAliasDecWarps * kRingBytes + 1024 + (1u << sb), stream>>>(
        blob, blob_size, offsets, sb, table, out, n, chunk_syms, n_chunks, status)))
}

}  // namespace rb200

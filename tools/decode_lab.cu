// decode_lab.cu -- one-binary experiment bench for the 32-way word-coder decode kernel (VERDICT r1, item 1).
//
// Builds a valid container with the product library (rb200_model_from_data + rb200_encode on device buffers), then
// times kernel VARIANTS of the decoder on it with CUDA events: the round-1 kernel, the persistent TMA-ring kernel at
// several occupancies / group sizes / with and without the IMAD.WIDE field extraction, texture-pipe offload of every
// k-th table gather, and ablations that delete one term of the step (conflict-free gather, no symbol store, no ring
// read, no refill).  Ablated variants produce garbage; every other variant is verified byte for byte against the input.
// One JSON line per variant on stdout.  Not part of the product: links librans_b200.so, includes the kernel headers.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Iinclude -Iryg_rans_b200/csrc \
//        -o build/decode_lab tools/decode_lab.cu -Lryg_rans_b200 -lrans_b200 -Xlinker -rpath -Xlinker '$ORIGIN/../ryg_rans_b200'
//   build/decode_lab [--n BYTES] [--chunk SYMS] [--reps K] [--dist uniform|text|zipf] [--only NAME] [--peak GBS]
//                    [--coder word|alias]
// --coder alias: the same for alias_decode_persist_kernel (scale_bits 16; BASELINE configs[2] is --dist zipf): the shipped
// configuration, other occupancies, the repacked ("lean") bucket entry, and the ablations of its step.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "rans_b200.h"
#include "word_decode_tma.cuh"
#include "alias_kernels.cuh"

using namespace rb200;

#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) {                                                                   \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            std::exit(2);                                                                          \
        }                                                                                          \
    } while (0)
#define RB(call)                                                                    \
    do {                                                                            \
        int r_ = (call);                                                            \
        if (r_ != RB200_OK) {                                                       \
            std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, rb200_strerror(r_)); \
            std::exit(2);                                                           \
        }                                                                           \
    } while (0)

__device__ __forceinline__ uint32_t mix32(uint64_t v)
{
    v ^= v >> 33; v *= 0xff51afd7ed558ccdull; v ^= v >> 33; v *= 0xc4ceb9fe1a85ec53ull; v ^= v >> 33;
    return static_cast<uint32_t>(v);
}
// bytes drawn i.i.d. from a 65536-entry inverse-CDF table (uniform: table[i] = i >> 8)
__global__ void gen_kernel(uint8_t* out, uint64_t n, const uint8_t* icdf, uint64_t seed)
{
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < n; i += stride)
        out[i] = icdf[mix32(i + seed) >> 16];
}
__global__ void compare_kernel(const uint8_t* a, const uint8_t* b, uint64_t n, unsigned long long* bad)
{
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    unsigned long long local = 0;
    for (uint64_t i = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < n / 16; i += stride) {
        const uint4 x = reinterpret_cast<const uint4*>(a)[i], y = reinterpret_cast<const uint4*>(b)[i];
        local += (x.x != y.x) + (x.y != y.y) + (x.z != y.z) + (x.w != y.w);
    }
    if (local) atomicAdd(bad, local);
}

struct Bench {
    const uint8_t* blob; uint64_t blob_size; const uint64_t* offsets; const uint32_t* table; uint8_t* out; uint64_t n;
    uint32_t chunk; uint32_t n_chunks; DecodeWork* work; uint32_t* status; cudaTextureObject_t tex; int sms;
};

struct Variant {
    std::string name;
    bool verify;
    std::function<void(const Bench&)> launch;
    std::string note;
};

template <class P>
Variant tma_variant(const char* name, const char* note = "")
{
    Variant v;
    v.name = name;
    v.verify = P::kAblate == 0;
    v.note = note;
    v.launch = [](const Bench& b) {
        auto k = word_decode_tma_kernel<P, false>;
        static bool configured = false;
        if (!configured) {
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, P::kSmemBytes));
            CK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
            configured = true;
        }
        uint32_t grid = static_cast<uint32_t>(b.sms) * P::kMinBlocks;
        const uint32_t want = (b.n_chunks + P::kWarps - 1) / P::kWarps;
        if (grid > want) grid = want;
        k<<<grid, P::kWarps * 32, P::kSmemBytes>>>(b.blob, b.blob_size, b.offsets, b.table, b.out, b.n, b.chunk, b.n_chunks, b.work,
                                                   b.status, b.tex);
    };
    return v;
}

template <class P>
void describe(const char* name)
{
    cudaFuncAttributes a;
    auto k = word_decode_tma_kernel<P, false>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, P::kSmemBytes));
    CK(cudaFuncGetAttributes(&a, k));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, P::kWarps * 32, P::kSmemBytes));
    std::printf("{\"describe\": \"%s\", \"regs\": %d, \"smem_dyn\": %u, \"ctas_per_sm\": %d, \"warps_per_sm\": %d}\n", name, a.numRegs,
                P::kSmemBytes, occ, occ * P::kWarps);
}

// ---------------------------------------------------------------------------------------------------------------------
// --coder alias
struct AliasBench {
    const uint8_t* blob; uint64_t blob_size; const uint64_t* offsets; const AliasDecEntry* dec; uint8_t* out; uint64_t n;
    uint32_t chunk; uint32_t n_chunks; DecodeWork* work; uint32_t* status; int sms;
};
struct AliasVariant {
    std::string name;
    bool verify;
    std::function<void(const AliasBench&)> launch;
    std::function<void()> describe;
    std::string note;
};
template <class P, int LEAN>
AliasVariant alias_variant(const char* name, const char* note = "")
{
    AliasVariant v;
    v.name = name;
    v.verify = P::kAblate == 0;
    v.note = note;
    v.launch = [](const AliasBench& b) {
        auto k = alias_decode_persist_kernel<16, P, LEAN>;
        static bool configured = false;
        if (!configured) {
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, P::kSmemBytes));
            CK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
            configured = true;
        }
        uint32_t grid = static_cast<uint32_t>(b.sms) * P::kMinBlocks;
        const uint32_t want = (b.n_chunks + P::kWarps - 1) / P::kWarps;
        if (grid > want) grid = want;
        k<<<grid, P::kWarps * 32, P::kSmemBytes>>>(b.blob, b.blob_size, b.offsets, 16u, b.dec, b.out, b.n, b.chunk, b.n_chunks, b.work,
                                                   b.status);
    };
    const std::string nm = name;
    v.describe = [nm]() {
        cudaFuncAttributes a;
        auto k = alias_decode_persist_kernel<16, P, LEAN>;
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, P::kSmemBytes));
        CK(cudaFuncGetAttributes(&a, k));
        int occ = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, P::kWarps * 32, P::kSmemBytes));
        std::printf("{\"describe\": \"%s\", \"regs\": %d, \"smem_dyn\": %u, \"ctas_per_sm\": %d, \"warps_per_sm\": %d}\n", nm.c_str(),
                    a.numRegs, P::kSmemBytes, occ, occ * P::kWarps);
    };
    return v;
}

static int run_alias(uint64_t n, uint32_t chunk, int reps, const std::string& dist, const std::string& only, double peak, int sms,
                     const uint8_t* d_in, uint8_t* d_out)
{
    rb200_ctx* ctx = nullptr;
    RB(rb200_ctx_create(&ctx, 0, nullptr));
    rb200_model* model = nullptr;
    uint32_t freqs[256];
    RB(rb200_model_from_data(ctx, RB200_CODER_ALIAS, 16, d_in, n, RB200_MEM_DEVICE, freqs, &model));
    const size_t n_chunks = rb200_chunk_count(n, chunk);
    const size_t bound = rb200_encode_bound(n, chunk);
    uint8_t* d_blob;
    uint64_t* d_offsets;
    CK(cudaMalloc(&d_blob, bound + 16));
    CK(cudaMalloc(&d_offsets, (n_chunks + 1) * sizeof(uint64_t)));
    RB(rb200_encode(ctx, model, d_in, n, chunk, d_blob, bound, d_offsets, nullptr, RB200_MEM_DEVICE));
    RB(rb200_sync(ctx));
    uint64_t blob_size = 0;
    CK(cudaMemcpy(&blob_size, d_offsets + n_chunks, sizeof blob_size, cudaMemcpyDeviceToHost));

    AliasDeviceTables* t = new AliasDeviceTables;
    if (build_alias_device_tables(freqs, 16, *t) != 0) { std::fprintf(stderr, "alias table build failed\n"); return 2; }
    AliasDecEntry* d_dec;
    CK(cudaMalloc(&d_dec, sizeof t->dec));
    CK(cudaMemcpy(d_dec, t->dec, sizeof t->dec, cudaMemcpyHostToDevice));
    DecodeWork* d_work;
    uint32_t* d_status;
    unsigned long long* d_bad;
    CK(cudaMalloc(&d_work, sizeof(DecodeWork)));
    CK(cudaMalloc(&d_status, 4));
    CK(cudaMalloc(&d_bad, 8));
    CK(cudaMemset(d_work, 0, sizeof(DecodeWork)));

    AliasBench b{d_blob, blob_size, d_offsets, d_dec, d_out, n, chunk, static_cast<uint32_t>(n_chunks), d_work, d_status, sms};
    const double alg_bytes = static_cast<double>(n) + static_cast<double>(blob_size);
    std::printf("{\"lab\": \"alias_decode\", \"n\": %llu, \"chunk\": %u, \"dist\": \"%s\", \"blob_bytes\": %llu, \"sms\": %d, \"peak_gbs\": %.1f}\n",
                (unsigned long long)n, chunk, dist.c_str(), (unsigned long long)blob_size, sms, peak);

    constexpr uint32_t kTab = 256 * kAliasDecReplicas * 16;
    //                     warps, CTAs/SM, group, refill, log2(unit), -, -, ablate, -, table bytes
    using Ship = AliasDecShip;                                                  // 2 x 20 warps
    static_assert(Ship::kWarps == 20 && Ship::kMinBlocks == 2 && kAliasLean == 1, "the variant names below assume the shipped configuration");
    using W24 = DecPolicy<24, 2, 8, kRefillCpAsync, 9, 0, 0, 0, false, kTab>;
    using W16x3 = DecPolicy<16, 3, 8, kRefillCpAsync, 9, 0, 0, 0, false, kTab>;
    using W32x1 = DecPolicy<32, 1, 8, kRefillCpAsync, 9, 0, 0, 0, false, kTab>;
    using G4 = DecPolicy<20, 2, 4, kRefillCpAsync, 9, 0, 0, 0, false, kTab>;
    using A2 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblNoSymbolStore, false, kTab>;
    using A4 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblNoRingRead, false, kTab>;
    using A8 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblNoRefill, false, kTab>;
    using A16 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblAliasOneByte, false, kTab>;
    using A14 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblNoSymbolStore | kAblNoRingRead | kAblNoRefill, false, kTab>;
    using A26 = DecPolicy<20, 2, 8, kRefillCpAsync, 9, 0, 0, kAblNoSymbolStore | kAblNoRefill | kAblAliasOneByte, false, kTab>;
    std::vector<AliasVariant> vs;
    vs.push_back(alias_variant<Ship, 1>("ship", "SHIPPED: persistent, 2 x 20 warps/SM, 8x replicated 16-byte bucket entries repacked at staging (lean entry: two selects, no byte permute, compare at the top of a word), cp.async ring"));
    vs.push_back(alias_variant<Ship, 0>("plain_entry", "the bucket entry as the host packs it {divider, alt0, alt1, adjusts}: +2 ALU-pipe, -1 FMA-pipe instructions per step (the first persistent version of round 2)"));
    vs.push_back(alias_variant<W24, 1>("ship_w24x2", "48 warps/SM"));
    vs.push_back(alias_variant<W24, 0>("plain_entry_w24x2", "plain entry, 48 warps/SM"));
    vs.push_back(alias_variant<W16x3, 1>("ship_w16x3", "48 warps/SM in CTAs of 16"));
    vs.push_back(alias_variant<W32x1, 1>("ship_w32x1", "32 warps/SM"));
    vs.push_back(alias_variant<G4, 1>("ship_g4", "fill check / ring wrap every 4 steps"));
    vs.push_back(alias_variant<A2, 1>("abl_no_symbol_store", "ABLATION on ship: no STG.U8"));
    vs.push_back(alias_variant<A4, 1>("abl_no_ring_read", "ABLATION: renormalisation bytes = the address, no LDS.U8 pair"));
    vs.push_back(alias_variant<A8, 1>("abl_no_refill", "ABLATION: no ring refills / waits (blob never read)"));
    vs.push_back(alias_variant<A16, 1>("abl_one_byte", "ABLATION: at most one renormalisation byte per step (second vote / ranks / load / merge gone: -8 instructions)"));
    vs.push_back(alias_variant<A14, 1>("abl_memory_side", "ABLATION: store + ring reads + refill gone: arithmetic, two votes and the bucket gather remain"));
    vs.push_back(alias_variant<A26, 1>("abl_one_byte_no_store_no_refill"));
    if (only.empty()) for (const AliasVariant& v : vs) v.describe();

    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (const AliasVariant& v : vs) {
        if (!only.empty() && only != v.name) continue;
        CK(cudaMemset(d_out, 0xAA, n));
        CK(cudaMemset(d_status, 0, 4));
        CK(cudaMemset(d_work, 0, sizeof(DecodeWork)));
        v.launch(b);
        cudaError_t le = cudaDeviceSynchronize();
        if (le != cudaSuccess) {
            std::printf("{\"variant\": \"%s\", \"error\": \"%s\"}\n", v.name.c_str(), cudaGetErrorString(le));
            return 3;
        }
        std::vector<float> ms(reps);
        for (int r = 0; r < reps; r++) {
            CK(cudaEventRecord(e0));
            v.launch(b);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&ms[r], e0, e1));
        }
        CK(cudaGetLastError());
        uint32_t status = 0;
        CK(cudaMemcpy(&status, d_status, 4, cudaMemcpyDeviceToHost));
        unsigned long long bad = 0;
        if (v.verify) {
            CK(cudaMemset(d_bad, 0, 8));
            compare_kernel<<<sms * 8, 256>>>(d_in, d_out, n, d_bad);
            CK(cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost));
        }
        std::sort(ms.begin(), ms.end());
        const double med = ms[reps / 2], mn = ms[0];
        std::printf("{\"variant\": \"%s\", \"ms_min\": %.4f, \"ms_median\": %.4f, \"gsym_s\": %.1f, \"gbs\": %.1f, \"roofline_frac\": %.4f, "
                    "\"verified\": %s, \"mismatch_words\": %llu, \"status\": %u, \"note\": \"%s\"}\n",
                    v.name.c_str(), mn, med, n / med * 1e-6, alg_bytes / med * 1e-6, alg_bytes / med * 1e-6 / peak,
                    v.verify ? (bad == 0 && status == 0 ? "true" : "false") : "null", bad, status, v.note.c_str());
        std::fflush(stdout);
    }
    rb200_model_destroy(model);
    rb200_ctx_destroy(ctx);
    return 0;
}

int main(int argc, char** argv)
{
    uint64_t n = 1ull << 30;
    uint32_t chunk = 8192;
    int reps = 5;
    std::string dist = "uniform", only, coder = "word";
    double peak = 3350.0;                       // GB/s: H100 SXM data-sheet HBM3 bandwidth; --peak for a measured one
    for (int i = 1; i < argc; i++) {
        auto arg = [&](const char* f) { return std::strcmp(argv[i], f) == 0 && i + 1 < argc; };
        if (arg("--n")) n = std::strtoull(argv[++i], nullptr, 0);
        else if (arg("--chunk")) chunk = static_cast<uint32_t>(std::atoi(argv[++i]));
        else if (arg("--reps")) reps = std::atoi(argv[++i]);
        else if (arg("--dist")) dist = argv[++i];
        else if (arg("--only")) only = argv[++i];
        else if (arg("--peak")) peak = std::atof(argv[++i]);
        else if (arg("--coder")) coder = argv[++i];
    }
    CK(cudaSetDevice(0));
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));

    // ---- data: i.i.d. bytes from an inverse-CDF table
    std::vector<uint8_t> icdf(65536);
    if (dist == "uniform") {
        for (int i = 0; i < 65536; i++) icdf[i] = static_cast<uint8_t>(i >> 8);
    } else if (dist == "zipf") {      // Zipf(1.1) over all 256 byte values (BASELINE configs[2])
        std::vector<double> p(256);
        double tot = 0;
        for (int s = 0; s < 256; s++) { p[s] = std::pow(1.0 + s, -1.1); tot += p[s]; }
        double acc = 0; int s = 0;
        for (int i = 0; i < 65536; i++) {
            while (s < 255 && (acc + p[s]) / tot * 65536.0 <= i) acc += p[s++];
            icdf[i] = static_cast<uint8_t>(s);
        }
    } else {      // "text": Zipf(1.0) over 96 symbols, about 5 bits per symbol
        std::vector<double> p(256, 0.0);
        double tot = 0;
        for (int s = 0; s < 96; s++) { p[32 + s] = 1.0 / (1 + s); tot += p[32 + s]; }
        double acc = 0; int s = 0;
        for (int i = 0; i < 65536; i++) {
            while (s < 255 && (acc + p[s]) / tot * 65536.0 <= i) acc += p[s++];
            icdf[i] = static_cast<uint8_t>(s);
        }
    }
    uint8_t *d_icdf, *d_in, *d_out, *d_blob;
    CK(cudaMalloc(&d_icdf, 65536));
    CK(cudaMemcpy(d_icdf, icdf.data(), 65536, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&d_in, n + 16));
    CK(cudaMalloc(&d_out, n + 16));
    gen_kernel<<<sms * 8, 256>>>(d_in, n, d_icdf, 0x1234);
    CK(cudaDeviceSynchronize());
    if (coder == "alias") return run_alias(n, chunk, reps, dist, only, peak, sms, d_in, d_out);

    // ---- container from the product library
    rb200_ctx* ctx = nullptr;
    RB(rb200_ctx_create(&ctx, 0, nullptr));
    rb200_model* model = nullptr;
    uint32_t freqs[256];
    RB(rb200_model_from_data(ctx, RB200_CODER_WORD, 12, d_in, n, RB200_MEM_DEVICE, freqs, &model));
    const size_t n_chunks = rb200_chunk_count(n, chunk);
    const size_t bound = rb200_encode_bound(n, chunk);
    uint64_t* d_offsets;
    CK(cudaMalloc(&d_blob, bound + 16));
    CK(cudaMalloc(&d_offsets, (n_chunks + 1) * sizeof(uint64_t)));
    RB(rb200_encode(ctx, model, d_in, n, chunk, d_blob, bound, d_offsets, nullptr, RB200_MEM_DEVICE));
    RB(rb200_sync(ctx));
    uint64_t blob_size = 0;
    CK(cudaMemcpy(&blob_size, d_offsets + n_chunks, sizeof blob_size, cudaMemcpyDeviceToHost));

    WordDeviceTables* t = new WordDeviceTables;
    if (build_word_device_tables(freqs, *t) != 0 || t->wide) { std::fprintf(stderr, "table build failed\n"); return 2; }
    uint32_t* d_table;
    CK(cudaMalloc(&d_table, sizeof t->dec));
    CK(cudaMemcpy(d_table, t->dec, sizeof t->dec, cudaMemcpyHostToDevice));
    cudaResourceDesc rd{};
    rd.resType = cudaResourceTypeLinear;
    rd.res.linear.devPtr = d_table;
    rd.res.linear.desc = cudaCreateChannelDesc<unsigned int>();
    rd.res.linear.sizeInBytes = sizeof t->dec;
    cudaTextureDesc td{};
    td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex = 0;
    CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));

    DecodeWork* d_work;
    uint32_t* d_status;
    unsigned long long* d_bad;
    CK(cudaMalloc(&d_work, sizeof(DecodeWork)));
    CK(cudaMalloc(&d_status, 4));
    CK(cudaMalloc(&d_bad, 8));
    CK(cudaMemset(d_work, 0, sizeof(DecodeWork)));

    Bench b{d_blob, blob_size, d_offsets, d_table, d_out, n, chunk, static_cast<uint32_t>(n_chunks), d_work, d_status, tex, sms};
    const double alg_bytes = static_cast<double>(n) + static_cast<double>(blob_size);
    std::printf("{\"lab\": \"decode\", \"n\": %llu, \"chunk\": %u, \"dist\": \"%s\", \"blob_bytes\": %llu, \"sms\": %d, \"peak_gbs\": %.1f}\n",
                (unsigned long long)n, chunk, dist.c_str(), (unsigned long long)blob_size, sms, peak);

    std::vector<Variant> vs;
    //                       warps, CTAs/SM, group, refill, log2(unit), wide-mul (1 state, 2 entry), tex-every, ablate, iadd3
    using Ship = DecShip;
    using Tma512 = DecPolicy<32, 2, 8, kRefillTma, 9, 2>;
    using Tma1k20 = DecPolicy<20, 2, 8, kRefillTma, 10, 2>;
    using CpaW3 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 3>;
    using CpaW1 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 1>;
    using CpaW0 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 0>;
    using CpaI = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, 0, true>;
    using CpaG4 = DecPolicy<32, 2, 4, kRefillCpAsync, 9, 2>;
    using CpaW24 = DecPolicy<24, 2, 8, kRefillCpAsync, 9, 2>;
    using CpaW16x4 = DecPolicy<16, 4, 8, kRefillCpAsync, 9, 2>;
    using Cpa1k20 = DecPolicy<20, 2, 8, kRefillCpAsync, 10, 2>;
    using CpaT8 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 8>;
    using CpaT4 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 4>;
    using A1 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblGatherConflictFree>;
    using A2 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblNoSymbolStore>;
    using A4 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblNoRingRead>;
    using A8 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblNoRefill>;
    using A3 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblGatherConflictFree | kAblNoSymbolStore>;
    using A9 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, kAblGatherConflictFree | kAblNoRefill>;
    using A15 = DecPolicy<32, 2, 8, kRefillCpAsync, 9, 2, 0, 15>;
    vs.push_back(tma_variant<Ship>("ship", "SHIPPED: persistent, 2 x 32 warps/SM, TMA-staged table, ring of 4 x 512 B by cp.async (LDGSTS), freq/bias by one IMAD.WIDE"));
    vs.push_back(tma_variant<CpaW3>("ship_wide_both", "field extraction by two IMAD.WIDE (16 instead of 18 instructions per step)"));
    vs.push_back(tma_variant<CpaW1>("ship_wide_state", "IMAD.WIDE for x >> 12 / slot address only"));
    vs.push_back(tma_variant<CpaW0>("ship_shifts_only", "no IMAD.WIDE: every field by shift / mask (18 instructions per step)"));
    vs.push_back(tma_variant<CpaI>("ship_iadd3", "refill address and cursor update on the ALU pipe (IADD3) instead of IMAD"));
    vs.push_back(tma_variant<CpaG4>("ship_g4", "fill check / ring wrap every 4 steps instead of 8"));
    vs.push_back(tma_variant<CpaW24>("ship_w24x2", "48 warps/SM"));
    vs.push_back(tma_variant<CpaW16x4>("ship_w16x4", "CTAs of 16 warps"));
    vs.push_back(tma_variant<Cpa1k20>("ship_1k_w20x2", "ring of 4 x 1 KiB; 40 warps/SM"));
    vs.push_back(tma_variant<Tma512>("tma512_w32x2", "ring filled by cp.async.bulk (TMA) + one mbarrier per slot instead of LDGSTS"));
    vs.push_back(tma_variant<Tma1k20>("tma1k_w20x2", "ring of 4 x 1 KiB by TMA; 40 warps/SM"));
    vs.push_back(tma_variant<CpaT4>("tex_every4", "every 4th table gather through the TEX pipe (tex1Dfetch)"));
    vs.push_back(tma_variant<CpaT8>("tex_every8", "every 8th table gather through the TEX pipe"));
    vs.push_back(tma_variant<A1>("abl_gather_conflict_free", "ABLATION on ship: gather address forced to bank = lane"));
    vs.push_back(tma_variant<A2>("abl_no_symbol_store", "ABLATION: no STG.U8"));
    vs.push_back(tma_variant<A4>("abl_no_ring_read", "ABLATION: refill word = address, no LDS.U16"));
    vs.push_back(tma_variant<A8>("abl_no_refill", "ABLATION: no ring refills / waits (blob never read)"));
    vs.push_back(tma_variant<A3>("abl_cf_gather_no_store"));
    vs.push_back(tma_variant<A9>("abl_cf_gather_no_refill"));
    vs.push_back(tma_variant<A15>("abl_all", "ABLATION: all four -- what the ALU/issue side alone costs"));
    if (only.empty()) {
        describe<Ship>("ship"); describe<CpaW3>("ship_wide_both"); describe<Tma512>("tma512_w32x2");
        describe<CpaW24>("ship_w24x2"); describe<CpaW16x4>("ship_w16x4");
    }

    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (const Variant& v : vs) {
        if (!only.empty() && only != v.name) continue;
        CK(cudaMemset(d_out, 0xAA, n));
        CK(cudaMemset(d_status, 0, 4));
        CK(cudaMemset(d_work, 0, sizeof(DecodeWork)));
        v.launch(b);                                   // warm-up
        cudaError_t le = cudaDeviceSynchronize();
        if (le != cudaSuccess) {
            std::printf("{\"variant\": \"%s\", \"error\": \"%s\"}\n", v.name.c_str(), cudaGetErrorString(le));
            return 3;                                  // a faulted context cannot run the remaining variants
        }
        std::vector<float> ms(reps);
        for (int r = 0; r < reps; r++) {
            CK(cudaEventRecord(e0));
            v.launch(b);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&ms[r], e0, e1));
        }
        CK(cudaGetLastError());
        uint32_t status = 0;
        CK(cudaMemcpy(&status, d_status, 4, cudaMemcpyDeviceToHost));
        unsigned long long bad = 0;
        if (v.verify) {
            CK(cudaMemset(d_bad, 0, 8));
            compare_kernel<<<sms * 8, 256>>>(d_in, d_out, n, d_bad);
            CK(cudaMemcpy(&bad, d_bad, 8, cudaMemcpyDeviceToHost));
        }
        std::sort(ms.begin(), ms.end());
        const double med = ms[reps / 2], mn = ms[0];
        std::printf("{\"variant\": \"%s\", \"ms_min\": %.4f, \"ms_median\": %.4f, \"gsym_s\": %.1f, \"gbs\": %.1f, \"roofline_frac\": %.4f, "
                    "\"verified\": %s, \"mismatch_words\": %llu, \"status\": %u, \"note\": \"%s\"}\n",
                    v.name.c_str(), mn, med, n / med * 1e-6, alg_bytes / med * 1e-6, alg_bytes / med * 1e-6 / peak,
                    v.verify ? (bad == 0 && status == 0 ? "true" : "false") : "null", bad, status, v.note.c_str());
        std::fflush(stdout);
    }
    rb200_model_destroy(model);
    rb200_ctx_destroy(ctx);
    return 0;
}

// container_format.h -- the layout of the self-describing container (container_host.cpp has the format comment) and
// the one parser every container call goes through.  Internal to the library.
#pragma once
#include <cstddef>
#include <cstdint>

#include "hd.h"
#include "rans_b200.h"

// The layout and the rules below are compiled for the host and, under nvcc, for the device too (RB200_HD): the kernels
// of rb200_container_decode_async / rb200_container_blocks_decode_async / rb200_container_blocks_coder_decode_async
// (container_decode.cuh) apply the same functions as the host parser.

namespace rb200 {

constexpr uint32_t kContainerMagic = 0x43324252u;   // "RB2C"
constexpr uint16_t kContainerVersion = 1;           // one model: 256 x u32
constexpr uint16_t kContainerVersionBlocks = 2;     // one model per block: n_blocks x 256 x u16, word coder
constexpr uint16_t kContainerVersionBlocksCoder = 3;  // version 2's layout with the byte or rans64 coder at scale_bits 8..15
constexpr uint16_t kContainerVersionBlocksAlias = 4;  // version 2's layout with the alias coder at scale_bits 8..15
constexpr uint16_t kContainerVersionBlocksStored = 5; // the layout of versions 2-4 for any of their pairs, with stored blocks
constexpr uint16_t kContainerVersionStored = 6;       // version 1's layout with a stored-chunk bitmap before the blob

struct ContainerHeader {        // 64 bytes
    uint32_t magic;
    uint16_t version;
    uint8_t coder;
    uint8_t scale_bits;
    uint32_t lanes;
    uint32_t chunk_syms;
    uint64_t n_symbols;
    uint64_t n_chunks;
    uint64_t blob_bytes;
    uint32_t flags;
    uint32_t meta_crc;          // header (crc fields zero) + model + offsets
    uint32_t blob_crc;          // valid when flags & RB200_CONTAINER_CRC_BLOB
    uint32_t block_size;        // versions 2-4: symbols per block (version 1: zero, not checked)
    uint32_t n_blocks;          // versions 2-4: blocks, >= 1 (version 1: zero, not checked)
    uint32_t reserved;          // versions 2-4: zero
};
static_assert(sizeof(ContainerHeader) == 64, "container header must stay 64 bytes");

constexpr size_t kContainerDirOffset = sizeof(ContainerHeader) + 256 * sizeof(uint32_t);   // version 1: 1088, 16-aligned
constexpr size_t kBlockModelBytes = 256 * sizeof(uint16_t);                                 // one block's frequencies

// versions 2, 3 and 4: a model per block, n_blocks x 256 x u16 (version 1: one model, 256 x u32)
RB200_HD inline bool container_per_block(const ContainerHeader& h)
{
    return h.version >= kContainerVersionBlocks && h.version <= kContainerVersionBlocksAlias;
}

// The layout, as functions of the (parsed) header: model section, directory, pad to 16, blob.  Version 1 keeps 1024
// bytes of model, so its directory stays at 1088; the per-block versions have 512 bytes per block, so their directory
// starts at 64 + 512 n_blocks, also 16-aligned.  64-bit throughout: n_blocks < 2^32 and n_chunks < 2^31 once parsed.
RB200_HD inline uint64_t container_model_bytes(const ContainerHeader& h)
{
    return container_per_block(h) ? kBlockModelBytes * h.n_blocks : 256 * sizeof(uint32_t);
}
RB200_HD inline uint64_t container_dir_offset(const ContainerHeader& h) { return sizeof(ContainerHeader) + container_model_bytes(h); }
RB200_HD inline uint64_t container_dir_end(const ContainerHeader& h) { return container_dir_offset(h) + (h.n_chunks + 1) * sizeof(uint64_t); }
RB200_HD inline uint64_t container_blob_offset(const ContainerHeader& h) { return (container_dir_end(h) + 15) & ~15ull; }

// the per-block version of a coder: word 2, byte and rans64 3, alias 4
RB200_HD inline uint16_t container_blocks_version(uint32_t coder)
{
    return coder == RB200_CODER_WORD ? kContainerVersionBlocks : coder == RB200_CODER_ALIAS ? kContainerVersionBlocksAlias
                                                                                         : kContainerVersionBlocksCoder;
}

// The coder and scale_bits of each per-block version, for its headers and for the arguments of its calls: the word
// coder at 12 (version 2), byte or rans64 at 8..15 (version 3), alias at 8..15 (version 4)
RB200_HD inline bool container_blocks_coder_ok(uint16_t version, uint32_t coder, uint32_t scale_bits)
{
    if (version == kContainerVersionBlocks) return coder == RB200_CODER_WORD && scale_bits == 12;
    const bool coder_ok = version == kContainerVersionBlocksCoder ? coder == RB200_CODER_BYTE || coder == RB200_CODER_RANS64
                                                                  : version == kContainerVersionBlocksAlias && coder == RB200_CODER_ALIAS;
    return coder_ok && scale_bits >= 8 && scale_bits <= 15;
}

// a header with only what the layout depends on: for sizes computed before there is a header
inline ContainerHeader container_shape(uint16_t version, uint32_t n_blocks, uint64_t n_chunks)
{
    ContainerHeader h{};
    h.version = version;
    h.n_blocks = n_blocks;
    h.n_chunks = n_chunks;
    return h;
}

// the chunk sizes the kernels take (32 .. 2^24 symbols)
RB200_HD inline bool container_chunk_ok(uint32_t chunk_syms) { return chunk_syms >= 32 && chunk_syms <= (1u << 24); }
// per-block geometry: whole chunks per block, at most 32 (one CTA per block, one warp per chunk)
RB200_HD inline bool container_blocks_geometry_ok(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms)
{
    return n_blocks && block_size && container_chunk_ok(chunk_syms) && block_size % chunk_syms == 0 && block_size / chunk_syms <= 32;
}

// Every rule of a header (already read from the first 64 of `size` bytes) for the one `version` the caller accepts:
// the fields agree with each other and with the geometry the decoders take, and every section fits `size`.  The
// per-block versions share every rule but the coder and scale_bits (container_blocks_coder_ok).
RB200_HD inline bool container_header_ok(const ContainerHeader& h, uint64_t size, uint16_t version)
{
    if (h.magic != kContainerMagic || h.version != version || h.lanes != RB200_LANES || !h.chunk_syms) return false;
    if (container_per_block(h)) {
        // what rb200_blocks_decode / rb200_blocks_coder_decode / rb200_blocks_alias_decode accept; n_blocks * block_size
        // cannot overflow 64 bits
        if (!container_blocks_coder_ok(version, h.coder, h.scale_bits) || !container_blocks_geometry_ok(h.n_blocks, h.block_size, h.chunk_syms)) return false;
        if (h.n_symbols != static_cast<uint64_t>(h.n_blocks) * h.block_size || h.n_chunks != h.n_symbols / h.chunk_syms ||
            h.n_chunks >= (1ull << 31) || (h.blob_bytes & 15) || h.reserved || (h.flags & ~RB200_CONTAINER_CRC_BLOB))
            return false;
    } else if (h.n_chunks != h.n_symbols / h.chunk_syms + (h.n_symbols % h.chunk_syms != 0) || h.n_chunks >= (1ull << 31) ||
               (h.blob_bytes & 15) || h.coder > RB200_CODER_RANS64 || h.scale_bits < 8 || h.scale_bits > 16) {
        return false;
    }
    const uint64_t boff = container_blob_offset(h);                 // < 2^42: n_chunks < 2^31, n_blocks < 2^32
    return boff <= size && h.blob_bytes <= size - boff;
}

// Version 5 (stored blocks) is the header of its twin -- the per-block version of its coder (2, 3 or 4) -- with the
// version field 5: every header rule and the layout are the twin's, so the twin's header is what the layout functions
// above take.  A coder past rans64 has no twin (version 0, which no rule accepts).
RB200_HD inline ContainerHeader container_stored_twin(ContainerHeader h)
{
    h.version = h.coder <= RB200_CODER_RANS64 ? container_blocks_version(h.coder) : 0;
    return h;
}
RB200_HD inline bool container_stored_header_ok(const ContainerHeader& h, uint64_t size)
{
    const ContainerHeader t = container_stored_twin(h);
    return h.version == kContainerVersionBlocksStored && t.version && container_header_ok(t, size, t.version);
}
// the header whose layout a header has (host): version 5's twin, any other version itself
inline ContainerHeader container_layout(const ContainerHeader& h)
{
    return h.version == kContainerVersionBlocksStored ? container_stored_twin(h) : h;
}

// what rb200_model_create would accept: a known coder, its scale_bits range, frequencies that sum to 1 << scale_bits
RB200_HD inline bool container_model_ok(uint32_t coder, uint32_t scale_bits, const uint32_t* freqs)
{
    if (coder > RB200_CODER_RANS64 || scale_bits < 8 || scale_bits > 16) return false;
    if (coder == RB200_CODER_WORD && scale_bits != 12) return false;
    uint64_t sum = 0;
    for (int s = 0; s < 256; s++) sum += freqs[s];
    return sum == (1ull << scale_bits);
}

// What the decoders take beyond what rb200_container_open checks.  A version 1 container can pass open and still be
// refused by the decode: rb200_container_decode returns RB200_E_ARG for the geometry and RB200_E_MODEL for the model.
// chunks of 32 .. 2^24 symbols, and a blob below 2^36 bytes (the decoders index it in 16-byte vectors with 32 bits)
RB200_HD inline bool container_geometry_decodable(uint32_t chunk_syms, uint64_t blob_bytes)
{
    return container_chunk_ok(chunk_syms) && (blob_bytes >> 36) == 0;
}
// the byte coder's frequencies are below 65536 (RansDecSymbol.freq is 16 bits wide, rans_byte.h:168-171)
RB200_HD inline bool container_model_decodable(uint32_t coder, const uint32_t* freqs)
{
    if (coder != RB200_CODER_BYTE) return true;
    for (int s = 0; s < 256; s++)
        if (freqs[s] >= 65536u) return false;
    return true;
}

// The coder choice of rb200_choose_coder and rb200_container_model_encode_auto_async (coder_choice_kernel), the same
// integer steps on host and device.  A candidate is RB200_CANDIDATE(coder, scale_bits).
// a pair rb200_container_model_encode_async accepts: word at 12; byte, alias or rans64 at 8..16
RB200_HD inline bool candidate_ok(uint32_t c)
{
    const uint32_t coder = c >> 8, sb = c & 0xffu;
    if (coder == RB200_CODER_WORD) return sb == 12;
    return coder <= RB200_CODER_RANS64 && sb >= 8 && sb <= 16;
}
// 1..16 valid candidates, no two alike
inline bool candidate_list_ok(const uint32_t* c, uint32_t n)
{
    if (!c || n == 0 || n > 16) return false;
    for (uint32_t i = 0; i < n; i++) {
        if (!candidate_ok(c[i])) return false;
        for (uint32_t j = 0; j < i; j++)
            if (c[j] == c[i]) return false;
    }
    return true;
}
// log2(f) in 16.16 fixed point, by squaring the mantissa: x = f << (31 - k) holds f / 2^k in [1, 2) as x / 2^31; each
// squaring that reaches 2 gives one fraction bit.  f <= 65536.
RB200_HD inline uint32_t log2q(uint32_t f)
{
    uint32_t k = 0;
    while ((f >> k) > 1) k++;
    uint64_t x = static_cast<uint64_t>(f) << (31 - k);
    uint32_t r = k << 16;
    for (int i = 15; i >= 0; i--) {
        x = (x * x) >> 31;
        if (x >= (1ull << 32)) {
            x >>= 1;
            r |= 1u << i;
        }
    }
    return r;
}
// symbol s's share of bits_q: count * -log2(f / 2^sb) in 16.16 (0 for a symbol that does not occur).  A symbol that
// occurs has f >= 1 once normalised, so the term is at most count * 2^20 and bits_q stays below 2^52 for n < 2^32.
RB200_HD inline uint64_t candidate_bits_q(uint32_t count, uint32_t f, uint32_t sb)
{
    return count ? static_cast<uint64_t>(count) * ((sb << 16) - log2q(f)) : 0;
}
// estimated container blob bytes: the coded bits, rounded up to bytes, and the 32 final states of every chunk
RB200_HD inline uint64_t candidate_cost(uint64_t bits_q, uint64_t n_chunks, uint32_t coder)
{
    return ((bits_q + (1ull << 19) - 1) >> 19) + n_chunks * (coder == RB200_CODER_RANS64 ? 256u : 128u);
}
// the first candidate whose cost is within tolerance_ppm of the smallest, or -1 when every cost is UINT64_MAX
RB200_HD inline int choose_candidate(const uint64_t* costs, uint32_t n, uint32_t tolerance_ppm)
{
    uint64_t min = ~0ull;
    for (uint32_t i = 0; i < n; i++) min = costs[i] < min ? costs[i] : min;
    if (min == ~0ull) return -1;
    const uint64_t bound = min + min * tolerance_ppm / 1000000u;        // min < 2^40, tolerance_ppm <= 10^6
    for (uint32_t i = 0; i < n; i++)
        if (costs[i] <= bound) return static_cast<int>(i);
    return -1;
}

// The per-block coder choice of rb200_choose_blocks_coder and rb200_container_blocks_model_encode_auto_async
// (blocks_choice_kernel): C7's steps per block, summed over the blocks.  A candidate is a pair some per-block version
// takes (container_blocks_coder_ok): word at 12, byte, rans64 or alias at 8..15.
RB200_HD inline bool blocks_candidate_ok(uint32_t c)
{
    const uint32_t coder = c >> 8, sb = c & 0xffu;
    return coder <= RB200_CODER_RANS64 && container_blocks_coder_ok(container_blocks_version(coder), coder, sb);
}
// 1..16 valid candidates, no two alike
inline bool blocks_candidate_list_ok(const uint32_t* c, uint32_t n)
{
    if (!candidate_list_ok(c, n)) return false;
    for (uint32_t i = 0; i < n; i++)
        if (!blocks_candidate_ok(c[i])) return false;
    return true;
}
// One block's cost under a candidate: candidate_cost of the block's bits_q and chunks, except for the word coder on a
// block of one symbol (one_symbol: a frequency of 4096), where K5's WIDE step writes a 16-bit word per symbol, so every
// chunk is 2 x chunk_syms + 128 bytes; rule C7 counts 0 bits there.
RB200_HD inline uint64_t blocks_candidate_cost(uint64_t bits_q, uint32_t block_size, uint32_t chunk_syms, uint32_t coder, bool one_symbol)
{
    const uint32_t per_block = block_size / chunk_syms;
    if (coder == RB200_CODER_WORD && one_symbol) return 2ull * block_size + 128ull * per_block;
    return candidate_cost(bits_q, per_block, coder);
}

// The per-element rules of a prefix, one block or one directory entry at a time.
// one block's 256 frequencies sum to total: 1 << scale_bits (4096 in version 2)
RB200_HD inline bool container_block_model_sums_to(const uint16_t* freqs, uint32_t total)
{
    uint32_t sum = 0;
    for (int s = 0; s < 256; s++) sum += freqs[s];
    return sum == total;
}
// entry c (< n_chunks) of the directory is not above the next one
RB200_HD inline bool container_dir_step_ok(const uint64_t* offsets, uint64_t c) { return offsets[c] <= offsets[c + 1]; }
// the first stream starts inside the first vector, the last entry is the blob size
RB200_HD inline bool container_dir_ends_ok(const uint64_t* offsets, uint64_t n_chunks, uint64_t blob_bytes)
{
    return offsets[n_chunks] == blob_bytes && (!n_chunks || offsets[0] < 16);
}

// Version 5: a block whose row is all zero is stored; every other row sums to 1 << scale_bits (container_block_model_sums_to)
RB200_HD inline bool container_block_model_stored(const uint16_t* freqs) { return container_block_model_sums_to(freqs, 0); }
// the stream of a stored chunk: its chunk_syms symbols, then zero bytes up to a multiple of 16
RB200_HD inline uint64_t container_stored_bytes(uint32_t chunk_syms) { return (chunk_syms + 15ull) & ~15ull; }
// chunk c of a stored block: its stream [offsets[c], offsets[c + 1] & ~15) is container_stored_bytes long and lies in the
// blob (so its bytes can be read once this holds, whatever the other entries say)
RB200_HD inline bool container_stored_step_ok(const uint64_t* offsets, uint64_t c, uint32_t chunk_syms, uint64_t blob_bytes)
{
    const uint64_t end = offsets[c + 1] & ~15ull;
    return end >= offsets[c] && end - offsets[c] == container_stored_bytes(chunk_syms) && end <= blob_bytes;
}
// and its padding, the bytes after the symbols, is zero
RB200_HD inline bool container_stored_pad_ok(const uint8_t* stream, uint32_t chunk_syms)
{
    for (uint64_t i = chunk_syms; i < container_stored_bytes(chunk_syms); i++)
        if (stream[i]) return false;
    return true;
}

// Version 6 (single model, stored chunks): version 1's header, model and directory at 1088, then, from the next
// 16-byte boundary, the stored-chunk bitmap -- ceil(n_chunks / 32) u32 words, bit c % 32 of word c / 32 set when chunk c
// is stored, zero-padded to 16 bytes -- then the blob.  meta_crc covers every byte before the blob: the header (crc
// fields zero), the model, the directory, the zero pad after it and the bitmap with its padding.
RB200_HD inline uint64_t container_bitmap_offset(uint64_t n_chunks) { return (kContainerDirOffset + (n_chunks + 1) * sizeof(uint64_t) + 15) & ~15ull; }
// the bitmap's words with its padding: a multiple of 4
RB200_HD inline uint64_t container_bitmap_words(uint64_t n_chunks) { return ((n_chunks + 31) / 32 + 3) & ~3ull; }
RB200_HD inline uint64_t container_bitmap_blob_offset(uint64_t n_chunks)
{
    return container_bitmap_offset(n_chunks) + container_bitmap_words(n_chunks) * sizeof(uint32_t);
}
// version 6's header rules: version 1's, with block_size, n_blocks and reserved zero and the bitmap's blob offset
RB200_HD inline bool container_chunks_stored_header_ok(const ContainerHeader& h, uint64_t size)
{
    if (h.version != kContainerVersionStored || h.block_size || h.n_blocks || h.reserved) return false;
    ContainerHeader v1 = h;
    v1.version = kContainerVersion;
    if (!container_header_ok(v1, size, kContainerVersion)) return false;
    const uint64_t boff = container_bitmap_blob_offset(h.n_chunks);
    return boff <= size && h.blob_bytes <= size - boff;
}
// m_c: the symbols of chunk c, chunk_syms but for a ragged last chunk
RB200_HD inline uint32_t container_chunk_symbols(uint64_t c, uint32_t chunk_syms, uint64_t n_symbols)
{
    const uint64_t left = n_symbols - c * chunk_syms;
    return left < chunk_syms ? static_cast<uint32_t>(left) : chunk_syms;
}
// chunk c's bit
RB200_HD inline bool container_chunk_stored(const uint32_t* bits, uint64_t c) { return (bits[c >> 5] >> (c & 31)) & 1u; }
// word w of the bitmap (padding included) has no bit at or past n_chunks
RB200_HD inline bool container_bitmap_word_ok(const uint32_t* bits, uint64_t w, uint64_t n_chunks)
{
    if (32 * w >= n_chunks) return bits[w] == 0;
    return n_chunks - 32 * w >= 32 || (bits[w] >> (n_chunks - 32 * w)) == 0;
}
// chunk c of version 6 is well formed: its directory step (every entry), and when its bit is set the step and zero
// padding of a stored stream of m_c symbols (container_stored_step_ok, container_stored_pad_ok: the padding is read
// only once the step puts the stream inside the blob)
RB200_HD inline bool container_v6_chunk_ok(const uint64_t* offsets, const uint32_t* bits, const uint8_t* blob, uint64_t c, uint32_t chunk_syms,
                                        uint64_t n_symbols, uint64_t blob_bytes)
{
    if (!container_dir_step_ok(offsets, c)) return false;
    if (!container_chunk_stored(bits, c)) return true;
    const uint32_t m = container_chunk_symbols(c, chunk_syms, n_symbols);
    return container_stored_step_ok(offsets, c, m, blob_bytes) && container_stored_pad_ok(blob + offsets[c], m);
}

// Version 7 (byte planes): a 64-byte header, a table of w {offset, size} entries, then w version 6 containers with no
// gaps, plane p holding byte p of every w-byte element.  The header: coder and scale_bits 0, lanes 32, chunk_syms, n
// input bytes (a nonzero multiple of w, n / w < 2^32), n_chunks 0, blob_bytes the bytes after the table, the caller's
// flags, meta_crc over the header (crc fields zero) and the table, blob_crc 0, block_size = n_blocks = w, reserved 0.
// Every plane is a version 6 container of n / w symbols with the header's chunk_syms and flags.
constexpr uint16_t kContainerVersionPlanes = 7;
struct PlaneEntry {
    uint64_t offset, size;
};
static_assert(sizeof(PlaneEntry) == 16, "plane table entries are 16 bytes");
RB200_HD inline bool container_planes_w_ok(uint32_t w) { return w == 2 || w == 4 || w == 8; }
// plane 0's offset, 16-aligned: the end of the table, and of the directory of dir_bytes after it (version 9; 0 for
// versions 7 and 8)
RB200_HD inline uint64_t container_planes_table_end(uint32_t w, uint64_t dir_bytes)
{
    return sizeof(ContainerHeader) + sizeof(PlaneEntry) * w + dir_bytes;
}
// Version 8 (a delta from a base tensor): version 7's layout and rules but for two header fields, version 8 and
// reserved = the CRC-32 of the base tensor's n bytes (covered by meta_crc, which zeroes only the two crc fields).  The
// planes hold d, not the input: for element i with x and b the w-byte little-endian integers of the input and the
// base, s = (x - b) mod 2^(8w) read as signed, d = (s << 1) ^ (s >> (8w - 1)) (arithmetic shift), byte k of d in plane
// k; the inverse x = b + ((d >> 1) ^ -(d & 1)) mod 2^(8w) is exact for every bit pattern.
constexpr uint16_t kContainerVersionDelta = 8;
// Version 9 (a list of tensors of one element width): version 7 of the concatenation of the T tensors' bytes, in list
// order with no padding, with a directory of the tensors' byte lengths between the table and plane 0.  The header
// differs from version 7's in n_blocks = T (1 <= T <= 2^20) and reserved = the CRC-32 of the directory's 8 T bytes
// (covered by meta_crc); n_symbols is the total n.  The directory is T u64 lengths, each a multiple of w (zero
// allowed), summing to n, zero-padded to 16 bytes; blob_bytes counts the planes' bytes, from plane 0's offset.
constexpr uint16_t kContainerVersionTensors = 9;
constexpr uint32_t kContainerTensorsMax = 1u << 20;
// the directory's bytes with its padding
RB200_HD inline uint64_t container_tensors_dir_bytes(uint32_t count) { return (8ull * count + 15) & ~15ull; }
// the directory bytes of a header of `version` (none for versions 7 and 8)
RB200_HD inline uint64_t container_planes_dir_bytes(const ContainerHeader& h, uint16_t version)
{
    return version == kContainerVersionTensors ? container_tensors_dir_bytes(h.n_blocks) : 0;
}
// the header rules of version 7, 8 or 9 (`version`, the one the caller accepts); the table, the directory and the
// planes fit `size`.  Only version 7 requires reserved == 0; only version 9 has n_blocks other than w.
RB200_HD inline bool container_planes_header_version_ok(const ContainerHeader& h, uint64_t size, uint16_t version)
{
    if (h.magic != kContainerMagic || h.version != version || h.coder || h.scale_bits || h.lanes != RB200_LANES) return false;
    const bool list_ok = version == kContainerVersionTensors ? h.n_blocks && h.n_blocks <= kContainerTensorsMax : h.n_blocks == h.block_size;
    if (!container_planes_w_ok(h.block_size) || !list_ok || h.n_chunks || h.blob_crc) return false;
    if (version == kContainerVersionPlanes && h.reserved) return false;
    if (!container_chunk_ok(h.chunk_syms) || !h.n_symbols || h.n_symbols % h.block_size || ((h.n_symbols / h.block_size) >> 32)) return false;
    const uint64_t t = container_planes_table_end(h.block_size, container_planes_dir_bytes(h, version));
    return t <= size && h.blob_bytes <= size - t;
}
// version 7's header rules; the table and the planes fit `size`
RB200_HD inline bool container_planes_header_ok(const ContainerHeader& h, uint64_t size)
{
    return container_planes_header_version_ok(h, size, kContainerVersionPlanes);
}
// the table: plane 0 right after it and the directory of dir_bytes (0 but for version 9), every plane right after the
// previous one, each at least a header long and a multiple of 16, and the last one ending where the blob does
RB200_HD inline bool container_planes_table_ok(const ContainerHeader& h, const PlaneEntry* t, uint64_t dir_bytes)
{
    uint64_t end = container_planes_table_end(h.block_size, dir_bytes);
    const uint64_t last = end + h.blob_bytes;
    for (uint32_t p = 0; p < h.block_size; p++) {
        if (t[p].offset != end || (t[p].size & 15) || t[p].size < sizeof(ContainerHeader) || t[p].size > last - end) return false;
        end += t[p].size;
    }
    return end == last;
}
// plane p's header (ph, read from the start of its size bytes): version 6 with n / w symbols, the header's chunk_syms
// and flags, and exactly size bytes long
RB200_HD inline bool container_planes_plane_ok(const ContainerHeader& h, const ContainerHeader& ph, uint64_t size)
{
    return ph.n_symbols == h.n_symbols / h.block_size && ph.chunk_syms == h.chunk_syms && ph.flags == h.flags &&
           container_chunks_stored_header_ok(ph, size) && container_bitmap_blob_offset(ph.n_chunks) + ph.blob_bytes == size;
}
// Version 9's directory rule, on entries [begin, end) of the T lengths `dir` of a header with w and n: each a
// multiple of w (2, 4 or 8) and at most n (so the sum of all T, below 2^20 n, cannot overflow); *sum accumulates them.  The
// directory passes when every part passes, the parts' sums add up to n and the padding word (dir[T], when T is odd) is
// zero.
RB200_HD inline bool container_tensors_dir_part_ok(const uint64_t* dir, uint32_t begin, uint32_t end, uint32_t w, uint64_t n, uint64_t* sum)
{
    bool ok = true;
    for (uint32_t i = begin; i < end; i++) {
        ok = ok && (dir[i] & (w - 1)) == 0 && dir[i] <= n;
        *sum += dir[i] <= n ? dir[i] : 0;
    }
    return ok;
}
RB200_HD inline bool container_tensors_dir_pad_ok(const uint64_t* dir, uint32_t count) { return count % 2 == 0 || dir[count] == 0; }

// the header rb200_container_pack writes (crc fields zero)
ContainerHeader container_header(int coder, uint32_t scale_bits, uint32_t chunk_syms, uint64_t n, uint64_t n_chunks,
                                 uint64_t blob_bytes, uint32_t flags);
// the header rb200_container_blocks_pack writes (crc fields zero)
ContainerHeader container_blocks_header(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, uint64_t blob_bytes, uint32_t flags);
// the header rb200_container_blocks_coder_pack (version 3) or rb200_container_blocks_alias_pack (version 4) writes (crc
// fields zero)
ContainerHeader container_blocks_coder_header(uint16_t version, int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                              uint64_t blob_bytes, uint32_t flags);
// version 5: every row is stored or sums to 1 << h.scale_bits, and every chunk of a stored block has its step and zero
// padding (container_stored_step_ok, container_stored_pad_ok); the directory rules hold already
bool container_stored_rows_ok(const ContainerHeader& h, const uint16_t* rows, const uint64_t* offsets, const uint8_t* blob);
// every block's 256 frequencies sum to total
bool container_block_models_sum_to(const uint16_t* block_freqs, uint32_t n_blocks, uint32_t total);
// the directory rules: the first stream starts inside the first vector, monotone, last entry == blob_bytes
bool container_directory_ok(const uint64_t* offsets, uint64_t n_chunks, uint64_t blob_bytes);
// zlib crc32 on the host (slicing-by-8)
uint32_t container_crc32(uint32_t crc, const void* data, size_t len);
// CRC-32 of the header with its crc fields zeroed: the first 64 bytes of what meta_crc covers
uint32_t container_header_crc(const ContainerHeader& h);
// meta_crc over header, model section (container_model_bytes(h) bytes) and offsets, on the host
uint32_t container_meta_crc(const ContainerHeader& h, const void* model, const uint64_t* offsets);

// The parser, in the order rb200_container_open applies it.  Each step returns RB200_OK or RB200_E_STREAM; the CRC
// values are the caller's, computed wherever the bytes live.
//  1. the 64-byte header against the buffer size (`size` bytes in all; `hdr` holds at least 64 of them); `version`
//     is the one the caller accepts (kContainerVersion, kContainerVersionBlocks, kContainerVersionBlocksCoder,
//     kContainerVersionBlocksAlias or kContainerVersionBlocksStored), any other is rejected
int container_parse_header(const uint8_t* hdr, size_t size, uint16_t version, ContainerHeader* h);
//  2. header + model + directory (`prefix`: container_blob_offset(h) bytes), given their CRC; version 5 (`buf`, its
//     blob included): the stored chunks' steps and padding as well
int container_check_prefix(const ContainerHeader& h, const uint8_t* prefix, uint32_t meta_crc);
//  3. the blob, given its CRC (only consulted when the header carries one)
int container_check_blob(const ContainerHeader& h, uint32_t blob_crc);

}  // namespace rb200

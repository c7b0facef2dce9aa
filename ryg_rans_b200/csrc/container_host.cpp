// container_host.cpp -- self-describing wire format around (model, directory, blob)  [SURVEY 8f.3].
//
// The reference defines no container: its drivers keep a pointer and the sizes in local variables
// (main.cpp:182-188).  The bulk API's natural output (blob + offsets + the caller's freqs) is enough
// for in-process use; this file adds the versioned, checksummed envelope needed to ship it:
//
//   version 1 (one model):       [ 64-byte header ][ freqs: 256 x u32 ][ offsets: (n_chunks + 1) x u64 ][ pad to 16 ][ blob ]
//   version 2 (a model per block): [ 64-byte header ][ block_freqs: n_blocks x 256 x u16 ][ offsets ][ pad to 16 ][ blob ]
//   version 3 (a model per block, byte or rans64 coder): version 2's layout
//   version 4 (a model per block, alias coder): version 2's layout
//
// All integers little-endian.  CRC-32 (zlib's: IEEE, reflected) over header (with the crc fields zeroed) + model +
// offsets always (meta_crc); over the blob when RB200_CONTAINER_CRC_BLOB is set.  The header layout is the same in
// every version.  Version 1 has its directory at 1088; version 2 (word coder, scale_bits 12, 32 lanes) carries
// block_size at byte 52 and n_blocks at byte 56, its model section is 512 n_blocks bytes, so its directory starts at
// 64 + 512 n_blocks, and the u32 at byte 60 is zero.  Its chunk order is the per-block calls': chunk = block *
// (block_size / chunk_syms) + chunk-in-block, so each block's chunks are ordinary 32-way word streams under that
// block's row of block_freqs.  A version 2 container is valid only if: chunk_syms and block_size are what
// rb200_blocks_decode accepts (block_size % chunk_syms == 0, at most 32 chunks per block), n_blocks >= 1,
// n_symbols == n_blocks * block_size, n_chunks == n_symbols / chunk_syms < 2^31, blob_bytes % 16 == 0, every section
// fits the buffer, no flag but RB200_CONTAINER_CRC_BLOB, meta_crc matches, every block's frequencies sum to 4096, the
// directory rules of version 1 hold (offsets[0] < 16, monotone, offsets[n_chunks] == blob_bytes), and the blob CRC
// matches when present.  Version 3 is version 2 with the header's own coder (RB200_CODER_BYTE or RB200_CODER_RANS64) and
// scale_bits (8..15); every other rule is version 2's, and in both every block's frequencies sum to 1 << scale_bits.
// Version 4 is version 3 with RB200_CODER_ALIAS (the per-block main_alias.cpp coder), also at 8..15.  Each call accepts
// exactly one version: rb200_container_* version 1, rb200_container_blocks_* version 2, rb200_container_blocks_coder_*
// version 3, rb200_container_blocks_alias_* version 4.
//
//   version 7 (byte planes):     [ 64-byte header ][ w x {u64 offset, u64 size} ][ plane 0: a version 6 container ] ... [ plane w-1 ]
//
// Plane p holds byte p of every w-byte element; the rules are container_planes_* in container_format.h, and each plane
// is checked by rb200_container_stored_open's.
//
//   version 8 (a delta from a base tensor): version 7's layout, version 8, reserved = CRC-32 of the base's n bytes
//
// Its planes hold the zigzag difference from the base (container_format.h); the _delta_ calls accept only version 8.
//
//   version 9 (a list of tensors): [ 64-byte header ][ w x {u64 offset, u64 size} ][ T x u64 lengths, pad to 16 ][ plane 0 ] ...
//
// Version 7 of the tensors' concatenated bytes, with n_blocks = T and reserved = CRC-32 of the directory's 8 T bytes
// (container_format.h); the _tensors_ calls accept only version 9.
//
// rb200_container_pack / _open and the _blocks_ forms here work on host buffers with a host CRC (slicing-by-8, ~1 GB/s
// on one core: the blob CRC is optional for that reason).  rb200_container_encode / _decode and the _blocks_ forms
// (rans_b200.cu) write and read the same bytes in host or device memory with the blob CRC on the GPU
// (crc_kernels.cuh); they validate through the parser below, so both sides apply one set of rules.  The _decode_async
// forms apply the same rules in kernels (container_decode.cuh): the header, model and per-element rules are the
// __host__ __device__ functions of container_format.h that the parser below calls.
#include "container_format.h"

#include <cstring>
#include <vector>

namespace rb200 {

namespace {

struct CrcTable {
    uint32_t t[8][256];
    CrcTable()
    {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
            t[0][i] = c;
        }
        for (uint32_t i = 0; i < 256; i++)
            for (int k = 1; k < 8; k++) t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xff];
    }
};

}  // namespace

uint32_t container_crc32(uint32_t crc, const void* data, size_t len)     // slicing-by-8
{
    static const CrcTable table;                                      // built once, thread-safe (C++11 static)
    const uint32_t (*T)[256] = table.t;
    const uint8_t* p = static_cast<const uint8_t*>(data);
    crc = ~crc;
    while (len >= 8) {
        uint32_t a, b;
        std::memcpy(&a, p, 4);
        std::memcpy(&b, p + 4, 4);
        a ^= crc;
        crc = T[7][a & 0xff] ^ T[6][(a >> 8) & 0xff] ^ T[5][(a >> 16) & 0xff] ^ T[4][a >> 24]
            ^ T[3][b & 0xff] ^ T[2][(b >> 8) & 0xff] ^ T[1][(b >> 16) & 0xff] ^ T[0][b >> 24];
        p += 8;
        len -= 8;
    }
    while (len--) crc = (crc >> 8) ^ T[0][(crc ^ *p++) & 0xff];
    return ~crc;
}

uint32_t container_header_crc(const ContainerHeader& h)
{
    ContainerHeader z = h;
    z.meta_crc = 0;
    z.blob_crc = 0;
    return container_crc32(0, &z, sizeof z);
}

uint32_t container_meta_crc(const ContainerHeader& h, const void* model, const uint64_t* offsets)
{
    uint32_t c = container_header_crc(h);
    c = container_crc32(c, model, container_model_bytes(container_layout(h)));
    return container_crc32(c, offsets, (h.n_chunks + 1) * sizeof(uint64_t));
}

bool container_block_models_sum_to(const uint16_t* block_freqs, uint32_t n_blocks, uint32_t total)
{
    for (uint64_t b = 0; b < n_blocks; b++)
        if (!container_block_model_sums_to(block_freqs + b * 256, total)) return false;
    return true;
}

bool container_stored_rows_ok(const ContainerHeader& h, const uint16_t* rows, const uint64_t* offsets, const uint8_t* blob)
{
    const uint32_t per_block = h.block_size / h.chunk_syms;
    for (uint64_t b = 0; b < h.n_blocks; b++) {
        const uint16_t* row = rows + b * 256;
        if (!container_block_model_stored(row)) {
            if (!container_block_model_sums_to(row, 1u << h.scale_bits)) return false;
            continue;
        }
        for (uint64_t c = b * per_block; c < (b + 1) * per_block; c++)
            if (!container_stored_step_ok(offsets, c, h.chunk_syms, h.blob_bytes) || !container_stored_pad_ok(blob + offsets[c], h.chunk_syms))
                return false;
    }
    return true;
}

bool container_directory_ok(const uint64_t* offsets, uint64_t n_chunks, uint64_t blob_bytes)
{
    if (!container_dir_ends_ok(offsets, n_chunks, blob_bytes)) return false;
    for (uint64_t c = 0; c < n_chunks; c++)
        if (!container_dir_step_ok(offsets, c)) return false;
    return true;
}

ContainerHeader container_header(int coder, uint32_t scale_bits, uint32_t chunk_syms, uint64_t n, uint64_t n_chunks,
                                 uint64_t blob_bytes, uint32_t flags)
{
    ContainerHeader h{};
    h.magic = kContainerMagic;
    h.version = kContainerVersion;
    h.coder = static_cast<uint8_t>(coder);
    h.scale_bits = static_cast<uint8_t>(scale_bits);
    h.lanes = RB200_LANES;
    h.chunk_syms = chunk_syms;
    h.n_symbols = n;
    h.n_chunks = n_chunks;
    h.blob_bytes = blob_bytes;
    h.flags = flags & RB200_CONTAINER_CRC_BLOB;
    return h;
}

ContainerHeader container_blocks_header(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, uint64_t blob_bytes, uint32_t flags)
{
    const uint64_t n = static_cast<uint64_t>(n_blocks) * block_size;
    ContainerHeader h = container_header(RB200_CODER_WORD, 12, chunk_syms, n, n / chunk_syms, blob_bytes, flags);
    h.version = kContainerVersionBlocks;
    h.block_size = block_size;
    h.n_blocks = n_blocks;
    return h;
}

ContainerHeader container_blocks_coder_header(uint16_t version, int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size,
                                              uint32_t chunk_syms, uint64_t blob_bytes, uint32_t flags)
{
    ContainerHeader h = container_blocks_header(n_blocks, block_size, chunk_syms, blob_bytes, flags);
    h.version = version;
    h.coder = static_cast<uint8_t>(coder);
    h.scale_bits = static_cast<uint8_t>(scale_bits);
    return h;
}

int container_parse_header(const uint8_t* hdr, size_t size, uint16_t version, ContainerHeader* out)
{
    if (size < sizeof(ContainerHeader)) return RB200_E_STREAM;
    ContainerHeader h;
    std::memcpy(&h, hdr, sizeof h);
    const bool ok = version == kContainerVersionBlocksStored ? container_stored_header_ok(h, size) : container_header_ok(h, size, version);
    if (!ok) return RB200_E_STREAM;
    *out = h;
    return RB200_OK;
}

int container_check_prefix(const ContainerHeader& h, const uint8_t* prefix, uint32_t meta_crc)
{
    const uint8_t* model = prefix + sizeof(ContainerHeader);
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(prefix + container_dir_offset(container_layout(h)));
    if (meta_crc != h.meta_crc) return RB200_E_STREAM;
    if (h.version == kContainerVersionBlocksStored) {
        const uint16_t* rows = reinterpret_cast<const uint16_t*>(model);
        if (!container_directory_ok(offsets, h.n_chunks, h.blob_bytes)) return RB200_E_STREAM;
        return container_stored_rows_ok(h, rows, offsets, prefix + container_blob_offset(container_layout(h))) ? RB200_OK : RB200_E_STREAM;
    }
    const bool model_ok = container_per_block(h)
                              ? container_block_models_sum_to(reinterpret_cast<const uint16_t*>(model), h.n_blocks, 1u << h.scale_bits)
                              : container_model_ok(h.coder, h.scale_bits, reinterpret_cast<const uint32_t*>(model));
    if (!model_ok) return RB200_E_STREAM;                                                  // CRC-valid but inconsistent
    return container_directory_ok(offsets, h.n_chunks, h.blob_bytes) ? RB200_OK : RB200_E_STREAM;
}

int container_check_blob(const ContainerHeader& h, uint32_t blob_crc)
{
    return (h.flags & RB200_CONTAINER_CRC_BLOB) && blob_crc != h.blob_crc ? RB200_E_STREAM : RB200_OK;
}

namespace {

// Every pack: header (CRCs filled in), model, directory, zero pad and blob into out[0, container_blob_offset(h) + blob).
void container_write(ContainerHeader h, const void* model, const uint64_t* offsets, const uint8_t* blob, uint8_t* out)
{
    h.meta_crc = container_meta_crc(h, model, offsets);
    if (h.flags & RB200_CONTAINER_CRC_BLOB) h.blob_crc = container_crc32(0, blob, h.blob_bytes);
    const ContainerHeader l = container_layout(h);
    const uint64_t dir = container_dir_offset(l), dir_end = container_dir_end(l), boff = container_blob_offset(l);
    std::memcpy(out, &h, sizeof h);
    std::memcpy(out + sizeof h, model, container_model_bytes(l));
    std::memcpy(out + dir, offsets, dir_end - dir);
    std::memset(out + dir_end, 0, boff - dir_end);
    if (h.blob_bytes) std::memcpy(out + boff, blob, h.blob_bytes);
}

// Every open: the parser's three steps on a host buffer (8-byte aligned) holding a container of `version`.
int container_open_checked(const uint8_t* buf, size_t size, uint16_t version, ContainerHeader* h)
{
    int rc = container_parse_header(buf, size, version, h);
    if (rc != RB200_OK) return rc;
    // model and offsets sit at 4- and 8-byte aligned positions when buf itself is 8-byte aligned (callers map or malloc it)
    if (reinterpret_cast<uintptr_t>(buf) & 7) return RB200_E_ARG;
    const ContainerHeader l = container_layout(*h);
    rc = container_check_prefix(*h, buf, container_meta_crc(*h, buf + sizeof(ContainerHeader),
                                                            reinterpret_cast<const uint64_t*>(buf + container_dir_offset(l))));
    if (rc == RB200_OK && (h->flags & RB200_CONTAINER_CRC_BLOB))
        rc = container_check_blob(*h, container_crc32(0, buf + container_blob_offset(l), h->blob_bytes));
    return rc;
}

// The pack of every per-block version, for the header h (crc fields zero) the caller built from a geometry it checked:
// the other argument rules, every block summing to 1 << h.scale_bits, then the bytes.
int container_blocks_pack(const ContainerHeader& h, const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob,
                          uint8_t* out, size_t out_cap, size_t* out_size)
{
    if (!block_freqs || !offsets || (!blob && h.blob_bytes) || !out || h.n_chunks >= (1ull << 31)) return RB200_E_ARG;
    if (!container_block_models_sum_to(block_freqs, h.n_blocks, 1u << h.scale_bits)) return RB200_E_MODEL;   // never write what open rejects
    if ((h.blob_bytes & 15) || !container_directory_ok(offsets, h.n_chunks, h.blob_bytes)) return RB200_E_ARG;
    const size_t total = container_blob_offset(container_layout(h)) + h.blob_bytes;
    if (total > out_cap) return RB200_E_SPACE;
    container_write(h, block_freqs, offsets, blob, out);
    if (out_size) *out_size = total;
    return RB200_OK;
}

// The open of every per-block version: the parser's steps for `version`, then the fields their info structs share.
template <class Info>
int container_blocks_open(const uint8_t* buf, size_t size, uint16_t version, Info* info, ContainerHeader* h)
{
    if (!buf || !info) return RB200_E_ARG;
    const int rc = container_open_checked(buf, size, version, h);
    if (rc != RB200_OK) return rc;
    info->n_blocks = h->n_blocks;
    info->block_size = h->block_size;
    info->chunk_syms = h->chunk_syms;
    info->flags = h->flags;
    info->n_symbols = h->n_symbols;
    info->n_chunks = h->n_chunks;
    info->blob_bytes = h->blob_bytes;
    info->block_freqs = reinterpret_cast<const uint16_t*>(buf + sizeof(ContainerHeader));
    info->offsets = reinterpret_cast<const uint64_t*>(buf + container_dir_offset(container_layout(*h)));
    info->blob = buf + container_blob_offset(container_layout(*h));
    return RB200_OK;
}

// The pack of versions 3 and 4: the version's coder rule, the geometry, then the shared pack
int container_blocks_coder_pack(uint16_t version, int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes, uint32_t flags,
                                uint8_t* out, size_t out_cap, size_t* out_size)
{
    if (coder < 0 || !container_blocks_coder_ok(version, static_cast<uint32_t>(coder), scale_bits)) return RB200_E_ARG;
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    return container_blocks_pack(container_blocks_coder_header(version, coder, scale_bits, n_blocks, block_size, chunk_syms, blob_bytes, flags),
                                 block_freqs, offsets, blob, out, out_cap, out_size);
}

// The open of versions 3 and 4, which also report the header's coder and scale_bits
int container_blocks_coder_open(const uint8_t* buf, size_t size, uint16_t version, rb200_container_blocks_coder_info* info)
{
    ContainerHeader h;
    const int rc = container_blocks_open(buf, size, version, info, &h);
    if (rc != RB200_OK) return rc;
    info->coder = h.coder;
    info->scale_bits = h.scale_bits;
    return RB200_OK;
}

}  // namespace

}  // namespace rb200

using namespace rb200;

extern "C" size_t rb200_container_size(size_t n_chunks, size_t blob_bytes)
{
    return container_blob_offset(container_shape(kContainerVersion, 0, n_chunks)) + blob_bytes;
}

extern "C" int rb200_container_pack(int coder, uint32_t scale_bits, uint32_t chunk_syms, size_t n, const uint32_t freqs[256],
                                    const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes, uint32_t flags, uint8_t* out,
                                    size_t out_cap, size_t* out_size)
{
    if (!freqs || !offsets || (!blob && blob_bytes) || !out || !chunk_syms) return RB200_E_ARG;
    if (coder < 0 || !container_model_ok(static_cast<uint32_t>(coder), scale_bits, freqs)) return RB200_E_MODEL;   // never write what open rejects
    const size_t n_chunks = rb200_chunk_count(n, chunk_syms);
    if (offsets[n_chunks] != blob_bytes || (blob_bytes & 15)) return RB200_E_ARG;
    const size_t total = rb200_container_size(n_chunks, blob_bytes);
    if (total > out_cap) return RB200_E_SPACE;
    container_write(container_header(coder, scale_bits, chunk_syms, n, n_chunks, blob_bytes, flags), freqs, offsets, blob, out);
    if (out_size) *out_size = total;
    return RB200_OK;
}

extern "C" int rb200_container_open(const uint8_t* buf, size_t size, rb200_container_info* info)
{
    if (!buf || !info) return RB200_E_ARG;
    ContainerHeader h;
    const int rc = container_open_checked(buf, size, kContainerVersion, &h);
    if (rc != RB200_OK) return rc;
    info->coder = h.coder;
    info->scale_bits = h.scale_bits;
    info->chunk_syms = h.chunk_syms;
    info->flags = h.flags;
    info->n_symbols = h.n_symbols;
    info->n_chunks = h.n_chunks;
    info->blob_bytes = h.blob_bytes;
    info->freqs = reinterpret_cast<const uint32_t*>(buf + sizeof(ContainerHeader));
    info->offsets = reinterpret_cast<const uint64_t*>(buf + container_dir_offset(h));
    info->blob = buf + container_blob_offset(h);
    return RB200_OK;
}

extern "C" size_t rb200_container_blocks_size(uint32_t n_blocks, size_t n_chunks, size_t blob_bytes)
{
    return container_blob_offset(container_shape(kContainerVersionBlocks, n_blocks, n_chunks)) + blob_bytes;
}

extern "C" int rb200_container_blocks_pack(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, const uint16_t* block_freqs,
                                           const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes, uint32_t flags, uint8_t* out,
                                           size_t out_cap, size_t* out_size)
{
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    return container_blocks_pack(container_blocks_header(n_blocks, block_size, chunk_syms, blob_bytes, flags), block_freqs, offsets, blob,
                                 out, out_cap, out_size);
}

extern "C" int rb200_container_blocks_open(const uint8_t* buf, size_t size, rb200_container_blocks_info* info)
{
    ContainerHeader h;
    return container_blocks_open(buf, size, kContainerVersionBlocks, info, &h);
}

extern "C" int rb200_container_blocks_coder_pack(int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                                 const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob,
                                                 size_t blob_bytes, uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size)
{
    return container_blocks_coder_pack(kContainerVersionBlocksCoder, coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs, offsets,
                                       blob, blob_bytes, flags, out, out_cap, out_size);
}

extern "C" int rb200_container_blocks_coder_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info)
{
    return container_blocks_coder_open(buf, size, kContainerVersionBlocksCoder, info);
}

extern "C" int rb200_container_blocks_alias_pack(uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                                 const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob,
                                                 size_t blob_bytes, uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size)
{
    return container_blocks_coder_pack(kContainerVersionBlocksAlias, RB200_CODER_ALIAS, scale_bits, n_blocks, block_size, chunk_syms,
                                       block_freqs, offsets, blob, blob_bytes, flags, out, out_cap, out_size);
}

extern "C" int rb200_container_blocks_alias_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info)
{
    return container_blocks_coder_open(buf, size, kContainerVersionBlocksAlias, info);
}

extern "C" size_t rb200_container_blocks_stored_bound(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms)
{
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return 0;
    const uint64_t n_chunks = static_cast<uint64_t>(n_blocks) * (block_size / chunk_syms);
    return container_blob_offset(container_shape(kContainerVersionBlocks, n_blocks, n_chunks)) + n_chunks * container_stored_bytes(chunk_syms);
}

extern "C" int rb200_container_blocks_stored_pack(int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                                  const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob,
                                                  size_t blob_bytes, uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size)
{
    if (coder < 0 || !blocks_candidate_ok(RB200_CANDIDATE(coder, scale_bits))) return RB200_E_ARG;
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    if (!block_freqs || !offsets || (!blob && blob_bytes) || !out) return RB200_E_ARG;
    ContainerHeader h = container_blocks_coder_header(container_blocks_version(static_cast<uint32_t>(coder)), coder, scale_bits, n_blocks,
                                                      block_size, chunk_syms, blob_bytes, flags);
    h.version = kContainerVersionBlocksStored;
    if (h.n_chunks >= (1ull << 31)) return RB200_E_ARG;
    for (uint64_t b = 0; b < n_blocks; b++)                          // never write what open rejects
        if (!container_block_model_stored(block_freqs + b * 256) && !container_block_model_sums_to(block_freqs + b * 256, 1u << scale_bits))
            return RB200_E_MODEL;
    if ((blob_bytes & 15) || !container_directory_ok(offsets, h.n_chunks, blob_bytes) || !container_stored_rows_ok(h, block_freqs, offsets, blob))
        return RB200_E_ARG;
    const size_t total = container_blob_offset(container_layout(h)) + blob_bytes;
    if (total > out_cap) return RB200_E_SPACE;
    container_write(h, block_freqs, offsets, blob, out);
    if (out_size) *out_size = total;
    return RB200_OK;
}

extern "C" int rb200_container_blocks_stored_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info)
{
    return container_blocks_coder_open(buf, size, kContainerVersionBlocksStored, info);
}

namespace {

// Version 6's prefix rules past the header, on a host buffer holding the whole container: meta_crc over [0, blob
// offset), the model, the directory's ends, every chunk (container_v6_chunk_ok) and every bitmap word.
int container_v6_check(const ContainerHeader& h, const uint8_t* buf)
{
    const uint64_t boff = container_bitmap_blob_offset(h.n_chunks);
    const uint32_t meta = container_crc32(container_header_crc(h), buf + sizeof(ContainerHeader), boff - sizeof(ContainerHeader));
    if (meta != h.meta_crc) return RB200_E_STREAM;
    if (!container_model_ok(h.coder, h.scale_bits, reinterpret_cast<const uint32_t*>(buf + sizeof(ContainerHeader)))) return RB200_E_STREAM;
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + kContainerDirOffset);
    const uint32_t* bits = reinterpret_cast<const uint32_t*>(buf + container_bitmap_offset(h.n_chunks));
    if (!container_dir_ends_ok(offsets, h.n_chunks, h.blob_bytes)) return RB200_E_STREAM;
    for (uint64_t w = 0; w < container_bitmap_words(h.n_chunks); w++)
        if (!container_bitmap_word_ok(bits, w, h.n_chunks)) return RB200_E_STREAM;
    for (uint64_t c = 0; c < h.n_chunks; c++)
        if (!container_v6_chunk_ok(offsets, bits, buf + boff, c, h.chunk_syms, h.n_symbols, h.blob_bytes)) return RB200_E_STREAM;
    return RB200_OK;
}

}  // namespace

extern "C" size_t rb200_container_stored_bound(size_t n, uint32_t chunk_syms)
{
    if (n == 0 || (n >> 32) || !container_chunk_ok(chunk_syms)) return 0;
    const uint64_t n_chunks = rb200_chunk_count(n, chunk_syms), tail = n % chunk_syms;
    return container_bitmap_blob_offset(n_chunks) + (n / chunk_syms) * container_stored_bytes(chunk_syms) +
           (tail ? container_stored_bytes(static_cast<uint32_t>(tail)) : 0);
}

extern "C" int rb200_container_stored_pack(int coder, uint32_t scale_bits, uint32_t chunk_syms, size_t n, const uint32_t freqs[256],
                                           const uint32_t* stored_bits, const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes,
                                           uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size)
{
    if (coder < 0 || !candidate_ok(RB200_CANDIDATE(coder, scale_bits)) || !rb200_container_stored_bound(n, chunk_syms)) return RB200_E_ARG;
    if (!freqs || !stored_bits || !offsets || (!blob && blob_bytes) || !out) return RB200_E_ARG;
    if (!container_model_ok(static_cast<uint32_t>(coder), scale_bits, freqs)) return RB200_E_MODEL;   // never write what open rejects
    const uint64_t n_chunks = rb200_chunk_count(n, chunk_syms);
    const uint64_t words = (n_chunks + 31) / 32;
    if (!container_bitmap_word_ok(stored_bits, words - 1, n_chunks) || (blob_bytes & 15) ||
        !container_dir_ends_ok(offsets, n_chunks, blob_bytes))
        return RB200_E_ARG;
    std::vector<uint32_t> bits(container_bitmap_words(n_chunks), 0u);
    std::memcpy(bits.data(), stored_bits, words * sizeof(uint32_t));
    for (uint64_t c = 0; c < n_chunks; c++)
        if (!container_v6_chunk_ok(offsets, bits.data(), blob, c, chunk_syms, n, blob_bytes)) return RB200_E_ARG;
    const uint64_t boff = container_bitmap_blob_offset(n_chunks), bitmap = container_bitmap_offset(n_chunks);
    const size_t total = boff + blob_bytes;
    if (total > out_cap) return RB200_E_SPACE;
    ContainerHeader h = container_header(coder, scale_bits, chunk_syms, n, n_chunks, blob_bytes, flags);
    h.version = kContainerVersionStored;
    std::memset(out, 0, boff);
    std::memcpy(out + sizeof h, freqs, 256 * sizeof(uint32_t));
    std::memcpy(out + kContainerDirOffset, offsets, (n_chunks + 1) * sizeof(uint64_t));
    std::memcpy(out + bitmap, bits.data(), bits.size() * sizeof(uint32_t));
    h.meta_crc = container_crc32(container_header_crc(h), out + sizeof h, boff - sizeof h);
    if (h.flags & RB200_CONTAINER_CRC_BLOB) h.blob_crc = container_crc32(0, blob, blob_bytes);
    std::memcpy(out, &h, sizeof h);
    if (blob_bytes) std::memcpy(out + boff, blob, blob_bytes);
    if (out_size) *out_size = total;
    return RB200_OK;
}

extern "C" int rb200_container_stored_open(const uint8_t* buf, size_t size, rb200_container_info* info, const uint32_t** stored_bits)
{
    if (!buf || !info || !stored_bits) return RB200_E_ARG;
    if (size < sizeof(ContainerHeader)) return RB200_E_STREAM;
    ContainerHeader h;
    std::memcpy(&h, buf, sizeof h);
    if (!container_chunks_stored_header_ok(h, size)) return RB200_E_STREAM;
    if (reinterpret_cast<uintptr_t>(buf) & 7) return RB200_E_ARG;
    int rc = container_v6_check(h, buf);
    if (rc == RB200_OK && (h.flags & RB200_CONTAINER_CRC_BLOB))
        rc = container_check_blob(h, container_crc32(0, buf + container_bitmap_blob_offset(h.n_chunks), h.blob_bytes));
    if (rc != RB200_OK) return rc;
    info->coder = h.coder;
    info->scale_bits = h.scale_bits;
    info->chunk_syms = h.chunk_syms;
    info->flags = h.flags;
    info->n_symbols = h.n_symbols;
    info->n_chunks = h.n_chunks;
    info->blob_bytes = h.blob_bytes;
    info->freqs = reinterpret_cast<const uint32_t*>(buf + sizeof(ContainerHeader));
    info->offsets = reinterpret_cast<const uint64_t*>(buf + kContainerDirOffset);
    info->blob = buf + container_bitmap_blob_offset(h.n_chunks);
    *stored_bits = reinterpret_cast<const uint32_t*>(buf + container_bitmap_offset(h.n_chunks));
    return RB200_OK;
}

extern "C" size_t rb200_container_planes_bound(size_t n, uint32_t elem_bytes, uint32_t chunk_syms)
{
    if (!container_planes_w_ok(elem_bytes) || n % elem_bytes) return 0;
    const size_t plane = rb200_container_stored_bound(n / elem_bytes, chunk_syms);
    return plane ? container_planes_table_end(elem_bytes, 0) + elem_bytes * plane : 0;
}

extern "C" size_t rb200_container_tensors_bound(size_t n_max, uint32_t count, uint32_t elem_bytes, uint32_t chunk_syms)
{
    if (!count || count > kContainerTensorsMax) return 0;
    const size_t b = rb200_container_planes_bound(n_max, elem_bytes, chunk_syms);
    return b ? b + container_tensors_dir_bytes(count) : 0;
}

namespace {

// a version 6 container that rb200_container_stored_open accepts, exactly `size` bytes long: its header in *h
int planes_plane_open(const uint8_t* plane, size_t size, ContainerHeader* h)
{
    rb200_container_info info;
    const uint32_t* bits = nullptr;
    const int rc = rb200_container_stored_open(plane, size, &info, &bits);
    if (rc != RB200_OK) return rc;
    std::memcpy(h, plane, sizeof *h);
    return container_bitmap_blob_offset(h->n_chunks) + h->blob_bytes == size ? RB200_OK : RB200_E_STREAM;
}

// the pack of version 7 (reserved 0), version 8 (reserved the base tensor's CRC) or version 9 (`lengths`: the
// directory of `count` tensors; reserved its CRC)
int planes_pack(uint16_t version, uint32_t reserved, uint32_t elem_bytes, const uint64_t* lengths, uint32_t count, const uint8_t* const* planes,
                const size_t* sizes, uint8_t* out, size_t out_cap, size_t* out_size)
{
    if (!container_planes_w_ok(elem_bytes) || !planes || !sizes || !out) return RB200_E_ARG;
    const bool list = version == kContainerVersionTensors;
    if (list && (!lengths || !count || count > kContainerTensorsMax)) return RB200_E_ARG;
    const uint64_t dir_bytes = list ? container_tensors_dir_bytes(count) : 0;
    ContainerHeader first{};
    PlaneEntry table[8];
    uint64_t end = container_planes_table_end(elem_bytes, dir_bytes);
    for (uint32_t p = 0; p < elem_bytes; p++) {
        ContainerHeader ph;
        if (!planes[p] || planes_plane_open(planes[p], sizes[p], &ph) != RB200_OK) return RB200_E_ARG;
        if (p == 0) first = ph;
        else if (ph.n_symbols != first.n_symbols || ph.chunk_syms != first.chunk_syms || ph.flags != first.flags) return RB200_E_ARG;
        table[p] = PlaneEntry{end, sizes[p]};
        end += sizes[p];
    }
    if (!container_chunk_ok(first.chunk_syms)) return RB200_E_ARG;          // the v7 rules take the encodes' chunk sizes
    const uint64_t n = first.n_symbols * elem_bytes;
    std::vector<uint64_t> dir(dir_bytes / sizeof(uint64_t), 0);
    if (list) {
        std::memcpy(dir.data(), lengths, sizeof(uint64_t) * count);
        uint64_t sum = 0;
        if (!container_tensors_dir_part_ok(dir.data(), 0, count, elem_bytes, n, &sum) || sum != n) return RB200_E_ARG;
        reserved = container_crc32(0, dir.data(), sizeof(uint64_t) * count);
    }
    if (end > out_cap) return RB200_E_SPACE;
    ContainerHeader h{};
    h.magic = kContainerMagic;
    h.version = version;
    h.lanes = RB200_LANES;
    h.chunk_syms = first.chunk_syms;
    h.n_symbols = n;
    h.blob_bytes = end - container_planes_table_end(elem_bytes, dir_bytes);
    h.flags = first.flags;
    h.block_size = elem_bytes;
    h.n_blocks = list ? count : elem_bytes;
    h.reserved = reserved;
    h.meta_crc = container_crc32(container_header_crc(h), table, sizeof(PlaneEntry) * elem_bytes);
    std::memcpy(out, &h, sizeof h);
    std::memcpy(out + sizeof h, table, sizeof(PlaneEntry) * elem_bytes);
    if (dir_bytes) std::memcpy(out + container_planes_table_end(elem_bytes, 0), dir.data(), dir_bytes);
    for (uint32_t p = 0; p < elem_bytes; p++) std::memcpy(out + table[p].offset, planes[p], sizes[p]);
    if (out_size) *out_size = end;
    return RB200_OK;
}

// the open of version 7, 8 or 9 (`version`, the one the caller accepts); *reserved receives the header's reserved word,
// and for version 9 *count and *lengths the directory, once its CRC (reserved) and rules pass
int planes_open(uint16_t version, const uint8_t* buf, size_t size, rb200_container_planes_info* info, uint32_t* reserved,
                uint32_t* count = nullptr, const uint64_t** lengths = nullptr)
{
    if (!buf || !info) return RB200_E_ARG;
    if (size < sizeof(ContainerHeader)) return RB200_E_STREAM;
    ContainerHeader h;
    std::memcpy(&h, buf, sizeof h);
    if (!container_planes_header_version_ok(h, size, version)) return RB200_E_STREAM;
    if (reinterpret_cast<uintptr_t>(buf) & 7) return RB200_E_ARG;
    const uint32_t w = h.block_size;
    const uint64_t dir_bytes = container_planes_dir_bytes(h, version);
    PlaneEntry table[8];
    std::memcpy(table, buf + sizeof h, sizeof(PlaneEntry) * w);
    if (container_crc32(container_header_crc(h), table, sizeof(PlaneEntry) * w) != h.meta_crc || !container_planes_table_ok(h, table, dir_bytes))
        return RB200_E_STREAM;
    if (version == kContainerVersionTensors) {                        // the directory lies in size (header rule)
        const uint64_t* dir = reinterpret_cast<const uint64_t*>(buf + container_planes_table_end(w, 0));
        uint64_t sum = 0;
        if (container_crc32(0, dir, sizeof(uint64_t) * h.n_blocks) != h.reserved ||
            !container_tensors_dir_part_ok(dir, 0, h.n_blocks, w, h.n_symbols, &sum) || sum != h.n_symbols ||
            !container_tensors_dir_pad_ok(dir, h.n_blocks))
            return RB200_E_STREAM;
        *count = h.n_blocks;
        *lengths = dir;
    }
    for (uint32_t p = 0; p < w; p++) {
        ContainerHeader ph;
        std::memcpy(&ph, buf + table[p].offset, sizeof ph);
        if (!container_planes_plane_ok(h, ph, table[p].size) || planes_plane_open(buf + table[p].offset, table[p].size, &ph) != RB200_OK)
            return RB200_E_STREAM;
    }
    std::memset(info, 0, sizeof *info);
    info->elem_bytes = w;
    info->chunk_syms = h.chunk_syms;
    info->flags = h.flags;
    info->n = h.n_symbols;
    for (uint32_t p = 0; p < w; p++) {
        info->planes[p] = buf + table[p].offset;
        info->sizes[p] = table[p].size;
    }
    *reserved = h.reserved;
    return RB200_OK;
}

}  // namespace

extern "C" int rb200_container_planes_pack(uint32_t elem_bytes, const uint8_t* const* planes, const size_t* sizes, uint8_t* out,
                                           size_t out_cap, size_t* out_size)
{
    return planes_pack(kContainerVersionPlanes, 0, elem_bytes, nullptr, 0, planes, sizes, out, out_cap, out_size);
}

extern "C" int rb200_container_planes_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info)
{
    uint32_t reserved;
    return planes_open(kContainerVersionPlanes, buf, size, info, &reserved);
}

extern "C" int rb200_container_delta_pack(uint32_t elem_bytes, const uint8_t* const* planes, const size_t* sizes, uint32_t base_crc,
                                          uint8_t* out, size_t out_cap, size_t* out_size)
{
    return planes_pack(kContainerVersionDelta, base_crc, elem_bytes, nullptr, 0, planes, sizes, out, out_cap, out_size);
}

extern "C" int rb200_container_delta_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info, uint32_t* base_crc)
{
    if (!base_crc) return RB200_E_ARG;
    return planes_open(kContainerVersionDelta, buf, size, info, base_crc);
}

extern "C" int rb200_container_tensors_pack(uint32_t elem_bytes, const uint64_t* lengths, uint32_t count, const uint8_t* const* planes,
                                            const size_t* sizes, uint8_t* out, size_t out_cap, size_t* out_size)
{
    return planes_pack(kContainerVersionTensors, 0, elem_bytes, lengths, count, planes, sizes, out, out_cap, out_size);
}

extern "C" int rb200_container_tensors_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info, uint32_t* count,
                                            const uint64_t** lengths)
{
    if (!count || !lengths) return RB200_E_ARG;
    uint32_t reserved;
    return planes_open(kContainerVersionTensors, buf, size, info, &reserved, count, lengths);
}

extern "C" int rb200_choose_coder(const uint64_t counts[256], size_t n, uint32_t chunk_syms, const uint32_t* candidates,
                                  uint32_t n_candidates, uint32_t tolerance_ppm, uint64_t* costs, uint32_t* chosen)
{
    if (!counts || !chosen || !candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!container_chunk_ok(chunk_syms) || (n >> 32)) return RB200_E_ARG;
    uint64_t total = 0;
    for (int s = 0; s < 256; s++) total += counts[s];                 // each count <= n < 2^32: no overflow
    if (total != n) return RB200_E_ARG;
    const uint64_t n_chunks = n / chunk_syms + (n % chunk_syms != 0);
    uint64_t cost[16];
    for (uint32_t i = 0; i < n_candidates; i++) {
        const uint32_t coder = candidates[i] >> 8, sb = candidates[i] & 0xffu;
        uint32_t f[256], cum[257];
        for (int s = 0; s < 256; s++) f[s] = static_cast<uint32_t>(counts[s]);
        cost[i] = ~0ull;
        if (n == 0 || rb200_normalize_freqs(f, cum, 1u << sb) != RB200_OK) continue;
        if (!container_model_ok(coder, sb, f) || !container_model_decodable(coder, f)) continue;
        uint64_t bits_q = 0;
        for (int s = 0; s < 256; s++) bits_q += candidate_bits_q(static_cast<uint32_t>(counts[s]), f[s], sb);
        cost[i] = candidate_cost(bits_q, n_chunks, coder);
    }
    if (costs) std::memcpy(costs, cost, n_candidates * sizeof(uint64_t));
    const int k = choose_candidate(cost, n_candidates, tolerance_ppm);
    if (k < 0) return RB200_E_MODEL;
    *chosen = static_cast<uint32_t>(k);
    return RB200_OK;
}

extern "C" int rb200_choose_blocks_coder(const uint32_t* block_counts, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                         const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm, uint64_t* costs,
                                         uint32_t* chosen)
{
    if (!block_counts || !chosen || !blocks_candidate_list_ok(candidates, n_candidates) || tolerance_ppm > 1000000u) return RB200_E_ARG;
    if (!container_blocks_geometry_ok(n_blocks, block_size, chunk_syms)) return RB200_E_ARG;
    for (uint32_t b = 0; b < n_blocks; b++) {
        uint64_t total = 0;
        for (int s = 0; s < 256; s++) total += block_counts[static_cast<size_t>(b) * 256 + s];
        if (total != block_size) return RB200_E_ARG;
    }
    uint64_t cost[16] = {};
    for (uint32_t b = 0; b < n_blocks; b++) {
        const uint32_t* counts = block_counts + static_cast<size_t>(b) * 256;
        for (uint32_t i = 0; i < n_candidates; i++) {
            const uint32_t coder = candidates[i] >> 8, sb = candidates[i] & 0xffu;
            uint32_t f[256], cum[257];
            std::memcpy(f, counts, sizeof f);
            if (rb200_normalize_freqs(f, cum, 1u << sb) != RB200_OK) return RB200_E_MODEL;   // not reached: targets >= 256
            uint64_t bits_q = 0;
            bool one_symbol = false;
            for (int s = 0; s < 256; s++) {
                bits_q += candidate_bits_q(counts[s], f[s], sb);
                one_symbol |= f[s] == (1u << sb);
            }
            cost[i] += blocks_candidate_cost(bits_q, block_size, chunk_syms, coder, one_symbol);
        }
    }
    if (costs) std::memcpy(costs, cost, n_candidates * sizeof(uint64_t));
    *chosen = static_cast<uint32_t>(choose_candidate(cost, n_candidates, tolerance_ppm));   // every cost is finite
    return RB200_OK;
}

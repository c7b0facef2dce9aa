// container_host.cpp -- self-describing wire format around (model, directory, blob)  [SURVEY 8f.3].
//
// The reference defines no container: its drivers keep a pointer and the sizes in local variables
// (main.cpp:182-188).  The bulk API's natural output (blob + offsets + the caller's freqs) is enough
// for in-process use; this file adds the versioned, checksummed envelope needed to ship it:
//
//   [ 64-byte header ][ freqs: 256 x u32 ][ offsets: (n_chunks + 1) x u64 ][ pad to 16 ][ blob ]
//
// All integers little-endian.  CRC-32 (zlib's: IEEE, reflected) over header (with the crc fields zeroed) + freqs +
// offsets always; over the blob when RB200_CONTAINER_CRC_BLOB is set.  rb200_container_pack / _open here work on host
// buffers with a host CRC (slicing-by-8, ~1 GB/s on one core: the blob CRC is optional for that reason).
// rb200_container_encode / _decode (rans_b200.cu) write and read the same bytes in host or device memory with the
// blob CRC on the GPU (crc_kernels.cuh); they validate through the parser below, so both sides apply one set of rules.
#include "container_format.h"

#include <cstring>

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

uint32_t container_meta_crc(const ContainerHeader& h, const uint32_t* freqs, const uint64_t* offsets)
{
    uint32_t c = container_header_crc(h);
    c = container_crc32(c, freqs, 256 * sizeof(uint32_t));
    return container_crc32(c, offsets, (h.n_chunks + 1) * sizeof(uint64_t));
}

bool container_model_ok(uint32_t coder, uint32_t scale_bits, const uint32_t* freqs)
{
    if (coder > RB200_CODER_RANS64 || scale_bits < 8 || scale_bits > 16) return false;
    if (coder == RB200_CODER_WORD && scale_bits != 12) return false;
    uint64_t sum = 0;
    for (int s = 0; s < 256; s++) sum += freqs[s];
    return sum == (1ull << scale_bits);
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

int container_parse_header(const uint8_t* hdr, size_t size, ContainerHeader* out)
{
    if (size < sizeof(ContainerHeader)) return RB200_E_STREAM;
    ContainerHeader h;
    std::memcpy(&h, hdr, sizeof h);
    if (h.magic != kContainerMagic || h.version != kContainerVersion || h.lanes != RB200_LANES || !h.chunk_syms) return RB200_E_STREAM;
    if (h.n_chunks != h.n_symbols / h.chunk_syms + (h.n_symbols % h.chunk_syms != 0) || h.n_chunks >= (1ull << 31) ||
        (h.blob_bytes & 15) || h.coder > RB200_CODER_RANS64 || h.scale_bits < 8 || h.scale_bits > 16)
        return RB200_E_STREAM;
    const size_t boff = container_blob_offset(h.n_chunks);
    if (boff > size || h.blob_bytes > size - boff) return RB200_E_STREAM;
    *out = h;
    return RB200_OK;
}

int container_check_prefix(const ContainerHeader& h, const uint8_t* prefix, uint32_t meta_crc)
{
    const uint32_t* freqs = reinterpret_cast<const uint32_t*>(prefix + sizeof(ContainerHeader));
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(prefix + kContainerDirOffset);
    if (meta_crc != h.meta_crc) return RB200_E_STREAM;
    if (!container_model_ok(h.coder, h.scale_bits, freqs)) return RB200_E_STREAM;        // CRC-valid but inconsistent
    if (offsets[h.n_chunks] != h.blob_bytes) return RB200_E_STREAM;
    if (h.n_chunks && offsets[0] >= 16) return RB200_E_STREAM;                           // the first stream starts inside the first vector
    for (uint64_t c = 0; c < h.n_chunks; c++)
        if (offsets[c] > offsets[c + 1]) return RB200_E_STREAM;
    return RB200_OK;
}

int container_check_blob(const ContainerHeader& h, uint32_t blob_crc)
{
    return (h.flags & RB200_CONTAINER_CRC_BLOB) && blob_crc != h.blob_crc ? RB200_E_STREAM : RB200_OK;
}

}  // namespace rb200

using namespace rb200;

extern "C" size_t rb200_container_size(size_t n_chunks, size_t blob_bytes) { return container_blob_offset(n_chunks) + blob_bytes; }

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
    ContainerHeader h = container_header(coder, scale_bits, chunk_syms, n, n_chunks, blob_bytes, flags);
    h.meta_crc = container_meta_crc(h, freqs, offsets);
    if (h.flags & RB200_CONTAINER_CRC_BLOB) h.blob_crc = container_crc32(0, blob, blob_bytes);
    uint8_t* p = out;
    std::memcpy(p, &h, sizeof h);
    p += sizeof h;
    std::memcpy(p, freqs, 256 * sizeof(uint32_t));
    p += 256 * sizeof(uint32_t);
    std::memcpy(p, offsets, (n_chunks + 1) * sizeof(uint64_t));
    p += (n_chunks + 1) * sizeof(uint64_t);
    const size_t boff = container_blob_offset(n_chunks);
    std::memset(p, 0, out + boff - p);
    if (blob_bytes) std::memcpy(out + boff, blob, blob_bytes);
    if (out_size) *out_size = total;
    return RB200_OK;
}

extern "C" int rb200_container_open(const uint8_t* buf, size_t size, rb200_container_info* info)
{
    if (!buf || !info) return RB200_E_ARG;
    ContainerHeader h;
    int rc = container_parse_header(buf, size, &h);
    if (rc != RB200_OK) return rc;
    // freqs/offsets sit at 4- and 8-byte aligned positions when buf itself is 8-byte aligned (callers map or malloc it)
    const uint32_t* freqs = reinterpret_cast<const uint32_t*>(buf + sizeof(ContainerHeader));
    const uint64_t* offsets = reinterpret_cast<const uint64_t*>(buf + kContainerDirOffset);
    if (reinterpret_cast<uintptr_t>(buf) & 7) return RB200_E_ARG;
    rc = container_check_prefix(h, buf, container_meta_crc(h, freqs, offsets));
    if (rc != RB200_OK) return rc;
    const size_t boff = container_blob_offset(h.n_chunks);
    if (h.flags & RB200_CONTAINER_CRC_BLOB) rc = container_check_blob(h, container_crc32(0, buf + boff, h.blob_bytes));
    if (rc != RB200_OK) return rc;
    info->coder = h.coder;
    info->scale_bits = h.scale_bits;
    info->chunk_syms = h.chunk_syms;
    info->flags = h.flags;
    info->n_symbols = h.n_symbols;
    info->n_chunks = h.n_chunks;
    info->blob_bytes = h.blob_bytes;
    info->freqs = freqs;
    info->offsets = offsets;
    info->blob = buf + boff;
    return RB200_OK;
}

// container_format.h -- the layout of the self-describing container (container_host.cpp has the format comment) and
// the one parser both rb200_container_open and rb200_container_decode go through.  Internal to the library.
#pragma once
#include <cstddef>
#include <cstdint>

#include "rans_b200.h"

namespace rb200 {

constexpr uint32_t kContainerMagic = 0x43324252u;   // "RB2C"
constexpr uint16_t kContainerVersion = 1;

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
    uint32_t meta_crc;          // header (crc fields zero) + freqs + offsets
    uint32_t blob_crc;          // valid when flags & RB200_CONTAINER_CRC_BLOB
    uint32_t reserved[3];
};
static_assert(sizeof(ContainerHeader) == 64, "container header must stay 64 bytes");

constexpr size_t kContainerDirOffset = sizeof(ContainerHeader) + 256 * sizeof(uint32_t);   // 1088, 16-aligned

inline size_t container_blob_offset(uint64_t n_chunks)
{
    return (kContainerDirOffset + (n_chunks + 1) * sizeof(uint64_t) + 15) & ~static_cast<size_t>(15);
}

// the header rb200_container_pack writes (crc fields zero)
ContainerHeader container_header(int coder, uint32_t scale_bits, uint32_t chunk_syms, uint64_t n, uint64_t n_chunks,
                                 uint64_t blob_bytes, uint32_t flags);
// what rb200_model_create would accept: a known coder, its scale_bits range, frequencies that sum to 1 << scale_bits
bool container_model_ok(uint32_t coder, uint32_t scale_bits, const uint32_t* freqs);
// zlib crc32 on the host (slicing-by-8)
uint32_t container_crc32(uint32_t crc, const void* data, size_t len);
// CRC-32 of the header with its crc fields zeroed: the first 64 bytes of what meta_crc covers
uint32_t container_header_crc(const ContainerHeader& h);
// meta_crc over header, freqs and offsets, on the host
uint32_t container_meta_crc(const ContainerHeader& h, const uint32_t* freqs, const uint64_t* offsets);

// The parser, in the order rb200_container_open applies it.  Each step returns RB200_OK or RB200_E_STREAM; the CRC
// values are the caller's, computed wherever the bytes live.
//  1. the 64-byte header against the buffer size (`size` bytes in all; `hdr` holds at least 64 of them)
int container_parse_header(const uint8_t* hdr, size_t size, ContainerHeader* h);
//  2. header + model + directory (`prefix`: container_blob_offset(h.n_chunks) bytes), given their CRC
int container_check_prefix(const ContainerHeader& h, const uint8_t* prefix, uint32_t meta_crc);
//  3. the blob, given its CRC (only consulted when the header carries one)
int container_check_blob(const ContainerHeader& h, uint32_t blob_crc);

}  // namespace rb200

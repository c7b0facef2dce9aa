/*
 * rans_b200.h -- bulk C-ABI of the GPU-native (H100, sm_90a) interleaved rANS coder.
 *
 * The reference (rygorous/ryg_rans) is header-only: its hot path is the per-symbol
 * step functions of rans_byte.h / rans64.h / rans_word_sse41.h inlined into the
 * driver loops of main.cpp / main64.cpp / main_simd.cpp / main_alias.cpp.  It has
 * no FFI.  This header is the boundary a replacement .so exports so that those
 * driver loops can be swapped for one bulk call each; every entry point names the
 * reference code it stands in for.  Plain C types only (no CUDA, no torch types):
 * the CUDA stream is passed as an opaque void* (a cudaStream_t).
 *
 * Container ("chunked N=32 streams", DESIGN.md section 3):
 *   the symbol buffer is cut into chunks of `chunk_syms` symbols.  Chunk c is one
 *   independent 32-way interleaved rANS stream laid out EXACTLY as the reference
 *   drivers lay out their N-way streams (main_simd.cpp:287-300 with 8 -> 32;
 *   main_alias.cpp:353-373 with 2 -> 32): 32 little-endian u32 final states, lane 0
 *   first, then the renormalisation units in decode order.  Stream c occupies
 *   blob[offsets[c] .. E_c) where E_c = offsets[c+1] & ~15 is 16-byte aligned
 *   (streams are END-aligned; the <16 bytes between E_c and offsets[c+1] are zero),
 *   and offsets[n_chunks] = blob size.  Any reference decoder primitive can decode
 *   one chunk stream given blob + offsets[c].
 */
#ifndef RANS_B200_H
#define RANS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB200_VERSION 2

/* status codes (the reference only has assert(); SURVEY section 5 asks for codes) */
#define RB200_OK          0
#define RB200_E_ARG      -1   /* bad argument (null, misaligned, size mismatch)         */
#define RB200_E_MODEL    -2   /* frequencies do not form a valid model                  */
#define RB200_E_SPACE    -3   /* output buffer too small                                */
#define RB200_E_STREAM   -4   /* corrupt / truncated stream detected while decoding     */
#define RB200_E_CUDA     -5   /* CUDA runtime error, see rb200_last_cuda_error          */
#define RB200_E_NOMEM    -6
#define RB200_E_SYMBOL   -7   /* encoder met a symbol whose model frequency is 0        */
#define RB200_E_NCCL     -8   /* NCCL missing or an NCCL call failed, see rb200_last_cuda_error */
#define RB200_E_STALL    -9   /* a bounded wait inside a kernel (8 s without progress) expired: a bug or a wedged
                                 device, never bad input -- the kernels give up instead of hanging the GPU            */
#define RB200_E_BASE    -10   /* a delta container's base is not the tensor it was encoded against (its CRC differs)  */

/* which memory the data pointers of a bulk call live in */
#define RB200_MEM_HOST    0   /* host pointers; the call copies H2D/D2H and is synchronous */
#define RB200_MEM_DEVICE  1   /* device pointers; the call only enqueues on the stream     */

/* coder families (one per reference header / driver) */
#define RB200_CODER_WORD    0 /* rans_word_sse41.h: 32-bit state, u16 renorm, scale_bits = 12          */
#define RB200_CODER_BYTE    1 /* rans_byte.h + cum2sym lookup as in main.cpp, scale_bits 8..16           */
#define RB200_CODER_ALIAS   2 /* rans_byte.h state machine + main_alias.cpp alias tables, scale_bits 8..16 */
#define RB200_CODER_RANS64  3 /* rans64.h: 64-bit state, u32 renorm, cum2sym lookup as in main64.cpp      */

#define RB200_LANES 32        /* interleave width of one chunk stream = one warp */

typedef struct rb200_ctx rb200_ctx;
typedef struct rb200_model rb200_model;

/* ---------------------------------------------------------------- host-side model */

/* SymbolStats::count_freqs, main.cpp:59-66 (host loop; the device version is
 * rb200_histogram). */
int rb200_count_freqs(const uint8_t* in, size_t n, uint32_t freqs[256]);

/* SymbolStats::calc_cum_freqs + normalize_freqs, main.cpp:68-129.  In: raw counts.
 * Out: freqs summing to target_total (a power of two >= 256) and cum_freqs[257].
 * Returns RB200_E_MODEL where the reference would assert. */
int rb200_normalize_freqs(uint32_t freqs[256], uint32_t cum_freqs[257], uint32_t target_total);

/* RansWordTablesInitSymbol for all 256 symbols, rans_word_sse41.h:64-72 /
 * main_simd.cpp:141-143.  slots[i] = freq | bias << 16 (RansWordSlot.u32). */
int rb200_word_tables_build(const uint32_t freqs[256], const uint32_t cum_freqs[257],
                            uint32_t slots[4096], uint8_t slot2sym[4096]);

/* SymbolStats::make_alias_table, main_alias.cpp:147-237.  alias_remap needs
 * cum_freqs[256] entries. */
int rb200_alias_tables_build(const uint32_t freqs[256], const uint32_t cum_freqs[257],
                             uint32_t divider[256], uint32_t slot_adjust[512],
                             uint32_t slot_freqs[512], uint8_t sym_id[512], uint32_t* alias_remap);

/* ---------------------------------------------------------------- context */

/* One context per (device, stream, calling thread).  stream = cudaStream_t or NULL. */
int rb200_ctx_create(rb200_ctx** out, int device, void* stream);
void rb200_ctx_destroy(rb200_ctx* ctx);
int rb200_ctx_set_stream(rb200_ctx* ctx, void* stream);
/* Wait for the stream, then report-and-clear what the kernels flagged
 * (RB200_OK, RB200_E_STREAM or RB200_E_SYMBOL). */
int rb200_sync(rb200_ctx* ctx);
const char* rb200_last_cuda_error(const rb200_ctx* ctx);
const char* rb200_strerror(int code);
int rb200_version(void);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t rb200_launch_count(const rb200_ctx* ctx);

/* ---------------------------------------------------------------- device model */

/* Upload the coding tables for one model.  freqs must already be normalised to
 * 1 << scale_bits (WORD: scale_bits must be 12, rans_word_sse41.h:37; BYTE / ALIAS / RANS64:
 * 8..16 -- main.cpp:136 and main64.cpp:136 use 14, main_alias.cpp:276 uses 16; BYTE needs every
 * freq < 65536 like the reference's 16-bit RansDecSymbol).  Replaces the table set-up at
 * main.cpp:145-162 / main64.cpp:145-164 / main_simd.cpp:141-143 / main_alias.cpp:279-282. */
int rb200_model_create(rb200_ctx* ctx, int coder, uint32_t scale_bits,
                       const uint32_t freqs[256], rb200_model** out);
void rb200_model_destroy(rb200_model* m);

/* ---------------------------------------------------------------- geometry */

size_t rb200_chunk_count(size_t n, uint32_t chunk_syms);
/* Worst-case blob size for n symbols: replaces the reference's guesses
 * (32 MB at main.cpp:150; n + n/8 + 128 at main_simd.cpp:145, not a true bound). */
size_t rb200_encode_bound(size_t n, uint32_t chunk_syms);

/* ---------------------------------------------------------------- the hot path */

/* Replaces the N-way encode loop + flush (main_simd.cpp:287-300 / main_alias.cpp:353-373).
 * in[n] symbols -> blob (<= blob_cap bytes) + offsets[n_chunks + 1].
 * HOST mode: synchronous; *blob_size receives offsets[n_chunks].
 * DEVICE mode: in/blob/offsets are device pointers (blob and offsets 16-byte aligned),
 * work is enqueued on the context stream, blob_size may be NULL (read offsets[n_chunks]). */
int rb200_encode(rb200_ctx* ctx, const rb200_model* model,
                 const uint8_t* in, size_t n, uint32_t chunk_syms,
                 uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind);

/* Replaces the N-way decode loop (main_simd.cpp:313-332 / main_alias.cpp:386-405).
 * blob/offsets as produced by rb200_encode (or by the reference primitives driven
 * with N = 32) -> out[n].  Reads are bounded by blob_size; a stream that does not
 * end where its chunk ends is reported as RB200_E_STREAM by rb200_sync (DEVICE
 * mode) or by the call itself (HOST mode). */
int rb200_decode(rb200_ctx* ctx, const rb200_model* model,
                 const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                 uint32_t chunk_syms, uint8_t* out, size_t n, int mem_kind);

/* Device SymbolStats::count_freqs (main.cpp:59-66) over a device or host buffer;
 * counts[256] is written to HOST memory, the call synchronises. */
int rb200_histogram(rb200_ctx* ctx, const uint8_t* in, size_t n, uint64_t counts[256], int mem_kind);

/* The whole model set-up of the drivers in one call, with the pass over the data on the GPU
 * (SURVEY 8f.1): stats.count_freqs (main.cpp:59-66; rb200_histogram's kernel), then
 * stats.normalize_freqs(1 << scale_bits) (main.cpp:75-129; 256 counters, on the host, the
 * reference's algorithm verbatim), then the table build of rb200_model_create.  Replaces
 * main_simd.cpp:131-143 / main.cpp:138-162 / main_alias.cpp:276-282.  freqs_out[256] (may be
 * NULL) receives the normalised frequencies -- the model a decoder needs.  n must be below
 * 2^32 like the reference's 32-bit histogram (RB200_E_ARG otherwise); an empty input or one
 * the reference would assert on is RB200_E_MODEL.  The call synchronises. */
int rb200_model_from_data(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* data, size_t n,
                          int mem_kind, uint32_t freqs_out[256], rb200_model** out);

/* ---------------------------------------------------------------- per-block models */

/* BASELINE config 5: n_blocks independent blocks of block_size symbols, each with
 * its own order-0 model at scale_bits 12 (word coder).  block_freqs is
 * [n_blocks][256] u16, normalised to 4096 per block (what RansWordTablesInitSymbol
 * would be fed, rans_word_sse41.h:64-72); the 4096-slot decode table of each block
 * is built in shared memory inside the kernel.  Each block is cut into chunks of
 * chunk_syms symbols (block_size % chunk_syms == 0, and at most 32 chunks per block: one CTA per
 * block, one warp per chunk -- RB200_E_ARG otherwise); chunk index = block *
 * (block_size / chunk_syms) + chunk-in-block; the container is the same as above. */
int rb200_blocks_build_models(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                              uint16_t* block_freqs, int mem_kind);
int rb200_blocks_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                        const uint16_t* block_freqs, uint32_t chunk_syms,
                        uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind);
int rb200_blocks_decode(rb200_ctx* ctx, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                        const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size,
                        uint32_t chunk_syms, uint8_t* out, int mem_kind);
/* rb200_blocks_build_models + rb200_blocks_encode in ONE launch: every block's model is built (count_freqs +
 * normalize_freqs(4096), main.cpp:59-129, bit-exact) by the CTA that then encodes the block, and returned in
 * block_freqs[n_blocks][256] -- what a decoder needs next to the blob.  A block has at most 32 chunks
 * (block_size / chunk_syms <= 32: one warp per chunk, one CTA per block); HOST mode pipelines slices of whole blocks
 * over three streams like rb200_encode. */
int rb200_blocks_model_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                              uint16_t* block_freqs, uint32_t chunk_syms,
                              uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind);

/* Per-block containers: the self-describing container (below) at version 2, holding every block's model.
 *
 *   [ 64-byte header ][ block_freqs: n_blocks x 256 x u16 ][ offsets: (n_chunks + 1) x u64 ][ pad to 16 ][ blob ]
 *
 * The header is version 1's with version = 2, the word coder, scale_bits 12, 32 lanes, block_size in the u32 at
 * byte 52, n_blocks in the u32 at byte 56 and a zero u32 at byte 60; meta_crc covers header, block_freqs and offsets.
 * The directory starts at 64 + 512 n_blocks.  rb200_container_blocks_open rejects with RB200_E_STREAM anything
 * rb200_blocks_decode would not take (geometry as above, n_blocks >= 1, n_symbols == n_blocks * block_size,
 * n_chunks == n_symbols / chunk_syms < 2^31), sections that do not fit `size`, a nonzero byte-60 word, an unknown
 * flag, a CRC mismatch, a block whose frequencies do not sum to 4096, and a directory that breaks version 1's rules.
 * rb200_container_open / _decode accept only version 1 and these calls only version 2.
 *
 * pack: host only; RB200_E_MODEL for a block that does not sum to 4096, RB200_E_ARG for bad geometry or a directory
 * that disagrees with the blob.  open: as rb200_container_open (pointers INTO buf, which must be 8-byte aligned). */
typedef struct rb200_container_blocks_info {
    uint32_t n_blocks, block_size, chunk_syms, flags;
    uint64_t n_symbols, n_chunks, blob_bytes;
    const uint16_t* block_freqs;    /* n_blocks x 256 */
    const uint64_t* offsets;        /* n_chunks + 1 */
    const uint8_t* blob;
} rb200_container_blocks_info;

size_t rb200_container_blocks_size(uint32_t n_blocks, size_t n_chunks, size_t blob_bytes);
int rb200_container_blocks_pack(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms, const uint16_t* block_freqs,
                                const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes, uint32_t flags,
                                uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_blocks_open(const uint8_t* buf, size_t size, rb200_container_blocks_info* info);
/* rb200_blocks_model_encode (block_freqs == NULL: every block's model is built on the GPU and written straight into
 * the container's model section) or rb200_blocks_encode (the caller's tables, in host or device memory as mem_kind)
 * + rb200_container_blocks_pack in one call, with the rules of rb200_container_encode: out 16-byte aligned (DEVICE)
 * or 8-byte aligned (HOST); out_cap below header, model and directory is RB200_E_SPACE from the call; a blob past
 * out_cap is RB200_E_SPACE from the call (HOST) or from rb200_sync (DEVICE, header then unwritten);
 * rb200_container_blocks_size(n_blocks, n_chunks, rb200_encode_bound(n, chunk_syms)) always suffices.  A caller table
 * that does not sum to 4096 is RB200_E_MODEL from the call in HOST mode; in DEVICE mode the block encoder codes such
 * a block with an empty model, so rb200_sync returns RB200_E_SYMBOL and the header is not written. */
int rb200_container_blocks_encode(rb200_ctx* ctx, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                  const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags,
                                  uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind);
/* rb200_container_blocks_open + rb200_blocks_decode in one call, with the rules of rb200_container_decode: *n_symbols
 * written and out_cap < n RB200_E_SPACE before any decoding; DEVICE mode checks both CRCs on the GPU before any
 * decode kernel runs (a rejected container leaves out untouched); HOST mode takes the blob CRC per slice. */
int rb200_container_blocks_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                  uint64_t* n_symbols, int mem_kind);
/* rb200_container_blocks_decode for a container in DEVICE memory, with nothing done on the host: the header, every
 * block's model, the directory, meta_crc and (when flagged) the blob CRC are checked by kernels, then the block decoder
 * runs -- all enqueued on the context stream; the call never synchronises, copies to the host or allocates, so it can
 * be captured in a CUDA graph.  buf and out 16-byte aligned.  size = bytes available at buf (a shorter container is
 * accepted, as by rb200_container_blocks_open).  d_n_symbols (device memory, may be NULL) receives n once header,
 * models and directory pass.  The call returns only RB200_E_ARG (null / misaligned / bad mem) or RB200_E_CUDA;
 * every verdict on the container comes from rb200_sync: RB200_E_STREAM for anything rb200_container_blocks_open
 * rejects, RB200_E_SPACE for n > out_cap; in both cases out is untouched.  One difference from
 * rb200_container_blocks_decode: a container that open accepts but the decoder refuses (a blob of 2^36 bytes or more),
 * which that call reports as RB200_E_ARG, is RB200_E_STREAM here, out untouched. */
int rb200_container_blocks_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                        uint64_t* d_n_symbols);
/* ---------------------------------------------------------------- per-block models for the byte and rans64 coders */

/* The per-block calls above for RB200_CODER_BYTE (main.cpp: rans_byte + cum2sym) and RB200_CODER_RANS64 (main64.cpp) at
 * scale_bits 8..15, with the same geometry (block_size % chunk_syms == 0, at most 32 chunks per block, chunk = block *
 * (block_size / chunk_syms) + chunk-in-block).  block_freqs is [n_blocks][256] u16, each row normalised to
 * 1 << scale_bits; every chunk is the coder's ordinary 32-way stream under its block's row, as rb200_encode writes it
 * with that model.  model_encode builds every block's model on the GPU (count_freqs + normalize_freqs(1 << scale_bits),
 * main.cpp:59-129, bit-exact) and writes it to block_freqs.  HOST mode pipelines slices of whole blocks like
 * rb200_blocks_encode; DEVICE mode only enqueues.  RB200_E_ARG (nothing launched) for a coder other than BYTE or RANS64,
 * scale_bits outside 8..15, a bad geometry, a null pointer, a bad mem_kind or 2^31 chunks or more.  A caller table
 * whose block does not sum to 1 << scale_bits is RB200_E_MODEL from the call in HOST mode; in DEVICE mode that block is
 * coded with an empty model and rb200_sync returns RB200_E_SYMBOL.  A symbol of frequency 0 is RB200_E_SYMBOL; a decode
 * table that does not sum, or a corrupt stream, is RB200_E_STREAM. */
int rb200_blocks_coder_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                              uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms,
                              uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind);
int rb200_blocks_coder_model_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                    uint32_t block_size, uint16_t* block_freqs, uint32_t chunk_syms,
                                    uint8_t* blob, size_t blob_cap, uint64_t* offsets, size_t* blob_size, int mem_kind);
int rb200_blocks_coder_decode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* blob, size_t blob_size,
                              const uint64_t* offsets, const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size,
                              uint32_t chunk_syms, uint8_t* out, int mem_kind);

/* Their container, version 3: version 2's layout (rb200_container_blocks_size gives its size) with the header's own
 * coder (byte 6: RB200_CODER_BYTE or RB200_CODER_RANS64) and scale_bits (byte 7: 8..15); every block's frequencies sum
 * to 1 << scale_bits, and every other rule is version 2's.  The _coder_ calls accept only version 3, the other container
 * calls reject it.  pack: host only; RB200_E_ARG for a bad coder or scale_bits and as rb200_container_blocks_pack,
 * RB200_E_MODEL for a block that does not sum.  open: as rb200_container_blocks_open, with coder and scale_bits.
 * encode: block_freqs == NULL builds the models on the GPU straight into the model section; otherwise the rules of
 * rb200_container_blocks_encode with the total 1 << scale_bits.  decode: the rules of rb200_container_blocks_decode.
 * The alias coder's per-block container is version 4 (rb200_container_blocks_alias_*, below). */
typedef struct rb200_container_blocks_coder_info {
    uint32_t coder, scale_bits;
    uint32_t n_blocks, block_size, chunk_syms, flags;
    uint64_t n_symbols, n_chunks, blob_bytes;
    const uint16_t* block_freqs;    /* n_blocks x 256 */
    const uint64_t* offsets;        /* n_chunks + 1 */
    const uint8_t* blob;
} rb200_container_blocks_coder_info;

int rb200_container_blocks_coder_pack(int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                      const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes,
                                      uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_blocks_coder_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info);
int rb200_container_blocks_coder_encode(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                        uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags,
                                        uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind);
int rb200_container_blocks_coder_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                        uint64_t* n_symbols, int mem_kind);
/* rb200_container_blocks_coder_decode(..., RB200_MEM_DEVICE) with nothing done on the host: the header, every block's
 * model, the directory, meta_crc and (when flagged) the blob CRC are checked by kernels, and the block decoder of the
 * header's coder and scale_bits is picked on the GPU -- all enqueued on the context stream.  The rules of
 * rb200_container_blocks_decode_async apply: DEVICE memory only, buf and out 16-byte aligned, d_n_symbols 8-byte
 * aligned or NULL; the call never synchronises, copies to or from the host or allocates, so it can be captured in a
 * CUDA graph, and returns only RB200_E_ARG (nothing launched) or RB200_E_CUDA.  *d_n_symbols receives n once header,
 * models and directory pass (also when the blob CRC then fails).  rb200_sync gives the verdict: RB200_E_STREAM for
 * anything rb200_container_blocks_coder_open rejects (version 1, 2 and 4 containers among them), RB200_E_SPACE for
 * n > out_cap, content errors first; in both cases out is untouched.  A corrupt stream that passes every check is
 * RB200_E_STREAM, as from rb200_blocks_coder_decode.  One difference from rb200_container_blocks_coder_decode: a
 * container that open accepts but the decoders refuse (a blob of 2^36 bytes or more), which that call reports as
 * RB200_E_ARG, is RB200_E_STREAM here, out untouched. */
int rb200_container_blocks_coder_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                              uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- per-block models for the alias coder */

/* The per-block calls of the byte and rans64 coders for RB200_CODER_ALIAS (main_alias.cpp: rans_byte + alias table) at
 * scale_bits 8..15: the same geometry, memory kinds, HOST slice pipeline and error codes.  Each block's alias table
 * (make_alias_table, main_alias.cpp:147-237, bit-exact with rb200_alias_tables_build) is built on the GPU from its
 * row of block_freqs by the encoding or decoding CTA; every chunk is the alias coder's ordinary 32-way stream under its
 * block's row, as rb200_encode writes it with that model.  RB200_E_ARG (nothing launched) for scale_bits outside 8..15,
 * a bad geometry, a null pointer, a bad mem_kind or 2^31 chunks or more. */
int rb200_blocks_alias_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                              const uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                              uint64_t* offsets, size_t* blob_size, int mem_kind);
int rb200_blocks_alias_model_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks, uint32_t block_size,
                                    uint16_t* block_freqs, uint32_t chunk_syms, uint8_t* blob, size_t blob_cap,
                                    uint64_t* offsets, size_t* blob_size, int mem_kind);
int rb200_blocks_alias_decode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* blob, size_t blob_size, const uint64_t* offsets,
                              const uint16_t* block_freqs, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                              uint8_t* out, int mem_kind);

/* Their container, version 4: version 3 with coder RB200_CODER_ALIAS (byte 6) at scale_bits 8..15 (byte 7); every other
 * rule is version 3's.  The _alias_ calls accept only version 4, every other container call (the version 1-3 async
 * decodes included) rejects it.  pack, open, encode and decode behave as the _coder_ calls; open fills the version 3
 * info struct. */
int rb200_container_blocks_alias_pack(uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                      const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob,
                                      size_t blob_bytes, uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_blocks_alias_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info);
int rb200_container_blocks_alias_encode(rb200_ctx* ctx, uint32_t scale_bits, const uint8_t* in, uint32_t n_blocks,
                                        uint32_t block_size, const uint16_t* block_freqs, uint32_t chunk_syms, uint32_t flags,
                                        uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind);
int rb200_container_blocks_alias_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                        uint64_t* n_symbols, int mem_kind);
/* rb200_container_blocks_alias_decode(..., RB200_MEM_DEVICE) with nothing done on the host: the header, every block's
 * model, the directory, meta_crc and (when flagged) the blob CRC are checked by kernels, the block decoder of the
 * header's scale_bits is picked on the GPU, and each decoding CTA builds its block's alias table -- all enqueued on the
 * context stream.  Exactly the contract of rb200_container_blocks_coder_decode_async with version 4 in place of
 * version 3: DEVICE memory only, buf and out 16-byte aligned, d_n_symbols 8-byte aligned or NULL; the call never
 * synchronises, copies to or from the host or allocates, so it can be captured in a CUDA graph, and returns only
 * RB200_E_ARG (nothing launched) or RB200_E_CUDA.  *d_n_symbols receives n once header, models and directory pass.
 * rb200_sync gives the verdict: RB200_E_STREAM for anything rb200_container_blocks_alias_open rejects (version 1, 2 and
 * 3 containers among them), RB200_E_SPACE for n > out_cap, content errors first; in both cases out is untouched.  A
 * corrupt stream that passes every check is RB200_E_STREAM, as from rb200_blocks_alias_decode.  A blob of 2^36 bytes or
 * more, which rb200_container_blocks_alias_decode reports as RB200_E_ARG, is RB200_E_STREAM here, out untouched. */
int rb200_container_blocks_alias_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                              uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- per-block containers with stored blocks */

/* Version 5: the layout of versions 2-4 (rb200_container_blocks_size gives its size) with the header of the per-block
 * version of its pair (bytes 6-7: word at 12; byte, rans64 or alias at 8..15) and the version field 5.  A block whose
 * row of block_freqs is all zero is STORED: each of its chunks is a stream of round16(chunk_syms) bytes, the chunk's
 * symbols and then zero bytes, placed in the blob and the directory by the rules of a coded stream of that length
 * (so the chunk's directory step, (offsets[c + 1] & ~15) - offsets[c], is exactly round16(chunk_syms)).  Every other
 * row sums to 1 << scale_bits and its block is coded as in versions 2-4.  Only the _stored_ calls accept version 5;
 * every other container call, rb200_container_blocks_any_decode_async included, rejects it (RB200_E_STREAM).
 *   bound: header + models + directory + n_chunks x round16(chunk_syms): the most any version 5 container of that
 *          geometry takes (0 for a geometry the per-block calls refuse).
 *   pack:  host only; block_freqs with zero rows for stored blocks.  RB200_E_ARG for a bad pair or geometry, a null
 *          pointer, and a directory that disagrees with the blob or gives a stored chunk the wrong step or nonzero
 *          padding; RB200_E_MODEL for a row that is neither zero nor sums to 1 << scale_bits; RB200_E_SPACE when out_cap
 *          is below the container.
 *   open:  as rb200_container_blocks_coder_open (the version 3 info struct), with the rules above and those of the
 *          twin version; RB200_E_STREAM for anything else, versions 1-4 among them. */
size_t rb200_container_blocks_stored_bound(uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms);
int rb200_container_blocks_stored_pack(int coder, uint32_t scale_bits, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                       const uint16_t* block_freqs, const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes,
                                       uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_blocks_stored_open(const uint8_t* buf, size_t size, rb200_container_blocks_coder_info* info);
/* A version 5 container of the blocks at `in`, in DEVICE memory with the models built on the GPU, enqueued only: the
 * pair is rb200_choose_blocks_coder's choice over `candidates` (every block counted, stored or not; one candidate is
 * encoded as it is, with no choice kernel), every block is encoded with it, and then a block is stored when its coded
 * chunks take more than (block_size / chunk_syms) x round16(chunk_syms) bytes of blob (each stream rounded up to 16).
 * The decision is made from the streams the encoder wrote, so out_cap >= rb200_container_blocks_stored_bound(n_blocks,
 * block_size, chunk_syms) always suffices.  Arguments, space and sync verdicts are those of
 * rb200_container_blocks_model_encode_auto_async: RB200_E_ARG (nothing launched) for a null ctx, in or out, a misaligned
 * out, an invalid list or candidate, tolerance_ppm > 10^6, a bad geometry or 2^31 chunks or more; RB200_E_SPACE when
 * out_cap is below the blob offset; rb200_sync returns RB200_E_SPACE when the blob does not fit out_cap, header
 * unwritten.  Capturable in a CUDA graph after one call with the same list and geometry outside the capture. */
int rb200_container_blocks_stored_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                               const uint8_t* in, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                                               uint32_t flags, uint8_t* out, size_t out_cap);
/* rb200_container_blocks_stored_encode_async with the block count read from device memory when the work runs: for
 * 1 <= *d_n_blocks <= n_blocks_max the container is byte for byte (header included) what the fixed call writes for
 * n_blocks = *d_n_blocks, so one captured graph writes a bounded container of any count up to n_blocks_max.  Only the
 * first *d_n_blocks blocks of in are read and nothing at or past the container's end is written.  n_blocks_max fixes
 * the launch shapes and the workspace; the bound grows with the count, so out_cap >=
 * rb200_container_blocks_stored_bound(n_blocks_max, block_size, chunk_syms) means rb200_sync never returns
 * RB200_E_SPACE, whatever the count.  The call returns RB200_E_ARG (nothing launched) for everything the fixed call
 * refuses, checked with n_blocks_max, for a null or not 4-byte aligned d_n_blocks and for n_blocks_max == 0;
 * RB200_E_SPACE when out_cap is below the blob offset for n_blocks_max.  rb200_sync returns RB200_E_ARG when
 * *d_n_blocks is 0 or above n_blocks_max, and then out is not written at all; every other verdict is the fixed call's,
 * with the header unwritten on every error.  The call only enqueues work (no copy, synchronisation or allocation); the
 * workspace grows for n_blocks_max, so a call with the same list, geometry and bound outside a capture must come first. */
int rb200_container_blocks_stored_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                      uint32_t tolerance_ppm, const uint8_t* in, const uint32_t* d_n_blocks,
                                                      uint32_t n_blocks_max, uint32_t block_size, uint32_t chunk_syms,
                                                      uint32_t flags, uint8_t* out, size_t out_cap);
/* The contract of rb200_container_blocks_alias_decode_async with version 5 in place of version 4: kernels check the
 * header, every row (zero or summing), the directory, every stored chunk's step and padding, meta_crc and the optional
 * blob CRC, then the block decoder of the header's pair runs, copying stored blocks and decoding the others.  DEVICE
 * memory only, buf and out 16-byte aligned, d_n_symbols 8-byte aligned or NULL; enqueue only; RB200_E_ARG (nothing
 * launched) or RB200_E_CUDA from the call.  rb200_sync gives the verdict: RB200_E_STREAM for anything
 * rb200_container_blocks_stored_open rejects (versions 1-4 among them) and for a blob of 2^36 bytes or more,
 * RB200_E_SPACE for n > out_cap, content errors first; in both cases out is untouched.  A corrupt coded stream that
 * passes every check is RB200_E_STREAM. */
int rb200_container_blocks_stored_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                               uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- single-model containers with stored chunks */

/* Version 6: version 1's header (version field 6; block_size, n_blocks and reserved zero, which is checked), model and
 * directory at 1088, then from the next 16-byte boundary a stored-chunk bitmap, ceil(n_chunks / 32) u32 words with bit
 * c % 32 of word c / 32 set when chunk c is stored, zero-padded to 16 bytes, then the blob.  Bits at or past n_chunks
 * and the padding are zero.  meta_crc covers every byte before the blob: header (crc fields zero), model, directory,
 * the zero pad after it and the bitmap.  A stored chunk of m_c symbols (chunk_syms, or fewer for a ragged last chunk)
 * is a stream of round16(m_c) bytes, its symbols and then zero bytes, placed by the rules of a coded stream of that
 * length: its directory step, (offsets[c + 1] & ~15) - offsets[c], is exactly round16(m_c).  The model is always
 * present and valid, even when every chunk is stored.  Only the _stored_ calls below accept version 6; every other
 * container call rejects it (RB200_E_STREAM), and they reject versions 1-5.
 *   bound: the blob offset + the sum of round16(m_c): the most any version 6 container of n symbols takes (0 for n == 0,
 *          n >= 2^32 or chunk_syms outside 32 .. 2^24).
 *   pack:  host only; stored_bits holds ceil(n_chunks / 32) words.  RB200_E_ARG for a bad pair (as
 *          rb200_container_model_encode_async takes it) or length, a null pointer, a bit at or past n_chunks, and a
 *          directory that disagrees with the blob or gives a stored chunk the wrong step or nonzero padding;
 *          RB200_E_MODEL for a model that does not sum to 1 << scale_bits; RB200_E_SPACE when out_cap is below the
 *          container.
 *   open:  as rb200_container_open, with the rules above; *stored_bits points at the bitmap in buf. */
struct rb200_container_info;   /* defined with rb200_container_open below */
size_t rb200_container_stored_bound(size_t n, uint32_t chunk_syms);
int rb200_container_stored_pack(int coder, uint32_t scale_bits, uint32_t chunk_syms, size_t n, const uint32_t freqs[256],
                                const uint32_t* stored_bits, const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes,
                                uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_stored_open(const uint8_t* buf, size_t size, struct rb200_container_info* info, const uint32_t** stored_bits);
/* A version 6 container of n symbols at `in`, DEVICE memory, enqueued only: the pair is the choice of
 * rb200_container_model_encode_auto_async (d_n NULL) over `candidates`, every chunk is encoded with it, and then chunk c
 * is stored when its stream, rounded up to 16, is longer than round16(m_c).  The decision is made from the streams the
 * encoder wrote, so out_cap >= rb200_container_stored_bound(n, chunk_syms) always suffices.  Arguments and verdicts are
 * those of rb200_container_model_encode_auto_async with d_n NULL: RB200_E_ARG (nothing launched), RB200_E_MODEL for
 * n == 0, RB200_E_SPACE when out_cap is below the blob offset; rb200_sync returns RB200_E_MODEL when no candidate is
 * feasible and RB200_E_SPACE when the blob does not fit out_cap, header unwritten.  Capturable in a CUDA graph after one
 * call with the same list and geometry outside the capture. */
int rb200_container_stored_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                        const uint8_t* in, size_t n, uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap);
/* rb200_container_stored_encode_async with the length read from device memory when the work runs: for
 * 1 <= *d_n <= n_max the container is byte for byte (header included) what the fixed call writes for n = *d_n, so one
 * captured graph writes a bounded container of any length up to n_max.  Only the first *d_n symbols of in are read
 * and nothing at or past the container's end is written.  n_max fixes the launch shapes and the workspace; the bound
 * grows with the length, so out_cap >= rb200_container_stored_bound(n_max, chunk_syms) means rb200_sync never returns
 * RB200_E_SPACE, whatever the length.  d_n is device memory, 8-byte aligned.  The call returns RB200_E_ARG (nothing
 * launched) for everything the fixed call refuses, checked with n_max and for every candidate, for a null or misaligned
 * d_n and for n_max == 0; RB200_E_SPACE when out_cap is below the blob offset for n_max.  rb200_sync returns
 * RB200_E_MODEL for *d_n == 0 (the fixed call's verdict for n == 0) and RB200_E_ARG for *d_n > n_max, and then out is
 * not written at all; every other verdict is the fixed call's, with the header unwritten on every error.  The call only
 * enqueues work (no copy, synchronisation or allocation); the workspace grows for n_max, so a call with the same list,
 * chunk_syms and n_max outside a capture must come first. */
int rb200_container_stored_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                               uint32_t tolerance_ppm, const uint8_t* in, const uint64_t* d_n, size_t n_max,
                                               uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap);
/* The contract of rb200_container_decode_async with version 6 in place of version 1: kernels check the header, the
 * model, the directory, the bitmap, every stored chunk's step and padding, meta_crc and the optional blob CRC; then the
 * decoder of the header's coder runs, copying stored chunks and decoding the others.  rb200_sync gives RB200_E_STREAM
 * for anything rb200_container_stored_open rejects (versions 1-5 among them) or the decoders refuse, RB200_E_SPACE for
 * n > out_cap, content errors first; in both cases out is untouched. */
int rb200_container_stored_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                        uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- byte-plane containers */

/* Version 7: the n bytes of a tensor of w-byte elements (w = elem_bytes, 2, 4 or 8) as w byte planes, plane p holding
 * byte p of every element in element order (little-endian, as the tensor lies in memory), each plane a complete version
 * 6 container of n / w symbols.  Layout: a 64-byte header (version 7, coder and scale_bits 0, lanes 32, chunk_syms, n
 * in n_symbols, n_chunks 0, blob_bytes = the bytes after the plane table, the caller's flags, meta_crc over the header
 * (crc fields zero) and the table, blob_crc 0, block_size = n_blocks = w, reserved 0), then w table entries {u64 offset,
 * u64 size}, then the planes with no gaps: offset[0] = 64 + 16 w, offset[p + 1] = offset[p] + size[p], size[p] the
 * plane's exact size.  Every plane has the header's chunk_syms (32 .. 2^24) and flags.  n is a nonzero multiple of w
 * with n / w < 2^32.  Only the _planes_ calls accept version 7, and they accept no other version.
 *   bound: 64 + 16 w + w * rb200_container_stored_bound(n / w, chunk_syms); 0 for arguments the encode refuses.
 *   pack:  host only, from w version 6 containers (each exactly sizes[p] bytes, 8-byte aligned) that agree on n,
 *          chunk_syms and flags.  RB200_E_ARG for a bad elem_bytes, a null pointer or a plane that
 *          rb200_container_stored_open rejects or that disagrees; RB200_E_SPACE when out_cap is below the container.
 *   open:  checks the header, the table, meta_crc and every plane by rb200_container_stored_open's rules; RB200_E_STREAM
 *          for anything else (versions 1-6 among them), RB200_E_ARG for a null pointer or a buf that is not 8-byte
 *          aligned.  info->planes[p] / sizes[p] are views into buf that rb200_container_stored_open accepts. */
typedef struct rb200_container_planes_info {
    uint32_t elem_bytes, chunk_syms, flags, reserved;
    uint64_t n;
    const uint8_t* planes[8];
    size_t sizes[8];
} rb200_container_planes_info;
size_t rb200_container_planes_bound(size_t n, uint32_t elem_bytes, uint32_t chunk_syms);
int rb200_container_planes_pack(uint32_t elem_bytes, const uint8_t* const* planes, const size_t* sizes, uint8_t* out, size_t out_cap,
                                size_t* out_size);
int rb200_container_planes_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info);
/* A version 7 container of the n bytes at `in`, DEVICE memory, enqueued only: plane p is byte for byte what
 * rb200_container_stored_encode_async writes for plane p's bytes with the same candidates, tolerance_ppm, chunk_syms
 * and flags, so each plane picks its own coder.  in and out 16-byte aligned.  The call returns RB200_E_ARG (nothing
 * launched) for everything rb200_container_stored_encode_async refuses for n / w symbols, an elem_bytes other than 2, 4
 * or 8, n == 0 or not a multiple of it, n / w >= 2^32, and a misaligned in; RB200_E_SPACE (nothing launched) when
 * out_cap is below rb200_container_planes_bound.  rb200_sync gives the first failing plane's verdict (RB200_E_MODEL when
 * no candidate is feasible for a plane), and the version 7 header is then not written.  Capturable in a CUDA graph
 * after one call with the same list and geometry outside the capture (the workspaces grow). */
int rb200_container_planes_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                        uint32_t elem_bytes, const uint8_t* in, size_t n, uint32_t chunk_syms, uint32_t flags,
                                        uint8_t* out, size_t out_cap);
/* rb200_container_planes_encode_async with the length in bytes read from device memory when the work runs: for
 * 1 <= *d_n <= n_max with *d_n a multiple of w = elem_bytes, the container is byte for byte (header included) what the
 * fixed call writes for n = *d_n with the same arguments, so one captured graph writes a version 7 container of any
 * such length.  Only the first *d_n bytes of in are read and nothing at or past the container's end (64 + 16 w +
 * blob_bytes) is written.  n_max fixes the launch shapes and the workspaces; rb200_container_planes_bound is monotone
 * in n, so out_cap >= rb200_container_planes_bound(n_max, w, chunk_syms) means rb200_sync never returns
 * RB200_E_SPACE, whatever the length.  d_n is device memory, 8-byte aligned.  The call returns RB200_E_ARG (nothing
 * launched) for everything the fixed call refuses, checked with n_max for n (n_max not a multiple of w, n_max / w >=
 * 2^32, every candidate at n_max / w symbols, a misaligned in), for a null or misaligned d_n and for n_max == 0;
 * RB200_E_SPACE (nothing launched) when out_cap is below rb200_container_planes_bound(n_max, w, chunk_syms).
 * rb200_sync returns RB200_E_ARG when *d_n is 0, not a multiple of w or above n_max (the fixed call's verdict for such
 * an n), and then out is not written at all; every other verdict is the fixed call's, the first failing plane's with
 * the version 7 header unwritten.  The call only enqueues work (no copy, synchronisation or allocation); the
 * workspaces grow for n_max, so a call with the same list, elem_bytes, chunk_syms and n_max outside a capture must
 * come first.  The version 7 decode needs no device-length form: captured with size = the bound, it reads every
 * shorter container. */
int rb200_container_planes_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                               uint32_t tolerance_ppm, uint32_t elem_bytes, const uint8_t* in,
                                               const uint64_t* d_n, size_t n_max, uint32_t chunk_syms, uint32_t flags,
                                               uint8_t* out, size_t out_cap);
/* The contract of rb200_container_stored_decode_async for version 7, with the element width the caller expects: kernels
 * check the header (its w must be elem_bytes), the table and meta_crc, and every plane through version 6's checks and
 * decoders, into a workspace of min(out_cap, w * 2^32) bytes; only when every check has passed does one kernel
 * interleave the planes into out.  *d_n_symbols receives n once the header, the table and the planes' headers pass.
 * rb200_sync gives RB200_E_STREAM for anything rb200_container_planes_open rejects, a w other than elem_bytes or a
 * plane that fails its checks, and RB200_E_SPACE for n > out_cap once the header and table pass (whatever the planes
 * hold); in both cases out is untouched.  A corrupt coded stream that passes every check is RB200_E_STREAM.
 * RB200_E_ARG (nothing launched) for a bad elem_bytes or the arguments rb200_container_stored_decode_async refuses.
 * Capturable after one call of the same size and out_cap outside the capture (the workspaces grow). */
int rb200_container_planes_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size, uint8_t* out,
                                        size_t out_cap, uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- delta byte-plane containers */

/* Version 8: a tensor of w-byte elements (w = elem_bytes, 2, 4 or 8) as its difference from a base tensor of the same n
 * bytes that the receiver already holds (the previous checkpoint or weight sync).  The layout and every rule are
 * version 7's, but for two header fields: version 8, and reserved = the CRC-32 (rb200_crc32's) of the base's n bytes,
 * which meta_crc covers.  The planes hold d, not the input: for element i, with x and b the w-byte little-endian
 * unsigned integers of the input and the base, s = (x - b) mod 2^(8w) read as signed and d = (s << 1) ^ (s >> (8w - 1))
 * (arithmetic shift, mod 2^(8w)); byte k of d is in plane k.  The inverse x = b + ((d >> 1) ^ -(d & 1)) mod 2^(8w) is
 * exact for every bit pattern (NaNs, infinities, sign changes, integer extremes).  An unchanged tensor gives constant
 * zero planes.  Only the _delta_ calls accept version 8, and they accept no other version: a delta is never decoded
 * as a whole tensor.  The size bound is rb200_container_planes_bound's.
 *   pack / open: rb200_container_planes_pack / _open for version 8, with the base CRC as an argument / output. */
int rb200_container_delta_pack(uint32_t elem_bytes, const uint8_t* const* planes, const size_t* sizes, uint32_t base_crc, uint8_t* out,
                               size_t out_cap, size_t* out_size);
int rb200_container_delta_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info, uint32_t* base_crc);
/* rb200_container_planes_encode_async of the difference of in from base (both n bytes, DEVICE memory, 16-byte aligned):
 * plane p is byte for byte what rb200_container_stored_encode_async writes for plane p of d.  The same refusals as that
 * call, and RB200_E_ARG (nothing launched) for a null or misaligned base; out_cap >= rb200_container_planes_bound(n, w,
 * chunk_syms).  Enqueue only, capturable in a CUDA graph after one call with the same list and geometry outside the
 * capture (the workspaces grow). */
int rb200_container_delta_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                       uint32_t elem_bytes, const uint8_t* in, const uint8_t* base, size_t n, uint32_t chunk_syms,
                                       uint32_t flags, uint8_t* out, size_t out_cap);
/* The contract of rb200_container_planes_decode_async for version 8, applying the delta to base (DEVICE memory, 16-byte
 * aligned): out = base is allowed and applies it in place, so the receiver needs no second copy of its tensor.  Any
 * other overlap of [out, out + out_cap) and [base, base + out_cap) is RB200_E_ARG, nothing launched.  After the
 * header, the table and every plane pass, and n <= out_cap, a kernel takes the CRC of base's n bytes; a CRC other than
 * the header's is RB200_E_BASE from rb200_sync.  out is written only after every check, the base's included, has
 * passed, so a rejected buffer or a wrong base leaves out (and so an in-place base) untouched.  base is never read past
 * the header's n, and not at all when the container is rejected or n > out_cap.  A corrupt container is
 * RB200_E_STREAM and n > out_cap RB200_E_SPACE, as for version 7. */
int rb200_container_delta_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size, const uint8_t* base,
                                       uint8_t* out, size_t out_cap, uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- tensor-list containers */

/* Version 9: a list of T tensors of one element width w (elem_bytes, 2, 4 or 8), such as the bf16 or the fp32 tensors of
 * a state dict, as one container: version 7 of the concatenation of their bytes, in list order with no padding, plus a
 * directory of their lengths.  Layout: the 64-byte header (version 7's fields but for version 9, n_blocks = T with
 * 1 <= T <= 2^20, n_symbols = the total n, blob_bytes = the planes' bytes, reserved = the CRC-32 of the directory's 8 T
 * bytes, which meta_crc covers), w table entries {u64 offset, u64 size}, the directory (T u64 byte lengths, zero-padded
 * to a multiple of 16), then the w version 6 planes with no gaps from offset 64 + 16 w + round16(8 T).  Every length is
 * a multiple of w (zero allowed), and they sum to n, a nonzero multiple of w with n / w < 2^32.  Plane p is byte for
 * byte plane p of a version 7 container of the concatenated bytes.  Only the _tensors_ calls accept version 9, and
 * they accept no other version.
 *   bound: rb200_container_planes_bound(n_max, w, chunk_syms) + round16(8 count); 0 for a count outside 1..2^20 or
 *          arguments the planes bound refuses.
 *   pack:  host only: rb200_container_planes_pack's rules, and RB200_E_ARG for a null lengths, a count outside 1..2^20
 *          or lengths that are not multiples of w summing to the planes' n.
 *   open:  rb200_container_planes_open's checks, and the directory's CRC and rules (RB200_E_STREAM); *count and
 *          *lengths (a view into buf) receive the directory. */
typedef struct rb200_tensor_ref {
    uint64_t ptr;     /* device address of the tensor's bytes */
    uint64_t bytes;   /* encode: its length; decode: its capacity */
} rb200_tensor_ref;
size_t rb200_container_tensors_bound(size_t n_max, uint32_t count, uint32_t elem_bytes, uint32_t chunk_syms);
int rb200_container_tensors_pack(uint32_t elem_bytes, const uint64_t* lengths, uint32_t count, const uint8_t* const* planes,
                                 const size_t* sizes, uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_tensors_open(const uint8_t* buf, size_t size, rb200_container_planes_info* info, uint32_t* count,
                                 const uint64_t** lengths);
/* A version 9 container of the count tensors that d_refs names, DEVICE memory, enqueued only.  d_refs (count entries, 16
 * bytes each, 16-byte aligned) lives in device memory and is read when the work runs, so one captured graph encodes
 * whatever tensors the list names at each replay: their addresses and lengths may change between replays, as long as
 * the count stays and the total stays within n_max.  Each entry's bytes is a multiple of w (zero allowed) and its ptr
 * is aligned to w when bytes is not zero (element alignment is enough: views into a flat buffer work); the total is
 * 1 .. n_max.  A list that breaks any of these is RB200_E_ARG from rb200_sync, and not one byte of out is written.
 * The container is byte for byte rb200_container_tensors_pack of the lengths and of the planes that
 * rb200_container_planes_encode_async writes for the concatenated bytes with the same arguments.  The call returns
 * RB200_E_ARG (nothing launched) for everything rb200_container_planes_encode_varlen_async refuses at n_max, a count
 * outside 1..2^20 and a null or misaligned d_refs, and RB200_E_SPACE (nothing launched) when out_cap is below
 * rb200_container_tensors_bound(n_max, count, w, chunk_syms).  Every other verdict is the version 7 call's, the
 * header then unwritten.  Capturable after one call with the same list, elem_bytes, count, chunk_syms and n_max
 * outside the capture (the workspaces grow). */
int rb200_container_tensors_encode_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm,
                                         uint32_t elem_bytes, const rb200_tensor_ref* d_refs, uint32_t count, size_t n_max,
                                         uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap);
/* The decode of a version 9 container into the count outputs d_refs names (DEVICE memory, 16-byte aligned, read when
 * the work runs: each entry's ptr and its capacity in bytes).  Tensor i goes to refs[i].ptr; its length comes from
 * the directory.  rb200_sync gives RB200_E_STREAM for anything rb200_container_tensors_open rejects, a w other than
 * elem_bytes, a container T other than count or a plane that fails its checks, and RB200_E_SPACE for a stored length
 * above its ref's capacity or a total above n_max; in every one of these cases no output is touched.  d_lengths (NULL
 * or count u64, 8-byte aligned) receives the directory once it passes (also when a capacity then fails).  Outputs that
 * overlap each other or buf are a precondition violation, as for memcpy.  The call returns RB200_E_ARG (nothing
 * launched) for a bad elem_bytes, a null or misaligned buf, d_refs or d_lengths, n_max == 0 and a count outside
 * 1..2^20.  Enqueue only; capturable after one call of the same size, count and n_max outside the capture. */
int rb200_container_tensors_decode_async(rb200_ctx* ctx, uint32_t elem_bytes, const uint8_t* buf, size_t size,
                                         const rb200_tensor_ref* d_refs, uint32_t count, size_t n_max, uint64_t* d_lengths);

/* rb200_container_decode(..., RB200_MEM_DEVICE) for a version 1 container of any coder, with nothing done on the host:
 * the header, the model, the directory, meta_crc and (when flagged) the blob CRC are checked by kernels, the model's
 * decode table is built on the GPU into the context, and the decoder the header calls for is picked on the GPU -- all
 * enqueued on the context stream.  The rules of rb200_container_blocks_decode_async apply: DEVICE memory only, buf and
 * out 16-byte aligned, d_n_symbols 8-byte aligned or NULL; the call never synchronises, copies to the host or
 * allocates, so it can be captured in a CUDA graph, and returns only RB200_E_ARG (nothing launched) or RB200_E_CUDA.
 * *d_n_symbols receives n once header, model and directory pass (also when the blob CRC then fails).  rb200_sync gives
 * the verdict: RB200_E_STREAM for anything rb200_container_open rejects, RB200_E_SPACE for n > out_cap, content errors
 * first; in both cases out is untouched.  One difference from rb200_container_decode: a container that open accepts
 * but the decoders refuse (chunk_syms outside 32 .. 2^24, a blob of 2^36 bytes or more, a byte-coder frequency of
 * 65536), which that call reports as RB200_E_ARG or RB200_E_MODEL, is RB200_E_STREAM here, out untouched.  Version 2,
 * 3 and 4 containers are rejected (RB200_E_STREAM). */
int rb200_container_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                 uint64_t* d_n_symbols);

/* The encode side of the same: rb200_model_from_data(ctx, coder, scale_bits, in, n, RB200_MEM_DEVICE, ...), then
 * rb200_container_encode(..., RB200_MEM_DEVICE) with that model, then rb200_model_destroy -- the same container bytes,
 * with the model built on the GPU, so that the call only enqueues work on the context's stream: it never synchronises
 * or copies to the host, and it allocates nothing for the model.  `in` and `out` are device memory, `out` 16-byte
 * aligned.  The encode workspace grows as in rb200_container_encode, so a call of the same geometry outside a CUDA
 * graph capture must come first.  The call returns RB200_E_ARG (nothing launched) for a null ctx, in or out, a
 * misaligned out, an unknown coder, the word coder with scale_bits != 12, scale_bits outside 8 .. 16, chunk_syms outside
 * 32 .. 2^24, n >= 2^32 (counts of 32 bits, as rb200_model_from_data) or 2^31 chunks or more; RB200_E_MODEL for n == 0;
 * RB200_E_SPACE when out_cap is below the blob offset.  rb200_sync returns RB200_E_MODEL when rb200_model_create would
 * refuse the model (the byte coder at scale_bits 16 on data of one symbol: a frequency of 65536), RB200_E_SPACE when
 * the blob does not fit out_cap, RB200_E_STALL as elsewhere.  On every error the header is not written.  The container
 * is rb200_container_size(n_chunks, blob_bytes) bytes, blob_bytes from its header. */
int rb200_container_model_encode_async(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in, size_t n,
                                       uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap);

/* rb200_container_model_encode_async with the length in device memory: the call reads n = *d_n when it executes (at
 * every replay of a CUDA graph that captured it) and writes the bytes rb200_container_model_encode_async(ctx, coder,
 * scale_bits, in, *d_n, chunk_syms, flags, out, out_cap) writes.  n_max is a host-side bound that fixes the launch
 * shapes and the workspace, so one graph serves every 1 <= *d_n <= n_max; nothing is written at or past the container's
 * end, rb200_container_size(n_chunks, blob_bytes).  d_n is device memory, 8-byte aligned.  The call returns
 * RB200_E_ARG (nothing launched) by the fixed call's rules with n_max in place of n, and for a null or misaligned d_n
 * or n_max == 0; RB200_E_SPACE when out_cap is below the blob offset for n_max.  rb200_sync returns RB200_E_MODEL for
 * *d_n == 0 and RB200_E_ARG for *d_n > n_max (out is not written at all in either case), and otherwise what it returns
 * for the fixed call.  On every error the header is not written.  The workspace grows for n_max as the fixed call's
 * for n, so a call with the same (coder, chunk_syms, n_max) outside a capture must come first. */
int rb200_container_model_encode_varlen_async(rb200_ctx* ctx, int coder, uint32_t scale_bits, const uint8_t* in,
                                              const uint64_t* d_n, size_t n_max, uint32_t chunk_syms, uint32_t flags,
                                              uint8_t* out, size_t out_cap);

/* Choosing the coder from the data.  A candidate is a pair (coder, scale_bits) that rb200_container_model_encode_async
 * accepts -- word at 12; byte, alias or rans64 at 8..16 -- written RB200_CANDIDATE(coder, scale_bits).  A list holds 1 to
 * 16 distinct candidates in the caller's order of preference.  The rule, the same integer steps on the host and the GPU:
 *   f_i      = normalize_freqs(counts, 1 << sb_i), as rb200_model_from_data builds it;
 *   feasible = rb200_model_create accepts f_i for the coder (so the byte coder at 16 on data of one symbol is not);
 *   log2q(f) = log2 f in 16.16 fixed point: k = floor(log2 f), x = f << (31 - k), r = k << 16, then for i = 15 .. 0:
 *              x = (x * x) >> 31 in 64 bits, and if x >= 2^32, x >>= 1 and r |= 1 << i;
 *   bits_q   = sum over the symbols with counts[s] > 0 of counts[s] * ((sb_i << 16) - log2q(f_i[s]));
 *   cost_i   = ceil(bits_q / 2^19) + n_chunks * H (H = 256 for rans64, 128 otherwise: the 32 final states of a chunk),
 *              an estimate of the blob bytes; UINT64_MAX for an infeasible candidate.
 * The choice is the first candidate in list order whose cost is at most min + floor(min * tolerance_ppm / 10^6), min the
 * smallest cost.  {WORD 12, ALIAS 16} with 20000 ppm: the word coder unless alias at 16 is more than 2 % smaller. */
#define RB200_CANDIDATE(coder, scale_bits) ((uint32_t)(coder) << 8 | (uint32_t)(scale_bits))

/* The rule on the host, for counts[256] of n symbols (rb200_histogram's) cut into chunks of chunk_syms: costs[i]
 * (may be NULL) receives every candidate's cost and *chosen the index of the choice; with it, a caller whose data is in
 * host memory calls rb200_model_from_data and rb200_container_encode.  RB200_E_ARG for a null counts or chosen, an
 * invalid list, tolerance_ppm > 10^6, chunk_syms outside 32 .. 2^24, n >= 2^32 or counts that do not sum to n;
 * RB200_E_MODEL when no candidate is feasible (n == 0 included): costs are written, *chosen is not. */
int rb200_choose_coder(const uint64_t counts[256], size_t n, uint32_t chunk_syms, const uint32_t* candidates,
                       uint32_t n_candidates, uint32_t tolerance_ppm, uint64_t* costs, uint32_t* chosen);

/* rb200_container_model_encode_async with (coder, scale_bits) chosen by the rule above on the GPU, from the data's
 * histogram, at every run: one captured graph writes whichever coder suits the data it meets, and
 * rb200_container_decode_async decodes it.  The container is byte for byte what rb200_container_model_encode_async
 * writes for the chosen pair; the choice is recorded only in the header (bytes 6-7).  d_n == NULL encodes n symbols;
 * otherwise n is n_max and the length is read from *d_n at every run, by the rules of
 * rb200_container_model_encode_varlen_async.  The call returns RB200_E_ARG (nothing launched) for everything the fixed
 * (or varlen) call refuses, checked for every candidate, for an invalid candidate list and for tolerance_ppm > 10^6;
 * RB200_E_MODEL for n == 0 with d_n NULL; RB200_E_SPACE when out_cap is below the blob offset.  rb200_sync returns
 * RB200_E_MODEL when no candidate is feasible, and otherwise what it returns for the fixed call with the chosen pair.
 * On every error the header is not written.  The workspace grows for the largest encode plan over the candidates, so a
 * call with the same list and geometry outside a capture must come first. */
int rb200_container_model_encode_auto_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                            uint32_t tolerance_ppm, const uint8_t* in, const uint64_t* d_n, size_t n,
                                            uint32_t chunk_syms, uint32_t flags, uint8_t* out, size_t out_cap);

/* Choosing the coder of a per-block container (versions 2-4) from the blocks.  A candidate is RB200_CANDIDATE(coder,
 * scale_bits) with a pair some per-block version takes: word at 12 (version 2), byte or rans64 at 8..15 (version 3),
 * alias at 8..15 (version 4); a list holds 1 to 16 distinct candidates in order of preference.  The rule above, per
 * block b (counts c_b, block_size / chunk_syms chunks) and summed over the blocks:
 *   f          = normalize_freqs(c_b, 1 << sb_i): the block's model exactly as the model-building per-block encode
 *                writes it for (coder_i, sb_i);
 *   block_cost = ceil(bits_q / 2^19) + (block_size / chunk_syms) * H, bits_q and H as above; except for the word coder
 *                on a block of one symbol (f holds 4096), which costs what its encoder writes: 2 * block_size + 128 per
 *                chunk (every step emits a 16-bit word);
 *   cost_i     = the sum of block_cost over the blocks (the 512-byte model of each block is the same in every version
 *                and is not counted).
 * Every candidate is feasible on every block, so every cost is finite.  The choice is the first candidate whose cost is
 * at most min + floor(min * tolerance_ppm / 10^6).
 * rb200_choose_blocks_coder applies it on the host to block_counts (n_blocks x 256 counts, each row summing to
 * block_size): costs (may be NULL) receives every cost, *chosen the index of the choice.  RB200_E_ARG for a null
 * block_counts or chosen, an invalid list or a candidate no per-block version takes, a geometry the per-block calls
 * refuse, tolerance_ppm > 10^6, or a row that does not sum to block_size. */
int rb200_choose_blocks_coder(const uint32_t* block_counts, uint32_t n_blocks, uint32_t block_size, uint32_t chunk_syms,
                              const uint32_t* candidates, uint32_t n_candidates, uint32_t tolerance_ppm, uint64_t* costs,
                              uint32_t* chosen);

/* rb200_container_blocks_encode, rb200_container_blocks_coder_encode or rb200_container_blocks_alias_encode in DEVICE
 * memory with the models built (block_freqs NULL), for the pair the rule above picks on the GPU from the blocks at
 * every run: one captured graph writes a version 2, 3 or 4 container, whichever suits the data it meets, byte for byte
 * (header included) what the fixed call writes for the chosen pair.  in and out are device memory, out 16-byte aligned;
 * the geometry rules are the per-block calls'.  The call only enqueues work: a memset and one choice kernel, one gated
 * encode group per distinct encoder instance the list needs (only the chosen group runs), the CRCs and the header
 * kernel.  It returns RB200_E_ARG (nothing launched) for a null ctx, in or out, a misaligned out, an invalid list or
 * candidate, tolerance_ppm > 10^6, a bad geometry or 2^31 chunks or more; RB200_E_SPACE when out_cap is below the blob
 * offset (64 + 512 n_blocks + the directory, rounded to 16).  rb200_sync returns RB200_E_SPACE when the chosen blob does
 * not fit out_cap, with the header not written, as for the fixed call.  The workspace grows for every group's plan, so
 * a call with the same list and geometry outside a capture must come first.  rb200_container_blocks_auto_costs copies
 * the costs of the last run's choice (n <= 16 of them, the list's order) to host memory; it synchronises. */
int rb200_container_blocks_model_encode_auto_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                   uint32_t tolerance_ppm, const uint8_t* in, uint32_t n_blocks,
                                                   uint32_t block_size, uint32_t chunk_syms, uint32_t flags, uint8_t* out,
                                                   size_t out_cap);
int rb200_container_blocks_auto_costs(rb200_ctx* ctx, uint64_t* costs, uint32_t n);

/* rb200_container_blocks_model_encode_auto_async with the block count read from device memory when the work runs: for
 * 1 <= *d_n_blocks <= n_blocks_max the container is byte for byte what the fixed call writes for n_blocks =
 * *d_n_blocks, so one captured graph takes any count up to n_blocks_max.  Only the first *d_n_blocks blocks of in are
 * read and nothing past the container's end is written.  n_blocks_max fixes the launch shapes and the workspace, and the
 * host checks it: the geometry, fewer than 2^31 chunks, and out_cap at least its blob offset (RB200_E_SPACE below it);
 * the layout offsets and the encode bound grow with the count, so rb200_container_blocks_size for n_blocks_max holds
 * every smaller count.  RB200_E_ARG (nothing launched) also for a null, or not 4-byte aligned, d_n_blocks and for
 * n_blocks_max == 0.  rb200_sync returns RB200_E_ARG when *d_n_blocks is 0 or above n_blocks_max (zero blocks is the
 * fixed call's RB200_E_ARG too), and then out is not written at all; the other verdicts are the fixed call's.  The call
 * only enqueues work: the plan kernel, the choice kernel on a grid of n_blocks_max (its CTAs past the count exit), one
 * gated encode group per distinct encoder instance, the CRCs and the header kernel.  With one candidate the pair is
 * known, so the choice kernel is not launched: the plan kernel writes the choice, and rb200_container_blocks_auto_costs
 * is then undefined (it reads the costs of the last call that ran the choice kernel, one with two or more candidates).
 * The workspace grows for every group's plan at n_blocks_max, so a call with the same list and bounds outside a
 * capture must come first. */
int rb200_container_blocks_model_encode_varlen_async(rb200_ctx* ctx, const uint32_t* candidates, uint32_t n_candidates,
                                                     uint32_t tolerance_ppm, const uint8_t* in, const uint32_t* d_n_blocks,
                                                     uint32_t n_blocks_max, uint32_t block_size, uint32_t chunk_syms, uint32_t flags,
                                                     uint8_t* out, size_t out_cap);

/* The async decode of a per-block container of any version: the header's version field (bytes 4-5) picks version 2, 3
 * or 4, and the call then reaches the verdict, status and output of rb200_container_blocks_decode_async,
 * rb200_container_blocks_coder_decode_async or rb200_container_blocks_alias_decode_async on it, under the same rules
 * (DEVICE memory only, buf and out 16-byte aligned, d_n_symbols 8-byte aligned or NULL, enqueue only, RB200_E_ARG or
 * RB200_E_CUDA from the call, the verdict from rb200_sync).  Any other version, version 1 included, is RB200_E_STREAM.
 * Thirteen launches: the checks, then the decoders of all three versions, of which only the header version's can run.
 * A host caller that does not capture can read the version field itself and call the synchronous decode of that
 * version. */
int rb200_container_blocks_any_decode_async(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                                            uint64_t* d_n_symbols);

/* ---------------------------------------------------------------- multi-GPU: gathering the shards' blobs (NCCL) */

/* Shards are independent (SURVEY 8e): every rank encodes / decodes its own contiguous range of symbols with no
 * communication.  The one exchange step is collecting the compressed blobs + directories on one rank, which these
 * calls do over NCCL / NVLink (ncclAllGather of the sizes, then grouped ncclSend / ncclRecv of the payloads straight
 * into their final position; the directories are rebased on the root).  The concatenation is itself a valid container
 * because every shard's blob ends 16-byte aligned.  The reference analogue is the driver keeping `rans_begin` per
 * buffer (main_simd.cpp:287-300); it has no multi-device story.  libnccl.so.2 is loaded on first use (dlopen), so
 * single-GPU users need no NCCL.
 *
 *   rank 0: rb200_comm_unique_id(id)  -> hand the 128 bytes to every rank (file, socket, MPI, torch.distributed ...)
 *   all   : rb200_comm_create(ctx, id, rank, world, &comm)             (collective: ncclCommInitRank)
 *   all   : rb200_gather_plan(comm, blob_size, n_chunks, totals)       (collective, synchronises: sizes of every shard)
 *   all   : rb200_gather_blobs(comm, root, d_blob, d_offsets, d_out_blob, out_cap, d_out_offsets)
 *           enqueued on the context's stream; only `root` needs the out buffers: totals[0] bytes of blob and
 *           totals[1] + 1 directory entries.  May be repeated while the planned sizes stay valid. */
typedef struct rb200_comm rb200_comm;
#define RB200_NCCL_ID_BYTES 128
int rb200_comm_unique_id(uint8_t id[RB200_NCCL_ID_BYTES]);
int rb200_comm_create(rb200_ctx* ctx, const uint8_t id[RB200_NCCL_ID_BYTES], int rank, int world, rb200_comm** out);
void rb200_comm_destroy(rb200_comm* comm);
int rb200_gather_plan(rb200_comm* comm, uint64_t blob_size, uint64_t n_chunks, uint64_t totals[2]);
int rb200_gather_blobs(rb200_comm* comm, int root, const uint8_t* d_blob, const uint64_t* d_offsets,
                       uint8_t* d_out_blob, uint64_t out_cap, uint64_t* d_out_offsets);

/* ---------------------------------------------------------------- wire format (host only) */

/* Self-describing envelope around (freqs, offsets, blob): versioned 64-byte header (coder, scale_bits,
 * lanes, chunk_syms, n, n_chunks, blob size), the model, the directory, the blob; CRC-32 over header +
 * model + directory always, over the blob when RB200_CONTAINER_CRC_BLOB is given.  The reference has
 * nothing comparable (it keeps a pointer, main.cpp:182-188).  rb200_container_open validates and
 * returns pointers INTO buf (which must be 8-byte aligned; the blob then sits 16-byte aligned). */
#define RB200_CONTAINER_CRC_BLOB 1u

typedef struct rb200_container_info {
    uint32_t coder, scale_bits, chunk_syms, flags;
    uint64_t n_symbols, n_chunks, blob_bytes;
    const uint32_t* freqs;      /* 256 */
    const uint64_t* offsets;    /* n_chunks + 1 */
    const uint8_t* blob;
} rb200_container_info;

size_t rb200_container_size(size_t n_chunks, size_t blob_bytes);
int rb200_container_pack(int coder, uint32_t scale_bits, uint32_t chunk_syms, size_t n, const uint32_t freqs[256],
                         const uint64_t* offsets, const uint8_t* blob, size_t blob_bytes, uint32_t flags,
                         uint8_t* out, size_t out_cap, size_t* out_size);
int rb200_container_open(const uint8_t* buf, size_t size, rb200_container_info* info);

/* ---------------------------------------------------------------- wire format on the GPU */

/* zlib's crc32 (IEEE, reflected, init and xor-out ~0; the container's checksum) of n bytes of a host or device
 * buffer, computed on the GPU.  Any n and any alignment.  crc_in chains like zlib: crc(a || b) =
 * rb200_crc32(b, rb200_crc32(a, 0)); pass 0 to start.  HOST mode stages the buffer through the context.  *crc_out is
 * written to host memory; the call synchronises. */
int rb200_crc32(rb200_ctx* ctx, const uint8_t* data, size_t n, uint32_t crc_in, uint32_t* crc_out, int mem_kind);

/* rb200_encode + rb200_container_pack in one call: the directory and the blob are encoded straight into their place
 * in `out`, and the bytes equal what rb200_container_pack writes for the same model, input, chunk_syms and flags.
 * The model section is the model's own frequencies.  out_cap must hold rb200_container_size(n_chunks, blob size);
 * rb200_container_size(rb200_chunk_count(n, chunk_syms), rb200_encode_bound(n, chunk_syms)) always does.
 * flags: RB200_CONTAINER_CRC_BLOB adds the blob CRC, taken on the GPU.
 * HOST mode: synchronous; out 8-byte aligned; *out_size (may be NULL) receives the container's size.
 * DEVICE mode: out 16-byte aligned; work is only enqueued on the context stream (encode, CRCs, a header kernel) and
 * out_size is not written: the size is rb200_container_size(n_chunks, blob_bytes) with blob_bytes from the header.
 * A blob that does not fit out_cap is RB200_E_SPACE, from the call (HOST) or from rb200_sync (DEVICE, as for
 * rb200_encode; the header is then not written).  out_cap below the header, model and directory is RB200_E_SPACE
 * from the call in both modes. */
int rb200_container_encode(rb200_ctx* ctx, const rb200_model* model, const uint8_t* in, size_t n, uint32_t chunk_syms,
                           uint32_t flags, uint8_t* out, size_t out_cap, size_t* out_size, int mem_kind);

/* rb200_container_open + rb200_model_create + rb200_decode in one call, on a container in host or device memory.
 * The container is validated by the same rules as rb200_container_open (RB200_E_STREAM on any failure); *n_symbols
 * (may be NULL) then receives its n, and out_cap < n returns RB200_E_SPACE before any decoding, so a caller can
 * allocate and call again.  The call synchronises and returns one status for the whole call.
 * HOST mode: buf and out 8-byte aligned.  The header, model and directory are checked before decoding; the blob CRC
 * is taken slice by slice while decoding, so on a blob CRC mismatch (RB200_E_STREAM) out has been written and its
 * contents are unspecified.
 * DEVICE mode: buf and out 16-byte aligned.  Both CRCs are taken on the GPU before anything is decoded: a container
 * that fails any check leaves out untouched. */
int rb200_container_decode(rb200_ctx* ctx, const uint8_t* buf, size_t size, uint8_t* out, size_t out_cap,
                           uint64_t* n_symbols, int mem_kind);

#ifdef __cplusplus
}
#endif
#endif /* RANS_B200_H */

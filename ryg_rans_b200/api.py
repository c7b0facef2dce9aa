"""ctypes view of include/rans_b200.h.  No compute happens in Python."""
import ctypes as C
import os

import numpy as np

from .build import LIB_PATH, build

CODER_WORD, CODER_BYTE, CODER_ALIAS, CODER_RANS64 = 0, 1, 2, 3
MEM_HOST, MEM_DEVICE = 0, 1
LANES = 32

_u8p = C.POINTER(C.c_uint8)
_u16p = C.POINTER(C.c_uint16)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)

# every symbol include/rans_b200.h declares: (name, restype, argtypes)
EXPORTS = [
    ("rb200_count_freqs", C.c_int, [C.c_void_p, C.c_size_t, _u32p]),
    ("rb200_normalize_freqs", C.c_int, [_u32p, _u32p, C.c_uint32]),
    ("rb200_word_tables_build", C.c_int, [_u32p, _u32p, _u32p, _u8p]),
    ("rb200_alias_tables_build", C.c_int, [_u32p, _u32p, _u32p, _u32p, _u32p, _u8p, _u32p]),
    ("rb200_ctx_create", C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_void_p]),
    ("rb200_ctx_destroy", None, [C.c_void_p]),
    ("rb200_ctx_set_stream", C.c_int, [C.c_void_p, C.c_void_p]),
    ("rb200_sync", C.c_int, [C.c_void_p]),
    ("rb200_last_cuda_error", C.c_char_p, [C.c_void_p]),
    ("rb200_strerror", C.c_char_p, [C.c_int]),
    ("rb200_version", C.c_int, []),
    ("rb200_launch_count", C.c_uint64, [C.c_void_p]),
    ("rb200_model_create", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, _u32p, C.POINTER(C.c_void_p)]),
    ("rb200_model_destroy", None, [C.c_void_p]),
    ("rb200_chunk_count", C.c_size_t, [C.c_size_t, C.c_uint32]),
    ("rb200_encode_bound", C.c_size_t, [C.c_size_t, C.c_uint32]),
    ("rb200_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t,
                               C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p,
                               C.c_size_t, C.c_int]),
    ("rb200_histogram", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _u64p, C.c_int]),
    ("rb200_model_from_data", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t, C.c_int, _u32p,
                                        C.POINTER(C.c_void_p)]),
    ("rb200_blocks_build_models", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]),
    ("rb200_blocks_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                      C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_model_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p,
                                            C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                      C.c_uint32, C.c_void_p, C.c_int]),
    ("rb200_container_blocks_size", C.c_size_t, [C.c_uint32, C.c_size_t, C.c_size_t]),
    ("rb200_container_blocks_pack", C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                              C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_blocks_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_blocks_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32,
                                                C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_container_blocks_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, _u64p, C.c_int]),
    ("rb200_container_blocks_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_blocks_coder_encode", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                            C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_coder_model_encode", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                  C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_coder_decode", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32,
                                            C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]),
    ("rb200_container_blocks_coder_pack", C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_blocks_coder_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_blocks_coder_encode", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                      C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_container_blocks_coder_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, _u64p, C.c_int]),
    ("rb200_container_blocks_coder_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_blocks_alias_encode", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                            C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_alias_model_encode", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                  C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_blocks_alias_decode", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint32,
                                            C.c_uint32, C.c_uint32, C.c_void_p, C.c_int]),
    ("rb200_container_blocks_alias_pack", C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_blocks_alias_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_blocks_alias_encode", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                      C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_container_blocks_alias_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, _u64p, C.c_int]),
    ("rb200_container_blocks_alias_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_model_encode_async", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32,
                                                     C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_model_encode_varlen_async", C.c_int, [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                            C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_choose_coder", C.c_int, [_u64p, C.c_size_t, C.c_uint32, _u32p, C.c_uint32, C.c_uint32, _u64p, _u32p]),
    ("rb200_container_model_encode_auto_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                                          C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_choose_blocks_coder", C.c_int, [_u32p, C.c_uint32, C.c_uint32, C.c_uint32, _u32p, C.c_uint32, C.c_uint32, _u64p, _u32p]),
    ("rb200_container_blocks_model_encode_auto_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_blocks_auto_costs", C.c_int, [C.c_void_p, _u64p, C.c_uint32]),
    ("rb200_container_blocks_model_encode_varlen_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                                   C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_blocks_any_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_blocks_stored_bound", C.c_size_t, [C.c_uint32, C.c_uint32, C.c_uint32]),
    ("rb200_container_blocks_stored_pack", C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                     C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_blocks_stored_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_blocks_stored_encode_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                                             C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_blocks_stored_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_stored_bound", C.c_size_t, [C.c_size_t, C.c_uint32]),
    ("rb200_container_stored_pack", C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_size_t, _u32p, _u32p, C.c_void_p, C.c_void_p,
                                              C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_stored_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(_u32p)]),
    ("rb200_container_stored_encode_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32,
                                                      C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_stored_decode_async", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_stored_encode_varlen_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                             C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_blocks_stored_encode_varlen_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                                    C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                                                    C.c_size_t]),
    ("rb200_container_planes_bound", C.c_size_t, [C.c_size_t, C.c_uint32, C.c_uint32]),
    ("rb200_container_planes_pack", C.c_int, [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_planes_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_container_planes_encode_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t,
                                                      C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_planes_encode_varlen_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                                             C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_planes_decode_async", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                      C.c_void_p]),
    ("rb200_container_delta_pack", C.c_int, [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t,
                                             C.POINTER(C.c_size_t)]),
    ("rb200_container_delta_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, _u32p]),
    ("rb200_container_delta_encode_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                     C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_delta_decode_async", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                     C.c_size_t, C.c_void_p]),
    ("rb200_container_tensors_bound", C.c_size_t, [C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("rb200_container_tensors_pack", C.c_int, [C.c_uint32, _u64p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                               C.POINTER(C.c_size_t)]),
    ("rb200_container_tensors_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, _u32p, C.POINTER(_u64p)]),
    ("rb200_container_tensors_encode_async", C.c_int, [C.c_void_p, _u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                                       C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("rb200_container_tensors_decode_async", C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32,
                                                       C.c_size_t, C.c_void_p]),
    ("rb200_comm_unique_id", C.c_int, [C.c_void_p]),
    ("rb200_comm_create", C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    ("rb200_comm_destroy", None, [C.c_void_p]),
    ("rb200_gather_plan", C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, _u64p]),
    ("rb200_gather_blobs", C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    ("rb200_container_size", C.c_size_t, [C.c_size_t, C.c_size_t]),
    ("rb200_container_pack", C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_size_t, _u32p, C.c_void_p, C.c_void_p, C.c_size_t,
                                       C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("rb200_container_open", C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p]),
    ("rb200_crc32", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, _u32p, C.c_int]),
    ("rb200_container_encode", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p,
                                         C.c_size_t, C.POINTER(C.c_size_t), C.c_int]),
    ("rb200_container_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, _u64p, C.c_int]),
]
CONTAINER_CRC_BLOB = 1
# status codes (include/rans_b200.h); rb200_strerror has the message of each
E_ARG, E_MODEL, E_SPACE, E_STREAM, E_CUDA, E_NOMEM, E_SYMBOL, E_NCCL, E_STALL, E_BASE = range(-1, -11, -1)


def CANDIDATE(coder, scale_bits):
    """RB200_CANDIDATE: one (coder, scale_bits) pair of a coder-choice list"""
    return (coder << 8) | scale_bits


def _candidates(candidates):
    return np.ascontiguousarray(candidates, dtype=np.uint32)


def choose_coder(counts, n, chunk_syms, candidates, tolerance_ppm=0):
    """rb200_choose_coder: the rule of the auto encode on the host.  counts: the 256 counts of n symbols (as
    Context.histogram returns them); candidates: CANDIDATE values in order of preference.  Returns (index, costs), costs
    as u64 with 2^64 - 1 for an infeasible candidate; RansError -2 when none is feasible."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.uint64)
    assert counts.size == 256
    cands = _candidates(candidates)
    costs = np.zeros(max(cands.size, 1), np.uint64)
    chosen = C.c_uint32(0)
    lib.check(lib.dll.rb200_choose_coder(counts.ctypes.data_as(_u64p), n, chunk_syms, cands.ctypes.data_as(_u32p), cands.size,
                                         tolerance_ppm, costs.ctypes.data_as(_u64p), C.byref(chosen)))
    return int(chosen.value), costs[:cands.size]


def choose_blocks_coder(block_counts, block_size, chunk_syms, candidates, tolerance_ppm=0):
    """rb200_choose_blocks_coder: the rule of the per-block auto encode on the host.  block_counts: n_blocks x 256 counts,
    each row summing to block_size; candidates: CANDIDATE values of per-block pairs (word 12; byte, rans64 or alias at
    8..15), in order of preference.  Returns (index, costs), costs as u64 in list order."""
    lib = load()
    counts = np.ascontiguousarray(block_counts, dtype=np.uint32).reshape(-1, 256)
    cands = _candidates(candidates)
    costs = np.zeros(max(cands.size, 1), np.uint64)
    chosen = C.c_uint32(0)
    lib.check(lib.dll.rb200_choose_blocks_coder(counts.ctypes.data_as(_u32p), counts.shape[0], block_size, chunk_syms,
                                                cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm, costs.ctypes.data_as(_u64p),
                                                C.byref(chosen)))
    return int(chosen.value), costs[:cands.size]


class ContainerInfo(C.Structure):
    _fields_ = [("coder", C.c_uint32), ("scale_bits", C.c_uint32), ("chunk_syms", C.c_uint32), ("flags", C.c_uint32),
                ("n_symbols", C.c_uint64), ("n_chunks", C.c_uint64), ("blob_bytes", C.c_uint64),
                ("freqs", _u32p), ("offsets", _u64p), ("blob", _u8p)]


def container_pack(coder, scale_bits, chunk_syms, n, freqs, offsets, blob, flags=0):
    lib = load()
    freqs = np.ascontiguousarray(freqs, dtype=np.uint32)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    total = int(lib.dll.rb200_container_size(offsets.size - 1, blob.size))
    out = np.zeros(total, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_pack(coder, scale_bits, chunk_syms, n, freqs.ctypes.data_as(_u32p), offsets.ctypes.data,
                                           blob.ctypes.data, blob.size, flags, out.ctypes.data, total, C.byref(size)))
    return out[:size.value]


def container_open(buf):
    """Returns (info dict, freqs, offsets, blob) as numpy views into buf."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerInfo()
    lib.check(lib.dll.rb200_container_open(buf.ctypes.data, buf.size, C.byref(info)))
    base = buf.ctypes.data
    f_off = C.addressof(info.freqs.contents) - base
    o_off = C.addressof(info.offsets.contents) - base
    b_off = (C.addressof(info.blob.contents) - base) if info.blob_bytes else buf.size
    freqs = buf[f_off:f_off + 1024].view(np.uint32)
    offsets = buf[o_off:o_off + 8 * (info.n_chunks + 1)].view(np.uint64)
    blob = buf[b_off:b_off + info.blob_bytes]
    meta = {k: int(getattr(info, k)) for k in ("coder", "scale_bits", "chunk_syms", "flags", "n_symbols", "n_chunks", "blob_bytes")}
    return meta, freqs, offsets, blob


def container_stored_bound(n, chunk_syms):
    """rb200_container_stored_bound: the most bytes a version 6 container of n symbols takes (0 for a length or chunk size
    the calls refuse)"""
    return int(load().dll.rb200_container_stored_bound(n, chunk_syms))


def container_stored_pack(coder, scale_bits, chunk_syms, n, freqs, stored_bits, offsets, blob, flags=0):
    """rb200_container_stored_pack: a version 6 container (one model; bit c of stored_bits, ceil(n_chunks / 32) u32 words,
    marks chunk c stored, its stream round16(m_c) bytes of its symbols and zero padding)"""
    lib = load()
    freqs = np.ascontiguousarray(freqs, dtype=np.uint32)
    bits = np.ascontiguousarray(stored_bits, dtype=np.uint32)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    n_chunks = offsets.size - 1
    bitmap = (1088 + 8 * (n_chunks + 1) + 15) // 16 * 16                  # the layout of include/rans_b200.h
    out = np.zeros(bitmap + 16 * ((n_chunks + 127) // 128) + blob.size, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_stored_pack(coder, scale_bits, chunk_syms, n, freqs.ctypes.data_as(_u32p), bits.ctypes.data_as(_u32p),
                                                  offsets.ctypes.data, blob.ctypes.data, blob.size, flags, out.ctypes.data, out.size,
                                                  C.byref(size)))
    return out[:size.value].copy()


def container_stored_open(buf):
    """Returns (info dict, freqs, stored_bits, offsets, blob) as numpy views into buf (stored_bits: ceil(n_chunks / 32)
    u32 words)."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerInfo()
    bits_p = _u32p()
    lib.check(lib.dll.rb200_container_stored_open(buf.ctypes.data, buf.size, C.byref(info), C.byref(bits_p)))
    base = buf.ctypes.data
    f_off = C.addressof(info.freqs.contents) - base
    o_off = C.addressof(info.offsets.contents) - base
    s_off = C.addressof(bits_p.contents) - base
    b_off = (C.addressof(info.blob.contents) - base) if info.blob_bytes else buf.size
    freqs = buf[f_off:f_off + 1024].view(np.uint32)
    offsets = buf[o_off:o_off + 8 * (info.n_chunks + 1)].view(np.uint64)
    bits = buf[s_off:s_off + 4 * ((info.n_chunks + 31) // 32)].view(np.uint32)
    blob = buf[b_off:b_off + info.blob_bytes]
    meta = {k: int(getattr(info, k)) for k in ("coder", "scale_bits", "chunk_syms", "flags", "n_symbols", "n_chunks", "blob_bytes")}
    return meta, freqs, bits, offsets, blob


def container_planes_bound(n, elem_bytes, chunk_syms):
    """rb200_container_planes_bound: the most bytes a version 7 container of n bytes of elem_bytes-byte elements takes
    (0 for arguments the encode refuses)"""
    return int(load().dll.rb200_container_planes_bound(n, elem_bytes, chunk_syms))


class ContainerPlanesInfo(C.Structure):
    _fields_ = [("elem_bytes", C.c_uint32), ("chunk_syms", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32),
                ("n", C.c_uint64), ("planes", C.c_void_p * 8), ("sizes", C.c_size_t * 8)]


def container_planes_pack(planes):
    """rb200_container_planes_pack: a version 7 container from w = len(planes) version 6 containers (uint8 arrays, one
    per byte plane, agreeing on n, chunk_syms and flags)"""
    lib = load()
    planes = [np.ascontiguousarray(p, dtype=np.uint8) for p in planes]
    w = len(planes)
    ptrs = (C.c_void_p * max(w, 1))(*[p.ctypes.data for p in planes])
    sizes = (C.c_size_t * max(w, 1))(*[p.size for p in planes])
    out = np.zeros(64 + 16 * w + sum(p.size for p in planes), np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_planes_pack(w, ptrs, sizes, out.ctypes.data, out.size, C.byref(size)))
    return out[:size.value]


def container_planes_open(buf):
    """Returns (info dict, planes): planes[p] is a view into buf of plane p's version 6 container."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerPlanesInfo()
    lib.check(lib.dll.rb200_container_planes_open(buf.ctypes.data, buf.size, C.byref(info)))
    base = buf.ctypes.data
    planes = [buf[info.planes[p] - base:info.planes[p] - base + info.sizes[p]] for p in range(info.elem_bytes)]
    meta = {k: int(getattr(info, k)) for k in ("elem_bytes", "chunk_syms", "flags", "n")}
    return meta, planes


def container_delta_pack(planes, base_crc):
    """rb200_container_delta_pack: a version 8 container from w = len(planes) version 6 containers of the planes of the
    difference d (as container_planes_pack) and the CRC-32 of the base tensor's n bytes"""
    lib = load()
    planes = [np.ascontiguousarray(p, dtype=np.uint8) for p in planes]
    w = len(planes)
    ptrs = (C.c_void_p * max(w, 1))(*[p.ctypes.data for p in planes])
    sizes = (C.c_size_t * max(w, 1))(*[p.size for p in planes])
    out = np.zeros(64 + 16 * w + sum(p.size for p in planes), np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_delta_pack(w, ptrs, sizes, base_crc, out.ctypes.data, out.size, C.byref(size)))
    return out[:size.value]


def container_delta_open(buf):
    """Returns (info dict with base_crc, planes) of a version 8 container: planes[p] is a view into buf of the version 6
    container of plane p of the difference."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerPlanesInfo()
    crc = C.c_uint32(0)
    lib.check(lib.dll.rb200_container_delta_open(buf.ctypes.data, buf.size, C.byref(info), C.byref(crc)))
    base = buf.ctypes.data
    planes = [buf[info.planes[p] - base:info.planes[p] - base + info.sizes[p]] for p in range(info.elem_bytes)]
    meta = {k: int(getattr(info, k)) for k in ("elem_bytes", "chunk_syms", "flags", "n")}
    meta["base_crc"] = int(crc.value)
    return meta, planes


def container_tensors_bound(n_max, count, elem_bytes, chunk_syms):
    """rb200_container_tensors_bound: the most bytes a version 9 container of count tensors of elem_bytes-byte elements,
    n_max bytes in all, takes (0 for arguments the encode refuses)"""
    return int(load().dll.rb200_container_tensors_bound(n_max, count, elem_bytes, chunk_syms))


def container_tensors_pack(lengths, planes):
    """rb200_container_tensors_pack: a version 9 container of a list of tensors with these byte lengths, from the w =
    len(planes) version 6 containers of the byte planes of their concatenated bytes (as container_planes_pack)"""
    lib = load()
    lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
    planes = [np.ascontiguousarray(p, dtype=np.uint8) for p in planes]
    w = len(planes)
    ptrs = (C.c_void_p * max(w, 1))(*[p.ctypes.data for p in planes])
    sizes = (C.c_size_t * max(w, 1))(*[p.size for p in planes])
    out = np.zeros(64 + 16 * w + 8 * lengths.size + 16 + sum(p.size for p in planes), np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_tensors_pack(w, lengths.ctypes.data_as(_u64p), lengths.size, ptrs, sizes, out.ctypes.data,
                                                   out.size, C.byref(size)))
    return out[:size.value]


def container_tensors_open(buf):
    """Returns (info dict, lengths, planes) of a version 9 container: lengths (uint64, one per tensor) and planes[p] (plane
    p's version 6 container) are views into buf."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerPlanesInfo()
    count = C.c_uint32(0)
    dir_ptr = _u64p()
    lib.check(lib.dll.rb200_container_tensors_open(buf.ctypes.data, buf.size, C.byref(info), C.byref(count), C.byref(dir_ptr)))
    base = buf.ctypes.data
    d_off = C.addressof(dir_ptr.contents) - base
    lengths = buf[d_off:d_off + 8 * count.value].view(np.uint64)
    planes = [buf[info.planes[p] - base:info.planes[p] - base + info.sizes[p]] for p in range(info.elem_bytes)]
    meta = {k: int(getattr(info, k)) for k in ("elem_bytes", "chunk_syms", "flags", "n")}
    meta["count"] = int(count.value)
    return meta, lengths, planes


class ContainerBlocksInfo(C.Structure):
    _fields_ = [("n_blocks", C.c_uint32), ("block_size", C.c_uint32), ("chunk_syms", C.c_uint32), ("flags", C.c_uint32),
                ("n_symbols", C.c_uint64), ("n_chunks", C.c_uint64), ("blob_bytes", C.c_uint64),
                ("block_freqs", _u16p), ("offsets", _u64p), ("blob", _u8p)]


def container_blocks_pack(n_blocks, block_size, chunk_syms, block_freqs, offsets, blob, flags=0):
    """rb200_container_blocks_pack: a per-block (version 2) container from the per-block calls' three arrays"""
    lib = load()
    block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    total = int(lib.dll.rb200_container_blocks_size(n_blocks, offsets.size - 1, blob.size))
    out = np.zeros(total, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_blocks_pack(n_blocks, block_size, chunk_syms, block_freqs.ctypes.data, offsets.ctypes.data,
                                                  blob.ctypes.data, blob.size, flags, out.ctypes.data, total, C.byref(size)))
    return out[:size.value]


def container_blocks_open(buf):
    """Returns (info dict, block_freqs [n_blocks, 256], offsets, blob) as numpy views into buf."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerBlocksInfo()
    lib.check(lib.dll.rb200_container_blocks_open(buf.ctypes.data, buf.size, C.byref(info)))
    base = buf.ctypes.data
    f_off = C.addressof(info.block_freqs.contents) - base
    o_off = C.addressof(info.offsets.contents) - base
    b_off = (C.addressof(info.blob.contents) - base) if info.blob_bytes else buf.size
    freqs = buf[f_off:f_off + 512 * info.n_blocks].view(np.uint16).reshape(info.n_blocks, 256)
    offsets = buf[o_off:o_off + 8 * (info.n_chunks + 1)].view(np.uint64)
    blob = buf[b_off:b_off + info.blob_bytes]
    meta = {k: int(getattr(info, k)) for k in ("n_blocks", "block_size", "chunk_syms", "flags", "n_symbols", "n_chunks", "blob_bytes")}
    return meta, freqs, offsets, blob


class ContainerBlocksCoderInfo(C.Structure):
    _fields_ = [("coder", C.c_uint32), ("scale_bits", C.c_uint32), ("n_blocks", C.c_uint32), ("block_size", C.c_uint32),
                ("chunk_syms", C.c_uint32), ("flags", C.c_uint32), ("n_symbols", C.c_uint64), ("n_chunks", C.c_uint64),
                ("blob_bytes", C.c_uint64), ("block_freqs", _u16p), ("offsets", _u64p), ("blob", _u8p)]


def container_blocks_coder_pack(coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs, offsets, blob, flags=0):
    """rb200_container_blocks_coder_pack: a version 3 container (byte or rans64 coder, a model per block)"""
    lib = load()
    block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    total = int(lib.dll.rb200_container_blocks_size(n_blocks, offsets.size - 1, blob.size))
    out = np.zeros(total, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_blocks_coder_pack(coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs.ctypes.data,
                                                        offsets.ctypes.data, blob.ctypes.data, blob.size, flags, out.ctypes.data, total,
                                                        C.byref(size)))
    return out[:size.value]


def container_blocks_alias_pack(scale_bits, n_blocks, block_size, chunk_syms, block_freqs, offsets, blob, flags=0):
    """rb200_container_blocks_alias_pack: a version 4 container (alias coder, a model per block)"""
    lib = load()
    block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    total = int(lib.dll.rb200_container_blocks_size(n_blocks, offsets.size - 1, blob.size))
    out = np.zeros(total, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_blocks_alias_pack(scale_bits, n_blocks, block_size, chunk_syms, block_freqs.ctypes.data,
                                                        offsets.ctypes.data, blob.ctypes.data, blob.size, flags, out.ctypes.data, total,
                                                        C.byref(size)))
    return out[:size.value]


def container_blocks_alias_open(buf):
    """rb200_container_blocks_alias_open: as container_blocks_coder_open, for version 4"""
    return container_blocks_coder_open(buf, _open="rb200_container_blocks_alias_open")


def container_blocks_stored_bound(n_blocks, block_size, chunk_syms):
    """rb200_container_blocks_stored_bound: the most bytes a version 5 container of this geometry takes (0 for a geometry
    the per-block calls refuse)"""
    return int(load().dll.rb200_container_blocks_stored_bound(n_blocks, block_size, chunk_syms))


def container_blocks_stored_pack(coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs, offsets, blob, flags=0):
    """rb200_container_blocks_stored_pack: a version 5 container (any per-block pair; a zero row of block_freqs marks a
    stored block, whose chunks are round16(chunk_syms)-byte streams of their symbols and zero padding)"""
    lib = load()
    block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    total = int(lib.dll.rb200_container_blocks_size(n_blocks, offsets.size - 1, blob.size))
    out = np.zeros(total, np.uint8)
    size = C.c_size_t(0)
    lib.check(lib.dll.rb200_container_blocks_stored_pack(coder, scale_bits, n_blocks, block_size, chunk_syms, block_freqs.ctypes.data,
                                                         offsets.ctypes.data, blob.ctypes.data, blob.size, flags, out.ctypes.data, total,
                                                         C.byref(size)))
    return out[:size.value]


def container_blocks_stored_open(buf):
    """rb200_container_blocks_stored_open: as container_blocks_coder_open, for version 5"""
    return container_blocks_coder_open(buf, _open="rb200_container_blocks_stored_open")


def container_blocks_coder_open(buf, _open="rb200_container_blocks_coder_open"):
    """Returns (info dict, block_freqs [n_blocks, 256], offsets, blob) as numpy views into buf."""
    lib = load()
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    info = ContainerBlocksCoderInfo()
    lib.check(getattr(lib.dll, _open)(buf.ctypes.data, buf.size, C.byref(info)))
    base = buf.ctypes.data
    f_off = C.addressof(info.block_freqs.contents) - base
    o_off = C.addressof(info.offsets.contents) - base
    b_off = (C.addressof(info.blob.contents) - base) if info.blob_bytes else buf.size
    freqs = buf[f_off:f_off + 512 * info.n_blocks].view(np.uint16).reshape(info.n_blocks, 256)
    offsets = buf[o_off:o_off + 8 * (info.n_chunks + 1)].view(np.uint64)
    blob = buf[b_off:b_off + info.blob_bytes]
    meta = {k: int(getattr(info, k)) for k in ("coder", "scale_bits", "n_blocks", "block_size", "chunk_syms", "flags", "n_symbols",
                                               "n_chunks", "blob_bytes")}
    return meta, freqs, offsets, blob


class RansError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"rb200 error {code}: {msg}")
        self.code = code


class Lib:
    def __init__(self, path=LIB_PATH):
        if not os.path.exists(path):
            build()
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing and could not be built; there is no CPU fallback")
        self.path = path
        self.dll = C.CDLL(path)
        for name, res, args in EXPORTS:
            f = getattr(self.dll, name)      # AttributeError if the .so lacks a declared symbol
            f.restype = res
            f.argtypes = args

    def check(self, rc, ctx=None):
        if rc != 0:
            msg = self.dll.rb200_strerror(rc).decode()
            if rc in (-5, -8) and ctx is not None:
                msg += ": " + self.dll.rb200_last_cuda_error(ctx).decode()
            raise RansError(rc, msg)


_LIB = None


def load():
    global _LIB
    if _LIB is None:
        _LIB = Lib()
    return _LIB


def _np_ptr(a):
    return a.ctypes.data


class SymbolStats:
    """Host-side mirror of the reference's SymbolStats (main.cpp:49-57, main_alias.cpp:47-72)."""

    def __init__(self):
        self.freqs = np.zeros(256, np.uint32)
        self.cum_freqs = np.zeros(257, np.uint32)

    def count_freqs(self, data):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        lib = load()
        lib.check(lib.dll.rb200_count_freqs(_np_ptr(data), data.size, self.freqs.ctypes.data_as(_u32p)))
        return self

    def normalize_freqs(self, target_total):
        lib = load()
        lib.check(lib.dll.rb200_normalize_freqs(self.freqs.ctypes.data_as(_u32p), self.cum_freqs.ctypes.data_as(_u32p),
                                                target_total))
        return self

    def word_tables(self):
        slots = np.zeros(4096, np.uint32)
        s2s = np.zeros(4096, np.uint8)
        lib = load()
        lib.check(lib.dll.rb200_word_tables_build(self.freqs.ctypes.data_as(_u32p), self.cum_freqs.ctypes.data_as(_u32p),
                                                  slots.ctypes.data_as(_u32p), s2s.ctypes.data_as(_u8p)))
        return slots, s2s

    def make_alias_table(self):
        self.divider = np.zeros(256, np.uint32)
        self.slot_adjust = np.zeros(512, np.uint32)
        self.slot_freqs = np.zeros(512, np.uint32)
        self.sym_id = np.zeros(512, np.uint8)
        self.alias_remap = np.zeros(int(self.cum_freqs[256]), np.uint32)
        lib = load()
        lib.check(lib.dll.rb200_alias_tables_build(
            self.freqs.ctypes.data_as(_u32p), self.cum_freqs.ctypes.data_as(_u32p), self.divider.ctypes.data_as(_u32p),
            self.slot_adjust.ctypes.data_as(_u32p), self.slot_freqs.ctypes.data_as(_u32p),
            self.sym_id.ctypes.data_as(_u8p), self.alias_remap.ctypes.data_as(_u32p)))
        return self


class Context:
    def __init__(self, device=0, stream=0):
        self.lib = load()
        h = C.c_void_p()
        self.lib.check(self.lib.dll.rb200_ctx_create(C.byref(h), device, C.c_void_p(stream or 0)))
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.dll.rb200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, stream):
        self.lib.check(self.lib.dll.rb200_ctx_set_stream(self.h, C.c_void_p(stream or 0)))

    def sync(self):
        self.lib.check(self.lib.dll.rb200_sync(self.h), self.h)

    @property
    def launches(self):
        return int(self.lib.dll.rb200_launch_count(self.h))

    def model(self, coder, scale_bits, freqs):
        return Model(self, coder, scale_bits, freqs)

    # ---- geometry
    def chunk_count(self, n, chunk_syms):
        return int(self.lib.dll.rb200_chunk_count(n, chunk_syms))

    def encode_bound(self, n, chunk_syms):
        return int(self.lib.dll.rb200_encode_bound(n, chunk_syms))

    # ---- host-buffer calls (numpy in / numpy out)
    def encode_host(self, model, data, chunk_syms, blob_cap=None):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        n_chunks = self.chunk_count(data.size, chunk_syms)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_chunks + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_encode(self.h, model.h, _np_ptr(data), data.size, chunk_syms, _np_ptr(blob), cap,
                                                 _np_ptr(offsets), C.byref(size), MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets

    def decode_host(self, model, blob, offsets, n, chunk_syms):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        out = np.zeros(max(n, 1), np.uint8)
        self.lib.check(self.lib.dll.rb200_decode(self.h, model.h, _np_ptr(blob), blob.size, _np_ptr(offsets), chunk_syms,
                                                 _np_ptr(out), n, MEM_HOST), self.h)
        return out[:n]

    # ---- device-pointer calls (integers = device addresses); asynchronous
    def encode_device(self, model, in_ptr, n, chunk_syms, blob_ptr, blob_cap, offsets_ptr):
        self.lib.check(self.lib.dll.rb200_encode(self.h, model.h, in_ptr, n, chunk_syms, blob_ptr, blob_cap, offsets_ptr,
                                                 None, MEM_DEVICE), self.h)

    def decode_device(self, model, blob_ptr, blob_size, offsets_ptr, chunk_syms, out_ptr, n):
        self.lib.check(self.lib.dll.rb200_decode(self.h, model.h, blob_ptr, blob_size, offsets_ptr, chunk_syms, out_ptr, n,
                                                 MEM_DEVICE), self.h)

    def histogram(self, data):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        counts = np.zeros(256, np.uint64)
        self.lib.check(self.lib.dll.rb200_histogram(self.h, _np_ptr(data), data.size, counts.ctypes.data_as(_u64p), MEM_HOST),
                       self.h)
        return counts

    def histogram_device(self, ptr, n):
        counts = np.zeros(256, np.uint64)
        self.lib.check(self.lib.dll.rb200_histogram(self.h, ptr, n, counts.ctypes.data_as(_u64p), MEM_DEVICE), self.h)
        return counts

    # ---- CRC-32 and the container in host or device memory
    def crc32(self, data, crc_in=0):
        """zlib.crc32 of a host array, computed on the GPU."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        out = C.c_uint32(0)
        self.lib.check(self.lib.dll.rb200_crc32(self.h, _np_ptr(data), data.size, crc_in, C.byref(out), MEM_HOST), self.h)
        return out.value

    def crc32_device(self, ptr, n, crc_in=0):
        out = C.c_uint32(0)
        self.lib.check(self.lib.dll.rb200_crc32(self.h, ptr, n, crc_in, C.byref(out), MEM_DEVICE), self.h)
        return out.value

    def container_capacity(self, n, chunk_syms):
        """bytes that always hold rb200_container_encode's output for n symbols"""
        return int(self.lib.dll.rb200_container_size(self.chunk_count(n, chunk_syms), self.encode_bound(n, chunk_syms)))

    def container_encode_host(self, model, data, chunk_syms, flags=0, out_cap=None):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        cap = self.container_capacity(data.size, chunk_syms) if out_cap is None else out_cap
        out = np.zeros(max(cap, 16), np.uint8)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_container_encode(self.h, model.h, _np_ptr(data), data.size, chunk_syms, flags, _np_ptr(out),
                                                           cap, C.byref(size), MEM_HOST), self.h)
        return out[:size.value].copy()

    def container_encode_device(self, model, in_ptr, n, chunk_syms, flags, out_ptr, out_cap):
        """asynchronous; errors come from sync()"""
        self.lib.check(self.lib.dll.rb200_container_encode(self.h, model.h, in_ptr, n, chunk_syms, flags, out_ptr, out_cap, None,
                                                           MEM_DEVICE), self.h)

    def container_decode_host(self, buf, out_cap=None):
        """returns the decoded symbols; out_cap defaults to the container's n"""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        n = C.c_uint64(0)
        if out_cap is None:
            rc = self.lib.dll.rb200_container_decode(self.h, _np_ptr(buf), buf.size, None, 0, C.byref(n), MEM_HOST)
            if rc not in (0, -3):
                self.lib.check(rc, self.h)
            out_cap = n.value
        out = np.zeros(max(out_cap, 1), np.uint8)
        self.lib.check(self.lib.dll.rb200_container_decode(self.h, _np_ptr(buf), buf.size, _np_ptr(out), out_cap, C.byref(n),
                                                           MEM_HOST), self.h)
        return out[:n.value]

    def container_decode_device(self, buf_ptr, size, out_ptr, out_cap):
        """synchronous; returns the container's n"""
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rb200_container_decode(self.h, buf_ptr, size, out_ptr, out_cap, C.byref(n), MEM_DEVICE), self.h)
        return n.value

    def container_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable), any coder; n_ptr: device address of a u64 that receives n, or 0.  The
        verdict on the container (-4 corrupt or not decodable, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None), self.h)

    def container_model_encode_async(self, coder, scale_bits, in_ptr, n, chunk_syms, flags, out_ptr, out_cap):
        """enqueue only (CUDA-graph capturable once a call of the same geometry has grown the workspace): the model built
        from the data on the GPU, then the container, as Model.from_data + container_encode_device.  The verdict (-2 a
        model rb200_model_create refuses, -3 out_cap too small for the blob, header unwritten) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_model_encode_async(self.h, coder, scale_bits, in_ptr, n, chunk_syms, flags, out_ptr,
                                                                       out_cap), self.h)

    def container_model_encode_varlen_async(self, coder, scale_bits, in_ptr, n_ptr, n_max, chunk_syms, flags, out_ptr, out_cap):
        """container_model_encode_async with the length read from device memory when the work runs: n_ptr is the device
        address of a u64 n, 1 <= n <= n_max.  n_max fixes the launch shapes and the workspace, so one captured call serves
        every such n.  The verdict (-2 for n == 0, -1 for n > n_max, both with out untouched; otherwise as
        container_model_encode_async) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_model_encode_varlen_async(self.h, coder, scale_bits, in_ptr, n_ptr, n_max, chunk_syms,
                                                                              flags, out_ptr, out_cap), self.h)

    def container_model_encode_auto_async(self, candidates, tolerance_ppm, in_ptr, n, chunk_syms, flags, out_ptr, out_cap, n_ptr=0):
        """container_model_encode_async with (coder, scale_bits) chosen on the GPU from the data at every run, by the
        rule of choose_coder over `candidates` (CANDIDATE values, in order of preference).  n_ptr: the device address of
        a u64 length read when the work runs, with n its bound n_max (as container_model_encode_varlen_async), or 0.
        The header records the choice.  The verdict (-2 when no candidate is feasible, otherwise as the fixed call for
        the chosen pair) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_model_encode_auto_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                            in_ptr, n_ptr or None, n, chunk_syms, flags, out_ptr, out_cap),
                       self.h)

    def container_stored_encode_async(self, candidates, tolerance_ppm, in_ptr, n, chunk_syms, flags, out_ptr, out_cap):
        """container_model_encode_auto_async's choice, model and (split) encoders, then every chunk whose stream is
        longer than its symbols is stored: a version 6 container of at most container_stored_bound bytes.  The verdict
        (-2 when no candidate is feasible, -3 when the blob does not fit, header unwritten) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_stored_encode_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                        in_ptr, n, chunk_syms, flags, out_ptr, out_cap), self.h)

    def container_stored_encode_varlen_async(self, candidates, tolerance_ppm, in_ptr, n_ptr, n_max, chunk_syms, flags, out_ptr, out_cap):
        """container_stored_encode_async with the length read from device memory when the work runs: n_ptr is the device
        address of a u64 n, 1 <= n <= n_max.  n_max fixes the launch shapes and the workspace, so one captured call serves
        every such n, and out_cap = container_stored_bound(n_max, chunk_syms) holds every one.  The verdict (-2 for n == 0,
        -1 for n > n_max, both with out untouched; otherwise as container_stored_encode_async) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_stored_encode_varlen_async(self.h, cands.ctypes.data_as(_u32p), cands.size,
                                                                               tolerance_ppm, in_ptr, n_ptr, n_max, chunk_syms, flags,
                                                                               out_ptr, out_cap), self.h)

    def container_planes_encode_async(self, candidates, tolerance_ppm, elem_bytes, in_ptr, n, chunk_syms, flags, out_ptr, out_cap):
        """A version 7 container of n bytes of elem_bytes-byte elements (2, 4 or 8): byte plane p of every element is a
        version 6 container, byte for byte what container_stored_encode_async writes for it.  out_cap >=
        container_planes_bound.  The verdict (the first failing plane's, header unwritten) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_planes_encode_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                        elem_bytes, in_ptr, n, chunk_syms, flags, out_ptr, out_cap), self.h)

    def container_planes_encode_varlen_async(self, candidates, tolerance_ppm, elem_bytes, in_ptr, n_ptr, n_max, chunk_syms, flags, out_ptr,
                                             out_cap):
        """container_planes_encode_async with the length in bytes read from device memory when the work runs: n_ptr is
        the device address of a u64 n, 1 <= n <= n_max and a multiple of elem_bytes.  n_max fixes the launch shapes and
        the workspaces, so one captured call serves every such n, and out_cap = container_planes_bound(n_max,
        elem_bytes, chunk_syms) holds every one (never -3 from sync()).  The verdict comes from sync(): -1 for an n of
        0, not a multiple of elem_bytes or above n_max, with out untouched; otherwise container_planes_encode_async's
        (the first failing plane's, header unwritten)"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_planes_encode_varlen_async(self.h, cands.ctypes.data_as(_u32p), cands.size,
                                                                               tolerance_ppm, elem_bytes, in_ptr, n_ptr, n_max, chunk_syms,
                                                                               flags, out_ptr, out_cap), self.h)

    def container_planes_decode_async(self, elem_bytes, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable once a call of the same size and out_cap has grown the workspaces): a
        version 7 container of elem_bytes-byte elements.  The verdict (-4 corrupt, -3 out_cap too small, output
        untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_planes_decode_async(self.h, elem_bytes, buf_ptr, size, out_ptr, out_cap, n_ptr or None),
                       self.h)

    def container_delta_encode_async(self, candidates, tolerance_ppm, elem_bytes, in_ptr, base_ptr, n, chunk_syms, flags, out_ptr,
                                     out_cap):
        """A version 8 container of the n bytes at in_ptr as their difference from the n bytes at base_ptr (both 16-byte
        aligned): container_planes_encode_async of the zigzag difference, with the base's CRC in the header.  out_cap >=
        container_planes_bound.  The verdict (the first failing plane's, header unwritten) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_delta_encode_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                       elem_bytes, in_ptr, base_ptr, n, chunk_syms, flags, out_ptr,
                                                                       out_cap), self.h)

    def container_delta_decode_async(self, elem_bytes, buf_ptr, size, base_ptr, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable once a call of the same size and out_cap has grown the workspaces): a
        version 8 container applied to the base at base_ptr, into out_ptr; out_ptr == base_ptr applies it in place, any
        other overlap is -1.  The verdict (-4 corrupt, -3 out_cap too small, -10 a base with another CRC; out untouched
        in every case) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_delta_decode_async(self.h, elem_bytes, buf_ptr, size, base_ptr, out_ptr, out_cap,
                                                                       n_ptr or None), self.h)

    def container_tensors_encode_async(self, candidates, tolerance_ppm, elem_bytes, refs_ptr, count, n_max, chunk_syms, flags, out_ptr,
                                       out_cap):
        """A version 9 container of the count tensors named by the rb200_tensor_ref list at refs_ptr (device memory, 16
        bytes per entry {u64 ptr, u64 bytes}, 16-byte aligned), read when the work runs: each bytes a multiple of
        elem_bytes, each ptr aligned to elem_bytes, the total 1 .. n_max.  out_cap >= container_tensors_bound(n_max, count,
        elem_bytes, chunk_syms).  The verdict comes from sync(): -1 for a bad list, with out untouched; otherwise
        container_planes_encode_async's of the concatenated bytes (the first failing plane's, header unwritten)"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_tensors_encode_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                         elem_bytes, refs_ptr, count, n_max, chunk_syms, flags, out_ptr,
                                                                         out_cap), self.h)

    def container_tensors_decode_async(self, elem_bytes, buf_ptr, size, refs_ptr, count, n_max, lengths_ptr=0):
        """enqueue only (CUDA-graph capturable once a call of the same size, count and n_max has grown the workspaces): a
        version 9 container of count tensors into the outputs of the rb200_tensor_ref list at refs_ptr (device memory:
        each entry's ptr and capacity in bytes).  lengths_ptr (device, count u64, or 0) receives the directory.  The
        verdict (-4 corrupt or another count, -3 a length above its capacity or a total above n_max; every output
        untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_tensors_decode_async(self.h, elem_bytes, buf_ptr, size, refs_ptr, count, n_max,
                                                                         lengths_ptr or None), self.h)

    def container_stored_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """the async decode of a version 6 container; enqueue only (CUDA-graph capturable).  The verdict (-4 corrupt or
        another version, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_stored_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None), self.h)

    # ---- per-block containers (version 2): every block's model, the directory and the blob in one buffer
    def container_blocks_capacity(self, n_blocks, block_size, chunk_syms):
        """bytes that always hold rb200_container_blocks_encode's output"""
        n = n_blocks * block_size
        return int(self.lib.dll.rb200_container_blocks_size(n_blocks, n // chunk_syms, self.encode_bound(n, chunk_syms)))

    def container_blocks_encode_host(self, data, n_blocks, block_size, chunk_syms, block_freqs=None, flags=0, out_cap=None):
        """block_freqs None: the models are built on the GPU; else the caller's [n_blocks, 256] u16 tables"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = None if block_freqs is None else np.ascontiguousarray(block_freqs, dtype=np.uint16)
        cap = self.container_blocks_capacity(n_blocks, block_size, chunk_syms) if out_cap is None else out_cap
        out = np.zeros(max(cap, 16), np.uint8)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_encode(self.h, _np_ptr(data), n_blocks, block_size,
                                                                  None if freqs is None else _np_ptr(freqs), chunk_syms, flags,
                                                                  _np_ptr(out), cap, C.byref(size), MEM_HOST), self.h)
        return out[:size.value].copy()

    def container_blocks_encode_device(self, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, flags, out_ptr, out_cap):
        """asynchronous; freqs_ptr None builds the models; errors come from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_encode(self.h, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, flags,
                                                                  out_ptr, out_cap, None, MEM_DEVICE), self.h)

    def container_blocks_decode_host(self, buf, out_cap=None):
        """returns the decoded symbols; out_cap defaults to the container's n"""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        n = C.c_uint64(0)
        if out_cap is None:
            rc = self.lib.dll.rb200_container_blocks_decode(self.h, _np_ptr(buf), buf.size, None, 0, C.byref(n), MEM_HOST)
            if rc not in (0, -3):
                self.lib.check(rc, self.h)
            out_cap = n.value
        out = np.zeros(max(out_cap, 1), np.uint8)
        self.lib.check(self.lib.dll.rb200_container_blocks_decode(self.h, _np_ptr(buf), buf.size, _np_ptr(out), out_cap, C.byref(n),
                                                                  MEM_HOST), self.h)
        return out[:n.value]

    def container_blocks_decode_device(self, buf_ptr, size, out_ptr, out_cap):
        """synchronous; returns the container's n"""
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_decode(self.h, buf_ptr, size, out_ptr, out_cap, C.byref(n), MEM_DEVICE),
                       self.h)
        return n.value

    def container_blocks_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable); n_ptr: device address of a u64 that receives n, or 0.  The verdict on
        the container (-4 corrupt, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None),
                       self.h)

    # ---- per-block containers of the byte and rans64 coders (version 3)
    def container_blocks_coder_encode_host(self, coder, scale_bits, data, n_blocks, block_size, chunk_syms, block_freqs=None, flags=0,
                                           out_cap=None):
        """block_freqs None: the models (normalised to 1 << scale_bits) are built on the GPU; else the caller's tables"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = None if block_freqs is None else np.ascontiguousarray(block_freqs, dtype=np.uint16)
        cap = self.container_blocks_capacity(n_blocks, block_size, chunk_syms) if out_cap is None else out_cap
        out = np.zeros(max(cap, 16), np.uint8)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_coder_encode(self.h, coder, scale_bits, _np_ptr(data), n_blocks, block_size,
                                                                        None if freqs is None else _np_ptr(freqs), chunk_syms, flags,
                                                                        _np_ptr(out), cap, C.byref(size), MEM_HOST), self.h)
        return out[:size.value].copy()

    def container_blocks_coder_encode_device(self, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, flags, out_ptr,
                                             out_cap):
        """asynchronous; freqs_ptr None builds the models; errors come from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_coder_encode(self.h, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr,
                                                                        chunk_syms, flags, out_ptr, out_cap, None, MEM_DEVICE), self.h)

    def container_blocks_coder_decode_host(self, buf, out_cap=None):
        """returns the decoded symbols; out_cap defaults to the container's n"""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        n = C.c_uint64(0)
        if out_cap is None:
            rc = self.lib.dll.rb200_container_blocks_coder_decode(self.h, _np_ptr(buf), buf.size, None, 0, C.byref(n), MEM_HOST)
            if rc not in (0, -3):
                self.lib.check(rc, self.h)
            out_cap = n.value
        out = np.zeros(max(out_cap, 1), np.uint8)
        self.lib.check(self.lib.dll.rb200_container_blocks_coder_decode(self.h, _np_ptr(buf), buf.size, _np_ptr(out), out_cap, C.byref(n),
                                                                        MEM_HOST), self.h)
        return out[:n.value]

    def container_blocks_coder_decode_device(self, buf_ptr, size, out_ptr, out_cap):
        """synchronous; returns the container's n"""
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_coder_decode(self.h, buf_ptr, size, out_ptr, out_cap, C.byref(n), MEM_DEVICE),
                       self.h)
        return n.value

    def container_blocks_coder_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable); n_ptr: device address of a u64 that receives n, or 0.  The verdict on
        the container (-4 corrupt, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_coder_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None),
                       self.h)

    # ---- per-block models of the byte and rans64 coders (scale_bits 8..15)
    def blocks_coder_encode_device(self, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap,
                                   offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_coder_encode(self.h, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms,
                                                              blob_ptr, blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_coder_model_encode_device(self, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap,
                                         offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_coder_model_encode(self.h, coder, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr,
                                                                    chunk_syms, blob_ptr, blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_coder_decode_device(self, coder, scale_bits, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks, block_size, chunk_syms,
                                   out_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_coder_decode(self.h, coder, scale_bits, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks,
                                                              block_size, chunk_syms, out_ptr, MEM_DEVICE), self.h)

    def blocks_coder_encode_host(self, coder, scale_bits, data, n_blocks, block_size, block_freqs, chunk_syms, blob_cap=None):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_blocks * (block_size // chunk_syms) + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_coder_encode(self.h, coder, scale_bits, _np_ptr(data), n_blocks, block_size,
                                                              _np_ptr(block_freqs), chunk_syms, _np_ptr(blob), cap, _np_ptr(offsets),
                                                              C.byref(size), MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets

    def blocks_coder_model_encode_host(self, coder, scale_bits, data, n_blocks, block_size, chunk_syms, blob_cap=None):
        """models + encode in one call; returns (blob, offsets, block_freqs)"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = np.zeros((n_blocks, 256), np.uint16)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_blocks * (block_size // chunk_syms) + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_coder_model_encode(self.h, coder, scale_bits, _np_ptr(data), n_blocks, block_size,
                                                                    _np_ptr(freqs), chunk_syms, _np_ptr(blob), cap, _np_ptr(offsets),
                                                                    C.byref(size), MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets, freqs

    def blocks_coder_decode_host(self, coder, scale_bits, blob, offsets, block_freqs, n_blocks, block_size, chunk_syms):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        out = np.zeros(n_blocks * block_size, np.uint8)
        self.lib.check(self.lib.dll.rb200_blocks_coder_decode(self.h, coder, scale_bits, _np_ptr(blob), blob.size, _np_ptr(offsets),
                                                              _np_ptr(block_freqs), n_blocks, block_size, chunk_syms, _np_ptr(out),
                                                              MEM_HOST), self.h)
        return out

    # ---- per-block models of the alias coder (scale_bits 8..15) and their container (version 4)
    def blocks_alias_encode_device(self, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap, offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_alias_encode(self.h, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms,
                                                              blob_ptr, blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_alias_model_encode_device(self, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap,
                                         offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_alias_model_encode(self.h, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr,
                                                                    chunk_syms, blob_ptr, blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_alias_decode_device(self, scale_bits, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks, block_size, chunk_syms, out_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_alias_decode(self.h, scale_bits, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks,
                                                              block_size, chunk_syms, out_ptr, MEM_DEVICE), self.h)

    def blocks_alias_encode_host(self, scale_bits, data, n_blocks, block_size, block_freqs, chunk_syms, blob_cap=None):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_blocks * (block_size // chunk_syms) + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_alias_encode(self.h, scale_bits, _np_ptr(data), n_blocks, block_size, _np_ptr(block_freqs),
                                                              chunk_syms, _np_ptr(blob), cap, _np_ptr(offsets), C.byref(size), MEM_HOST),
                       self.h)
        return blob[:size.value].copy(), offsets

    def blocks_alias_model_encode_host(self, scale_bits, data, n_blocks, block_size, chunk_syms, blob_cap=None):
        """models + encode in one call; returns (blob, offsets, block_freqs)"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = np.zeros((n_blocks, 256), np.uint16)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_blocks * (block_size // chunk_syms) + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_alias_model_encode(self.h, scale_bits, _np_ptr(data), n_blocks, block_size, _np_ptr(freqs),
                                                                    chunk_syms, _np_ptr(blob), cap, _np_ptr(offsets), C.byref(size),
                                                                    MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets, freqs

    def blocks_alias_decode_host(self, scale_bits, blob, offsets, block_freqs, n_blocks, block_size, chunk_syms):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        out = np.zeros(n_blocks * block_size, np.uint8)
        self.lib.check(self.lib.dll.rb200_blocks_alias_decode(self.h, scale_bits, _np_ptr(blob), blob.size, _np_ptr(offsets),
                                                              _np_ptr(block_freqs), n_blocks, block_size, chunk_syms, _np_ptr(out), MEM_HOST),
                       self.h)
        return out

    def container_blocks_alias_encode_host(self, scale_bits, data, n_blocks, block_size, chunk_syms, block_freqs=None, flags=0, out_cap=None):
        """block_freqs None: the models (normalised to 1 << scale_bits) are built on the GPU; else the caller's tables"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = None if block_freqs is None else np.ascontiguousarray(block_freqs, dtype=np.uint16)
        cap = self.container_blocks_capacity(n_blocks, block_size, chunk_syms) if out_cap is None else out_cap
        out = np.zeros(max(cap, 16), np.uint8)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_alias_encode(self.h, scale_bits, _np_ptr(data), n_blocks, block_size,
                                                                        None if freqs is None else _np_ptr(freqs), chunk_syms, flags,
                                                                        _np_ptr(out), cap, C.byref(size), MEM_HOST), self.h)
        return out[:size.value].copy()

    def container_blocks_alias_encode_device(self, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, flags, out_ptr, out_cap):
        """asynchronous; freqs_ptr None builds the models; errors come from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_alias_encode(self.h, scale_bits, in_ptr, n_blocks, block_size, freqs_ptr,
                                                                        chunk_syms, flags, out_ptr, out_cap, None, MEM_DEVICE), self.h)

    def container_blocks_alias_decode_host(self, buf, out_cap=None):
        """returns the decoded symbols; out_cap defaults to the container's n"""
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        n = C.c_uint64(0)
        if out_cap is None:
            rc = self.lib.dll.rb200_container_blocks_alias_decode(self.h, _np_ptr(buf), buf.size, None, 0, C.byref(n), MEM_HOST)
            if rc not in (0, -3):
                self.lib.check(rc, self.h)
            out_cap = n.value
        out = np.zeros(max(out_cap, 1), np.uint8)
        self.lib.check(self.lib.dll.rb200_container_blocks_alias_decode(self.h, _np_ptr(buf), buf.size, _np_ptr(out), out_cap, C.byref(n),
                                                                        MEM_HOST), self.h)
        return out[:n.value]

    def container_blocks_alias_decode_device(self, buf_ptr, size, out_ptr, out_cap):
        """synchronous; returns the container's n"""
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rb200_container_blocks_alias_decode(self.h, buf_ptr, size, out_ptr, out_cap, C.byref(n), MEM_DEVICE),
                       self.h)
        return n.value

    def container_blocks_model_encode_auto_async(self, candidates, tolerance_ppm, in_ptr, n_blocks, block_size, chunk_syms, flags, out_ptr,
                                                 out_cap):
        """the per-block container encode (DEVICE, models built) with (coder, scale_bits) chosen on the GPU from the blocks
        at every run, by the rule of choose_blocks_coder over `candidates`: a version 2, 3 or 4 container, byte for byte
        the fixed call's for the chosen pair.  The verdict (-3 when the chosen blob does not fit, header unwritten) comes
        from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_blocks_model_encode_auto_async(self.h, cands.ctypes.data_as(_u32p), cands.size,
                                                                                   tolerance_ppm, in_ptr, n_blocks, block_size, chunk_syms,
                                                                                   flags, out_ptr, out_cap), self.h)

    def container_blocks_model_encode_varlen_async(self, candidates, tolerance_ppm, in_ptr, n_blocks_ptr, n_blocks_max, block_size, chunk_syms,
                                                   flags, out_ptr, out_cap):
        """container_blocks_model_encode_auto_async with the block count read from device memory when the work runs:
        n_blocks_ptr is the device address of a u32 count, 1 <= count <= n_blocks_max.  n_blocks_max fixes the launch
        shapes and the workspace, so one captured call serves every such count; out_cap =
        container_blocks_capacity(n_blocks_max, ...) holds every one.  With one candidate no choice kernel runs and
        container_blocks_auto_costs is undefined after it.  The verdict (-1 for a count of 0 or above n_blocks_max, with
        out untouched; otherwise as the fixed call) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_blocks_model_encode_varlen_async(self.h, cands.ctypes.data_as(_u32p), cands.size,
                                                                                     tolerance_ppm, in_ptr, n_blocks_ptr, n_blocks_max,
                                                                                     block_size, chunk_syms, flags, out_ptr, out_cap), self.h)

    def container_blocks_auto_costs(self, n):
        """the n candidate costs of the last container_blocks_model_encode_auto_async run (synchronises)"""
        costs = np.zeros(max(n, 1), np.uint64)
        self.lib.check(self.lib.dll.rb200_container_blocks_auto_costs(self.h, costs.ctypes.data_as(_u64p), n), self.h)
        return costs[:n]

    def container_blocks_any_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """the async decode of a per-block container of version 2, 3 or 4, whichever the header names; enqueue only
        (CUDA-graph capturable).  The verdict (-4 corrupt or another version, -3 out_cap too small, output untouched)
        comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_any_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None), self.h)

    def container_blocks_stored_encode_async(self, candidates, tolerance_ppm, in_ptr, n_blocks, block_size, chunk_syms, flags, out_ptr,
                                             out_cap):
        """container_blocks_model_encode_auto_async's choice and encoders, then every block whose coded chunks take more
        than its stored size is stored: a version 5 container of at most container_blocks_stored_bound bytes.  The
        verdict (-3 when the blob does not fit, header unwritten) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_blocks_stored_encode_async(self.h, cands.ctypes.data_as(_u32p), cands.size, tolerance_ppm,
                                                                               in_ptr, n_blocks, block_size, chunk_syms, flags, out_ptr,
                                                                               out_cap), self.h)

    def container_blocks_stored_encode_varlen_async(self, candidates, tolerance_ppm, in_ptr, n_blocks_ptr, n_blocks_max, block_size,
                                                    chunk_syms, flags, out_ptr, out_cap):
        """container_blocks_stored_encode_async with the block count read from device memory when the work runs:
        n_blocks_ptr is the device address of a u32 count, 1 <= count <= n_blocks_max.  n_blocks_max fixes the launch
        shapes and the workspace, so one captured call serves every such count, and out_cap =
        container_blocks_stored_bound(n_blocks_max, ...) holds every one.  The verdict (-1 for a count of 0 or above
        n_blocks_max, with out untouched; otherwise as container_blocks_stored_encode_async) comes from sync()"""
        cands = _candidates(candidates)
        self.lib.check(self.lib.dll.rb200_container_blocks_stored_encode_varlen_async(self.h, cands.ctypes.data_as(_u32p), cands.size,
                                                                                      tolerance_ppm, in_ptr, n_blocks_ptr, n_blocks_max,
                                                                                      block_size, chunk_syms, flags, out_ptr, out_cap),
                       self.h)

    def container_blocks_stored_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """the async decode of a version 5 container; enqueue only (CUDA-graph capturable).  The verdict (-4 corrupt or
        another version, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_stored_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None),
                       self.h)

    def container_blocks_alias_decode_async(self, buf_ptr, size, out_ptr, out_cap, n_ptr=0):
        """enqueue only (CUDA-graph capturable); n_ptr: device address of a u64 that receives n, or 0.  The verdict on
        the container (-4 corrupt, -3 out_cap too small, output untouched) comes from sync()"""
        self.lib.check(self.lib.dll.rb200_container_blocks_alias_decode_async(self.h, buf_ptr, size, out_ptr, out_cap, n_ptr or None),
                       self.h)

    # ---- per-block models, device pointers (asynchronous)
    def blocks_build_models_device(self, in_ptr, n_blocks, block_size, freqs_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_build_models(self.h, in_ptr, n_blocks, block_size, freqs_ptr, MEM_DEVICE), self.h)

    def blocks_encode_device(self, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap, offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_encode(self.h, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr,
                                                        blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_model_encode_device(self, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr, blob_cap, offsets_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_model_encode(self.h, in_ptr, n_blocks, block_size, freqs_ptr, chunk_syms, blob_ptr,
                                                              blob_cap, offsets_ptr, None, MEM_DEVICE), self.h)

    def blocks_decode_device(self, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks, block_size, chunk_syms, out_ptr):
        self.lib.check(self.lib.dll.rb200_blocks_decode(self.h, blob_ptr, blob_size, offsets_ptr, freqs_ptr, n_blocks, block_size,
                                                        chunk_syms, out_ptr, MEM_DEVICE), self.h)

    # ---- per-block models, host buffers
    def blocks_build_models(self, data, n_blocks, block_size):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = np.zeros((n_blocks, 256), np.uint16)
        self.lib.check(self.lib.dll.rb200_blocks_build_models(self.h, _np_ptr(data), n_blocks, block_size, _np_ptr(freqs),
                                                              MEM_HOST), self.h)
        return freqs

    def blocks_encode_host(self, data, n_blocks, block_size, block_freqs, chunk_syms, blob_cap=None):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        n_chunks = n_blocks * (block_size // chunk_syms)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_chunks + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_encode(self.h, _np_ptr(data), n_blocks, block_size, _np_ptr(block_freqs),
                                                        chunk_syms, _np_ptr(blob), cap, _np_ptr(offsets), C.byref(size),
                                                        MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets

    def blocks_model_encode_host(self, data, n_blocks, block_size, chunk_syms, blob_cap=None):
        """models + encode in one call; returns (blob, offsets, block_freqs)"""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        freqs = np.zeros((n_blocks, 256), np.uint16)
        n_chunks = n_blocks * (block_size // chunk_syms)
        cap = self.encode_bound(data.size, chunk_syms) if blob_cap is None else blob_cap
        blob = np.zeros(max(cap, 16), np.uint8)
        offsets = np.zeros(n_chunks + 1, np.uint64)
        size = C.c_size_t(0)
        self.lib.check(self.lib.dll.rb200_blocks_model_encode(self.h, _np_ptr(data), n_blocks, block_size, _np_ptr(freqs), chunk_syms,
                                                              _np_ptr(blob), cap, _np_ptr(offsets), C.byref(size), MEM_HOST), self.h)
        return blob[:size.value].copy(), offsets, freqs

    def blocks_decode_host(self, blob, offsets, block_freqs, n_blocks, block_size, chunk_syms):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        block_freqs = np.ascontiguousarray(block_freqs, dtype=np.uint16)
        out = np.zeros(n_blocks * block_size, np.uint8)
        self.lib.check(self.lib.dll.rb200_blocks_decode(self.h, _np_ptr(blob), blob.size, _np_ptr(offsets),
                                                        _np_ptr(block_freqs), n_blocks, block_size, chunk_syms, _np_ptr(out),
                                                        MEM_HOST), self.h)
        return out


class Model:
    def __init__(self, ctx, coder, scale_bits, freqs, _handle=None):
        self.ctx = ctx
        self.coder = coder
        self.scale_bits = scale_bits
        freqs = np.ascontiguousarray(freqs, dtype=np.uint32)
        assert freqs.size == 256
        self.freqs = freqs
        if _handle is not None:
            self.h = _handle
            return
        h = C.c_void_p()
        ctx.lib.check(ctx.lib.dll.rb200_model_create(ctx.h, coder, scale_bits, freqs.ctypes.data_as(_u32p), C.byref(h)), ctx.h)
        self.h = h

    @classmethod
    def from_data(cls, ctx, coder, scale_bits, data=None, device_ptr=None, n=None):
        """rb200_model_from_data: histogram on the GPU + the reference's normalize_freqs + tables.  Pass a host
        array as `data`, or `device_ptr` + `n` for symbols that already live on the device."""
        freqs = np.zeros(256, np.uint32)
        h = C.c_void_p()
        if device_ptr is None:
            data = np.ascontiguousarray(data, dtype=np.uint8)
            ptr, n, kind = _np_ptr(data), data.size, MEM_HOST
        else:
            ptr, kind = device_ptr, MEM_DEVICE
        ctx.lib.check(ctx.lib.dll.rb200_model_from_data(ctx.h, coder, scale_bits, ptr, n, kind, freqs.ctypes.data_as(_u32p),
                                                        C.byref(h)), ctx.h)
        return cls(ctx, coder, scale_bits, freqs, _handle=h)

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx.lib.dll.rb200_model_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

"""block_alias_tables and block_alias_remap, the CTA-parallel make_alias_table (main_alias.cpp:147-237) of the per-block
alias kernels, against the host builder rb200_alias_tables_build (alias_tables_core) entry for entry: divider,
slot_adjust, slot_freqs, sym_id and every slot of alias_remap, for every table of the crafted corpus of
test_model_builders_on_gpu.py at scale_bits 8..15, at 128, 256 and 1024 threads.

tests/alias_device/pairing.cu is compiled here with the library's nvcc flags; it calls the shipped device functions
from a one-CTA-per-model kernel.  A stream reads only the entries its symbols visit, so the stream tests of
test_gpu_blocks_alias.py cannot see a wrong entry elsewhere."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import ryg_rans_b200 as rb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_model_builders_on_gpu as mb  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pd(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from ryg_rans_b200.build import NVCC_FLAGS, _nvcc
    out = str(tmp_path_factory.mktemp("alias_device") / "libpairing.so")
    subprocess.check_call([_nvcc(), *NVCC_FLAGS, "-shared", "-o", out, os.path.join(ROOT, "tests", "alias_device", "pairing.cu")])
    dll = C.CDLL(out)
    dll.pd_alias_tables.restype = C.c_int
    dll.pd_alias_tables.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    return dll


@pytest.fixture(scope="module")
def host_build():
    """rb200_alias_tables_build of the library, taking array addresses"""
    fn = C.CDLL(rb.LIB_PATH).rb200_alias_tables_build
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p] * 7
    return fn


def host_tables(fn, f, sb):
    """rb200_alias_tables_build: (rc, divider, slot_adjust, slot_freqs, sym_id, remap as u16)"""
    f = np.ascontiguousarray(f, dtype=np.uint32)
    cum = np.concatenate([[0], np.cumsum(f)]).astype(np.uint32)
    div, adj, sf = np.zeros(256, np.uint32), np.zeros(512, np.uint32), np.zeros(512, np.uint32)
    sym, remap = np.zeros(512, np.uint8), np.zeros(1 << sb, np.uint32)
    rc = fn(f.ctypes.data, cum.ctypes.data, div.ctypes.data, adj.ctypes.data, sf.ctypes.data, sym.ctypes.data, remap.ctypes.data)
    return rc, div, adj, sf, sym, remap.astype(np.uint16)


@pytest.mark.parametrize("threads", [128, 256, 1024])
@pytest.mark.parametrize("sb", list(range(8, 16)))
def test_block_alias_tables_equal_host_builder(pd, host_build, sb, threads):
    import torch
    M = 1 << sb
    tables = mb._tables(sb)
    rows = np.stack([f for _, f in tables])
    assert (rows.sum(axis=1) == M).all() and rows.max() <= M
    # one row that does not sum: block_prefix refuses it before any pairing
    bad = rows[0].copy()
    bad[int(np.argmax(bad))] -= 1
    rows = np.concatenate([rows, bad[None]]).astype(np.uint16)
    n = rows.shape[0]
    d_rows = torch.from_numpy(rows.reshape(-1).view(np.uint8).copy()).cuda()
    outs = {k: torch.zeros(n * size, dtype=torch.uint8, device="cuda")
            for k, size in (("div", 1024), ("adj", 2048), ("sf", 2048), ("sym", 512), ("remap", 2 * M), ("flags", 4))}
    assert pd.pd_alias_tables(d_rows.data_ptr(), n, sb, threads, *(outs[k].data_ptr() for k in ("div", "adj", "sf", "sym", "remap",
                                                                                                  "flags"))) == 0
    got = {k: v.cpu().numpy() for k, v in outs.items()}
    div = got["div"].view(np.uint32).reshape(n, 256)
    adj, sf = got["adj"].view(np.uint32).reshape(n, 512), got["sf"].view(np.uint32).reshape(n, 512)
    sym, remap = got["sym"].reshape(n, 512), got["remap"].view(np.uint16).reshape(n, M)
    flags = got["flags"].view(np.uint32)
    assert flags[-1] == 0
    for i, (name, f) in enumerate(tables):
        rc, hd, ha, hs, hy, hr = host_tables(host_build, f, sb)
        assert rc == 0, name
        assert flags[i] == 3, name
        assert np.array_equal(div[i], hd), (name, "divider")
        assert np.array_equal(adj[i], ha), (name, "slot_adjust")
        assert np.array_equal(sf[i], hs), (name, "slot_freqs")
        assert np.array_equal(sym[i], hy), (name, "sym_id")
        assert np.array_equal(remap[i], hr), (name, "remap")

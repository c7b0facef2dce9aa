"""In-tree build of librans_b200.so (and the C++ example driver) with nvcc for sm_90a (H100)."""
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.environ.get("RB200_LIB") or os.path.join(_HERE, "librans_b200.so")   # RB200_LIB: A/B-test another build
EXAM_PATH = os.path.join(_HERE, "exam_gpu")
EXAM_MULTI_PATH = os.path.join(_HERE, "exam_gpu_multi")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-Wall", "-I" + os.path.join(_ROOT, "include"), "-I" + CSRC,
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build librans_b200.so")
    return exe


def _sources():
    out = []
    for d, _, files in os.walk(CSRC):
        out += [os.path.join(d, f) for f in files]
    out.append(os.path.join(_ROOT, "include", "rans_b200.h"))
    return out


def _stale(target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in _sources())


def build(force=False, verbose=False):
    """Compile every CUDA/C++ source of the package.  Idempotent; returns LIB_PATH."""
    nvcc = _nvcc()
    if force or _stale(LIB_PATH):
        cmd = [nvcc, *NVCC_FLAGS, "-shared", "-o", LIB_PATH,
               os.path.join(CSRC, "rans_b200.cu"), os.path.join(CSRC, "model_host.cpp"), os.path.join(CSRC, "container_host.cpp")]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        subprocess.check_call(cmd)
    exam_src = os.path.join(CSRC, "exam_gpu.cpp")
    if os.path.exists(exam_src) and (force or _stale(EXAM_PATH)):
        subprocess.check_call([shutil.which("g++") or "g++", "-O2", "-std=c++17", "-I" + os.path.join(_ROOT, "include"),
                               "-o", EXAM_PATH, exam_src, "-L" + _HERE, "-lrans_b200", "-Wl,-rpath,$ORIGIN"])
    multi_src = os.path.join(CSRC, "exam_gpu_multi.cpp")          # the sharded driver: needs the CUDA runtime for its buffers
    if os.path.exists(multi_src) and (force or _stale(EXAM_MULTI_PATH)):
        subprocess.check_call([nvcc, "-Wno-deprecated-gpu-targets", "-O2", "-std=c++17", "-I" + os.path.join(_ROOT, "include"), "-o", EXAM_MULTI_PATH, multi_src,
                               "-L" + _HERE, "-lrans_b200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"])
    return LIB_PATH

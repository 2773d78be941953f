"""Build libcvnets_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python ml-cvnets_b200/csrc/build.py [--force] [--verbose]
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["gemm.cu", "gemm_tc.cu", "wgrad_tc.cu", "dwconv.cu", "dwconv_dilated.cu", "norm.cu", "linattn.cu", "mha.cu", "mha_tc.cu", "mha_long.cu", "optim.cu", "loss.cu", "conv.cu", "clip.cu", "se.cu", "dropout.cu"]
LIB = os.path.join(HERE, "libcvnets_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "--use_fast_math",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _digest():
    h = hashlib.sha256()
    for fn in sorted(SOURCES + ["common.cuh", "mha_wgmma.cuh", "../../include/cvnets_b200.h", "build.py"]):
        with open(os.path.join(HERE, fn), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    stamp = os.path.join(HERE, ".build_stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    objs = []

    def compile_one(src):
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(HERE, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))

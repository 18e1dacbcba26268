"""In-tree build of the CUDA engine (sm_90a only) into ``howtotrainyourmamlpytorch_b200/lib``.

``python -m howtotrainyourmamlpytorch_b200.build`` or ``build_native()``.  nvcc cross-compiles
without a GPU; the resulting ``libmaml_b200.so`` is git-ignored.
"""
import hashlib
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libmaml_b200.so")
SOURCES = ["kernels_conv.cu", "kernels_bn.cu", "kernels_head.cu", "kernels_param.cu", "kernels_tc.cu", "engine.cu"]
HEADERS = ["common.cuh", "tc_common.cuh", "head_body.cuh", "head_body_impl.inc", os.path.join("..", "..", "include", "maml_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest():
    hsh = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            hsh.update(fh.read())
    hsh.update(" ".join(NVCC_FLAGS).encode())
    return hsh.hexdigest()


def build_native(force=False, verbose=False):
    """Compile every .cu of the engine and link ``libmaml_b200.so``.  Returns the library path."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out))
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv))

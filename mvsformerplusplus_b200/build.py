"""Builds libmvsf_b200.so in-tree with nvcc for sm_90a (no torch headers involved: the library is pure CUDA
runtime behind a C ABI).  Usage: python -m mvsformerplusplus_b200.build [--force] [--verbose]"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmvsf_b200.so")
STAMP = os.path.join(HERE, ".libmvsf_b200.stamp")
SOURCES = ["api.cu", "geometry.cu", "warp_corr.cu", "warp_tile.cu", "vis_cnn.cu", "costreg_unet.cu", "costreg_tr.cu", "fmt.cu", "linear_tc.cu", "conv3d_tc.cu", "fpn.cu", "vit_decoder.cu", "vit.cu", "fusion.cu", "image_prep.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--extended-lambda"] + os.environ.get("MVSF_EXTRA_NVCC_FLAGS", "").split()


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _digest():
    h = hashlib.sha256()
    names = sorted(os.listdir(CSRC)) + ["../../include/mvsf_b200.h"]
    for n in names:
        p = os.path.join(CSRC, n)
        if os.path.isfile(p):
            h.update(n.encode())
            h.update(open(p, "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(f"---- {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed (see output above)")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static", "-lrt", "-lpthread", "-ldl"]
    subprocess.check_call(cmd)
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))

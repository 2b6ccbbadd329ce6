"""Build libb200_e2eft.so (sm_90a only) in-tree with nvcc.  No torch dependency: the library is a
plain C-ABI shared object (include/b200_e2eft.h) loaded through ctypes."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200_e2eft.so")
OBJ = os.path.join(HERE, "build")
SOURCES = ["gemm_conv.cu", "attention.cu", "attention_bwd.cu", "attention_d512_bwd.cu", "norm.cu", "elementwise.cu", "conv_small.cu", "loss.cu", "optim.cu", "backward.cu", "postproc.cu",
           "evaluation.cu", "data.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC"]


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                h.update(open(os.path.join(root, f), "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "stamp")
    dg = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dg:
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; cannot build {OUT}")

    def cc(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(cc, SOURCES))
    r = subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    open(stamp, "w").write(dg)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

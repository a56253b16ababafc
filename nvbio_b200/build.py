"""In-tree build of libnvbio_b200.so (sm_90a only): one nvcc compile per .cu in parallel, then a link.

    python -m nvbio_b200.build            # build if stale
    python -m nvbio_b200.build --force

The .so and the objects under build/ are git-ignored build products."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libnvbio_b200.so")
SOURCES = ["fm_kernels.cu", "gotoh_kernels.cu", "sa_build.cu", "pipeline.cu", "host_pipeline.cu", "map_kernels.cu", "finish.cu", "bam.cu", "bgzf.cu", "bam_sort.cu", "sam.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
         "-Wno-deprecated-declarations", "-Xcompiler", "-fPIC"] + os.environ.get("NVB_NVCC_EXTRA", "").split()


def _deps():
    d = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    d.append(os.path.join(os.path.dirname(HERE), "include", "nvbio_b200.h"))
    return d


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps())


def build(force=False, verbose=False):
    if not force and not stale():
        return LIB
    os.makedirs(OBJ, exist_ok=True)

    def cc(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose and r.stderr:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(cc, SOURCES))
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))

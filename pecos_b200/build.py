"""Builds ``pecos_b200/lib/libpecos_b200_float32.so`` in-tree with nvcc for sm_90a (H100) (cross-compiles without a GPU)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libpecos_b200_float32.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "-fmad=false",            # score paths must not contract x*w+acc into an FMA (bit parity with the reference)
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function,-O3",
    "-shared",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = glob.glob(os.path.join(CSRC, "*")) + [os.path.join(HERE, "..", "include", "pecos_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + sources() + ["-o", LIB_PATH]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or out.returncode != 0:
        sys.stdout.write(out.stdout)
    if out.returncode != 0:
        raise RuntimeError("nvcc failed building libpecos_b200_float32.so")
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)

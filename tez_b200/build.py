"""Builds libtezgpu.so (hand-written CUDA for sm_90a + the C-ABI) in-tree with nvcc.

The .so is git-ignored; build() rebuilds it when a source is newer.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtezgpu.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-shared",
]


def _sources():
    out = []
    for root, _, files in os.walk(SRC):
        for f in files:
            if f.endswith((".cu", ".cuh", ".h", ".inl", ".cc")):
                out.append(os.path.join(root, f))
    out.append(os.path.join(os.path.dirname(HERE), "include", "tezgpu.h"))
    return out


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in _sources() if os.path.exists(s))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    units = [os.path.join(SRC, "tezgpu_api.cu")]
    host = os.path.join(SRC, "host")
    if os.path.isdir(host):
        units += sorted(os.path.join(host, f) for f in os.listdir(host) if f.endswith((".cc", ".cu")))
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + units + ["-lz"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building libtezgpu.so")
    if verbose:
        print(r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

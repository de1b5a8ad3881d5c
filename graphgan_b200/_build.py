"""Compile libgraphgan_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, no torch extension).

The shared object lands next to this file (git-ignored), so the package is importable from the source tree."""
import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgraphgan_b200.so")
STAMP = LIB + ".hash"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-ldl",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def source_hash():
    """sha256 over every file the library is built from (names + contents) and the compiler flags."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    deps = sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + sorted(glob.glob(os.path.join(HERE, "..", "include", "*.h")))
    for p in deps:
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def stale():
    """True when the .so is missing or was built from other sources than the ones in the tree (content hash in a
    sidecar file, so that copying the tree -- which changes mtimes -- does not trigger rebuilds)."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != source_hash()


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return p if os.path.exists(p) else None


def build_variant(name, defines):
    """A/B library libgraphgan_b200.<name>.so with extra -D flags (tools/variants.py); load it with GG_LIB=<path>."""
    out_path = os.path.join(HERE, "libgraphgan_b200.%s.so" % name)
    cmd = [nvcc_path()] + NVCC_FLAGS + ["-D%s" % d for d in defines] + ["-o", out_path] + sources()
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if out.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + out.stdout)
    return out_path


def build(force=False, verbose=False):
    if not force and not stale():
        return LIB
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libgraphgan_b200.so")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + sources()
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if out.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + out.stdout)
    if verbose:
        print(out.stdout)
    with open(STAMP, "w") as f:
        f.write(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))

"""Build libvrgdg_b200.so (sm_90a only) in-tree with nvcc.  No GPU is needed to build.

    python comfyui-vrgamedevgirl_b200/build.py [--force]

The library lands in comfyui-vrgamedevgirl_b200/lib/ (git-ignored, travels to the GPU box with the snapshot).
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libvrgdg_b200.so")
STAMP = LIB + ".srchash"
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
UNITS = ["vrgdg_abi.cu", "vrgdg_f32.cu", "vrgdg_f16.cu", "vrgdg_bf16.cu", "vrgdg_u8.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-Xfatbin", "-compress-all", "-I", INCLUDE,
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; libvrgdg_b200.so cannot be built")
    return exe


def _sources():
    out = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    out.append(os.path.join(INCLUDE, "vrgdg_b200.h"))
    return out


def _source_hash():
    """Content hash of every source the library is built from (mtimes do not survive a copy of the tree to another box)."""
    h = hashlib.sha256()
    for path in sorted(_sources()):
        h.update(os.path.basename(path).encode())
        with open(path, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS[:-1]).encode())
    return h.hexdigest()


def is_fresh():
    """The library exists and was built from exactly the sources that are in the tree now."""
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return False
    with open(STAMP, encoding="utf-8") as fh:
        return fh.read().strip() == _source_hash()


def build(force=False, verbose=True):
    if not force and is_fresh():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(unit):
        obj = os.path.join(OBJDIR, unit.replace(".cu", ".o"))
        src = os.path.join(CSRC, unit)
        deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + [os.path.join(INCLUDE, "vrgdg_b200.h")]
        if not force and os.path.exists(obj) and all(os.path.getmtime(d) <= os.path.getmtime(obj) for d in deps):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (unit, r.stdout, r.stderr))
        return obj

    with ThreadPoolExecutor(max_workers=len(UNITS)) as ex:
        objs = list(ex.map(compile_one, UNITS))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-Xcompiler", "-fPIC", "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(STAMP, "w", encoding="utf-8") as fh:
        fh.write(_source_hash() + "\n")
    if verbose:
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)

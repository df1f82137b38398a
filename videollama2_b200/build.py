"""Build libvl2.so (the sm_90a kernel library + C-ABI) in-tree with nvcc.

`python -m videollama2_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.  The libraries and
object files are build products (git-ignored).
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libvl2.so")
OBJ_DIR = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libvl2.so cannot be built")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


# The same sources build twice: bf16 storage (libvl2.so) and, with -DVL2_HALF, IEEE fp16 storage (libvl2_f16.so) - the
# reference's own inference dtype.  See csrc/ptx.cuh.
VARIANTS = {
    "bf16": (OUT, OBJ_DIR, []),
    "f16": (os.path.join(HERE, "libvl2_f16.so"), os.path.join(HERE, "build_f16"), ["-DVL2_HALF"]),
}


def lib_path(variant: str = "bf16") -> str:
    return VARIANTS[variant][0]


def build(force: bool = False, verbose: bool = False) -> str:
    """Builds every variant that is stale; returns the bf16 library's path."""
    dig = _digest()
    todo = []
    for name, (out, obj_dir, defs) in VARIANTS.items():
        os.makedirs(obj_dir, exist_ok=True)
        stamp = os.path.join(obj_dir, "stamp")
        if force or not (os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == dig):
            todo.append((name, out, obj_dir, defs, stamp))
    if not todo:
        return OUT
    nvcc = _nvcc()
    srcs = _sources()
    jobs = [(src, os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o"), defs) for _, _, obj_dir, defs, _ in todo for src in srcs]

    def compile_one(job):
        src, obj, defs = job
        cmd = [nvcc, *NVCC_FLAGS, *defs, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
        for src, r in ex.map(compile_one, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}")
    for name, out, obj_dir, defs, stamp in todo:
        objs = [os.path.join(obj_dir, os.path.basename(s)[:-3] + ".o") for s in srcs]
        tmp = out + ".tmp"   # link next to the target, then rename: a reader never sees a partial library
        link = [nvcc, "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(link, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"link of {os.path.basename(out)} failed")
        os.replace(tmp, out)
        with open(stamp, "w") as fh:
            fh.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

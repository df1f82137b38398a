"""The compiled GEMM kernels, read from the built library's SASS (no GPU needed).

Every consumer warp of the GEMM releases a ring slot once per k-block.  A slot release that publishes no data must not
carry a memory fence: `mbarrier.arrive.release.cluster` compiles to MEMBAR.ALL.GPU in front of the arrive, i.e. a
GPU-scope fence in every k-block of the pair kernel that also waits for the previous tile's global stores.  These tests
pin that the k-loop of every instantiation is free of GPU-scope fences, that the GEMM kernels do not spill, and that the
epilogue stays rolled (a small kernel)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "videollama2_b200", n) for n in ("libvl2.so", "libvl2_f16.so")]
KERNEL = "gemm_bf16_wgmma_kernel"


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module", params=LIBS, ids=lambda p: os.path.basename(p))
def library(request):
    if _cuobjdump() is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(request.param):
        pytest.skip(f"{os.path.basename(request.param)} is not built")
    return request.param


def sass_functions(path):
    """{mangled name: [(address, instruction text)]} of every GEMM kernel in the library."""
    out = subprocess.run([_cuobjdump(), "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if KERNEL in m.group(1) else None
            if cur is not None:
                funcs[cur] = []
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;", line)
        if cur is not None and m:
            funcs[cur].append((int(m.group(1), 16), m.group(2)))
    return funcs


def k_loop(instrs):
    """(first HGMMA, back edge) addresses: the back edge is the first branch after the first HGMMA that jumps to or
    before it, i.e. the end of the innermost loop that issues the MMAs."""
    first = next(a for a, s in instrs if re.search(r"\bHGMMA\b", s))
    for a, s in instrs:
        m = re.search(r"\bBRA\s+(?:`\()?0x([0-9a-f]+)", s)
        if a > first and m and int(m.group(1), 16) <= first:
            return first, a
    raise AssertionError("no loop around the first HGMMA")


def test_k_loop_has_no_gpu_scope_fence(library):
    funcs = sass_functions(library)
    # 7 single-CTA widths (64..256) and 5 pair widths (128..256)
    assert len(funcs) == 12, sorted(funcs)
    for name, instrs in funcs.items():
        first, back = k_loop(instrs)
        fences = [(hex(a), s) for a, s in instrs if first <= a <= back and re.search(r"\bMEMBAR\.\S*GPU", s)]
        assert not fences, f"{name}: GPU-scope fence in the k-loop {hex(first)}..{hex(back)}: {fences}"


# Stack bytes a GEMM kernel may use: ptxas may keep one 64-bit address on the stack across the split-K owner's sum of the
# other slices' partials (split-K is off by default); nothing else may spill.
STACK_ALLOWED = 8


def test_gemm_kernels_do_not_spill(library):
    out = subprocess.run([_cuobjdump(), "-res-usage", library], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    seen = 0
    for i, line in enumerate(lines):
        if "Function" in line and KERNEL in line:
            usage = lines[i + 1]
            regs = int(re.search(r"REG:(\d+)", usage).group(1))
            stack = int(re.search(r"STACK:(\d+)", usage).group(1))
            local = int(re.search(r"LOCAL:(\d+)", usage).group(1))
            print(f"{line.split()[-1].rstrip(':')}: {regs} registers, {stack} bytes stack, {local} bytes local")
            assert local == 0 and stack <= STACK_ALLOWED, f"{line.strip()} spills: {usage.strip()}"
            seen += 1
    assert seen == 12


def test_epilogue_is_not_unrolled_over_the_tile(library):
    """The epilogue loops over 32-column slots and 8-column groups (~3.5 k instructions per kernel).  Unrolled over the
    whole tile it was ~25 k instructions (~400 KB), more than the SM's instruction caches hold, and the epilogue of a
    128 x 256 tile took ~200 k cycles instead of ~50 k."""
    for name, instrs in sass_functions(library).items():
        assert len(instrs) < 8000, f"{name}: {len(instrs)} instructions"

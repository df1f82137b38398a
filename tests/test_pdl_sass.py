"""Programmatic dependent launch (PDL), read from the built libraries' SASS (no GPU needed).

Every kernel is launched through launch_kernel, which adds the programmatic-stream-serialization attribute when PDL is on
(vl2_set_pdl, VL2_PDL=1, the decode graph's decode_pdl).  Under that attribute a kernel may start as soon as its
predecessor in the stream executes griddepcontrol.launch_dependents - the GEMM does so at its first instruction - and
only griddepcontrol.wait makes the predecessor's stores visible and its reads finished.  A kernel that touches global
memory before the wait can read inputs that are not written yet, or overwrite memory its predecessor still reads.

On sm_90a griddepcontrol.wait compiles to ACQBULK and griddepcontrol.launch_dependents to PREEXIT.  For every kernel of
both builds this test asserts that there is an ACQBULK and that no global-memory instruction precedes the first one in
address order.  Address order is not control flow: the check is conservative for the straight-line prologues these
kernels have (a global access placed after the wait in address order but reached before it by a branch would pass, so
the wait belongs at the top of the kernel, ahead of any branch that leads to memory).

Exemptions, each for a stated reason:
  * l2_prefetch_kernel has no wait: it issues L2 prefetch hints (UBLKPF) only and moves no data.
  * gemv_kernel issues bulk copies (UBLKCP) of its weight rows W before the wait, so that they stream while the
    producer of x drains.  Its contract: W is a constant that the launch just before it does not write.  No other
    global access may precede its wait."""
import functools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = [os.path.join(ROOT, "videollama2_b200", n) for n in ("libvl2.so", "libvl2_f16.so")]

# opcodes (before the first '.') that read or write global memory; shared-memory (LDS / STS / ATOMS), local, constant,
# mbarrier (SYNCS), tensor-map cache control and bulk L2 prefetch (UBLKPF) instructions do not count
GLOBAL_OPS = {"LDG", "LDGMC", "LDGSTS", "STG", "LD", "ST", "ATOMG", "ATOM", "RED", "REDG", "UTMALDG", "UTMASTG",
              "UTMAREDG", "UBLKCP", "UBLKRED"}
NO_WAIT = {"l2_prefetch_kernel": "issues L2 prefetch hints only and moves no data"}
EARLY_OPS = {"gemv_kernel": ({"UBLKCP"}, "bulk-loads its constant weights W before the wait")}


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


@functools.lru_cache(maxsize=None)
def kernels(path):
    """{mangled name: [(address, opcode)]} of every function in the library; the opcode without predicate or modifiers."""
    out = subprocess.run([_cuobjdump(), "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", line)
        if cur is not None and m:
            funcs[cur].append((int(m.group(1), 16), m.group(2)))
    return funcs


def _rule(name, table):
    return next((v for k, v in table.items() if re.search(r"\d" + k + r"[EI]", name)), None)


def violations(funcs):
    """[(kernel, what is wrong)] for every kernel that has no wait or touches global memory before its first wait."""
    bad = []
    for name, instrs in sorted(funcs.items()):
        waits = [a for a, op in instrs if op == "ACQBULK"]
        if not waits:
            if _rule(name, NO_WAIT) is None:
                bad.append((name, "no griddepcontrol.wait (ACQBULK)"))
            continue
        allowed = (_rule(name, EARLY_OPS) or (set(), ""))[0]
        early = [(hex(a), op) for a, op in instrs if a < waits[0] and op in GLOBAL_OPS and op not in allowed]
        if early:
            bad.append((name, f"global-memory access before the first ACQBULK at {hex(waits[0])}: {early[:4]}"))
    return bad


def test_every_kernel_waits_before_touching_global_memory(library):
    funcs = kernels(library)
    print(f"{os.path.basename(library)}: {len(funcs)} kernels checked")
    assert len(funcs) >= 50, sorted(funcs)
    for table in (NO_WAIT, EARLY_OPS):   # every exemption names a kernel that exists
        for k in table:
            assert any(_rule(n, {k: 1}) for n in funcs), f"exemption {k} matches no kernel"
    bad = violations(funcs)
    assert not bad, "\n".join(f"{n}: {w}" for n, w in bad)


def test_gemv_waits_before_reading_x_and_triggers_before_its_stores(library):
    """The GEMV's exemption covers its weight bulk copies only; x is read after the wait, and the dependents are
    released (PREEXIT) before the output stores."""
    for name, instrs in kernels(library).items():
        if _rule(name, {"gemv_kernel": 1}) is None:
            continue
        wait = next(a for a, op in instrs if op == "ACQBULK")
        assert not [a for a, op in instrs if op in ("LDG", "LD") and a < wait], name
        trigger = next(a for a, op in instrs if op == "PREEXIT")
        assert trigger > wait and any(op == "STG" and a > trigger for a, op in instrs), name

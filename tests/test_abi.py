"""The C-ABI library builds, loads on a CPU-only box and exports every symbol include/vl2.h declares
(no compute calls here: without a GPU every compute entry point must fail with VL2_E_CUDA, never fall back)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from videollama2_b200 import _lib, build
    build.build()
    return _lib.load()


def header_symbols():
    src = open(os.path.join(ROOT, "include", "vl2.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vl2_[a-z0-9_]+)\s*\(", src)))


def test_header_matches_binding_list():
    from videollama2_b200 import _lib
    assert header_symbols() == sorted(_lib.SYMBOLS)


def test_library_exports_every_declared_symbol(lib):
    for sym in header_symbols():
        assert hasattr(lib, sym), f"libvl2.so does not export {sym}"
    assert lib.vl2_version() == 100
    assert isinstance(lib.vl2_last_error(), bytes)


def test_struct_layouts_match_header():
    from videollama2_b200._lib import AttnArgs, GemmArgs
    assert ctypes.sizeof(GemmArgs) == 6 * 8 + 4 * 8 + 6 * 4 + 8 * 8 + 8 + 2 * 4 + 2 * 8 + 2 * 4 + 2 * 4 + 2 * 8 + 3 * 8 + 6 * 4 + 8 + 4 * 4 
    assert ctypes.sizeof(AttnArgs) == 4 * 8 + 4 * 8 + 8 * 4


BADSHAPE, BADALIGN = -1, -3
A16, MIS = 4096, 4104          # fake device addresses: 16-byte aligned, and 8 bytes off (never dereferenced)
ROW_ARGUMENT_CASES = [
    # odd P: a pixel pair at an odd element offset would be loaded as one misaligned 4-byte word
    ("vl2_patch_im2col", (A16, A16, 1, 15, 16, 15, 680, None), BADSHAPE),
    ("vl2_patch_im2col", (A16, A16, 1, 14, 14, 7, 152, None), BADSHAPE),
    ("vl2_patch_im2col", (A16 + 2, A16, 1, 14, 14, 14, 592, None), BADALIGN),
    # 16-byte vector accesses: every pointer they touch is checked
    ("vl2_se_scale", (MIS, A16, 1, 4, 64, None), BADALIGN),
    ("vl2_se_scale", (A16, MIS, 1, 4, 64, None), BADALIGN),
    ("vl2_clip_embed_finish", (A16, A16, A16, MIS, A16, A16, 1, 4, 64, 1e-5, None), BADALIGN),
    ("vl2_clip_embed_finish", (A16, A16, A16, A16, MIS, A16, 1, 4, 64, 1e-5, None), BADALIGN),
    ("vl2_embed_splice", (A16, A16, 2, MIS, 100, A16, 64, None), BADALIGN),
    ("vl2_embed_splice", (A16, A16, 2, A16, 100, MIS, 64, None), BADALIGN),
    ("vl2_conv3d_im2col", (MIS, A16, 2, 4, 4, 64, 1, 2, 3, 3, None), BADALIGN),
    ("vl2_conv3d_im2col", (A16, MIS, 2, 4, 4, 64, 1, 2, 3, 3, None), BADALIGN),
    ("vl2_decode_rope_append", (MIS, A16, 768, A16, 4, 1, 128, A16, 1, None), BADALIGN),
    ("vl2_decode_rope_append", (A16, MIS, 768, A16, 4, 1, 128, A16, 1, None), BADALIGN),
]


def test_argument_validation_without_gpu(lib):
    """Shape/alignment checks run before any CUDA call, so they are testable on CPU.  Odd patch sizes and misaligned
    pointers are refused with VL2_E_BADSHAPE / VL2_E_BADALIGN (the kernels would fault on a misaligned vector access)."""
    from videollama2_b200._lib import GemmArgs
    a = GemmArgs(A=16, W=16, C=16, lda=8, ldw=8, ldc=8, ldr=0, M=4, N=8, K=12, act=0, out_f32=0)
    assert lib.vl2_gemm_bf16(ctypes.byref(a), None) == -1 and b"multiples of 8" in lib.vl2_last_error()
    a = GemmArgs(A=17, W=16, C=16, lda=8, ldw=8, ldc=8, ldr=0, M=4, N=8, K=8, act=0, out_f32=0)
    assert lib.vl2_gemm_bf16(ctypes.byref(a), None) == -3
    a = GemmArgs(A=16, W=16, C=16, lda=8, ldw=8, ldc=8, ldr=0, M=4, N=8, K=8, act=9, out_f32=0)
    assert lib.vl2_gemm_bf16(ctypes.byref(a), None) == -6
    for name, args, code in ROW_ARGUMENT_CASES:
        assert getattr(lib, name)(*args) == code, (name, args, lib.vl2_last_error())


def _tp_args(**kw):
    """vl2_tp_allreduce_args of rank 0 of 2 over fake, 16-byte aligned buffers; `kw` overrides fields."""
    from videollama2_b200._lib import TpAllReduceArgs
    a = TpAllReduceArgs(rank=0, world=2, S=4, H=64, epoch=1, inswitch_reduce=0)
    for r in range(8):
        a.part[r], a.xout[r], a.stats[r], a.pads[r] = A16, A16 + 4096, A16 + 8192, A16 + 12288
    for k, v in kw.items():
        if isinstance(v, tuple):                  # (array field, index, value)
            getattr(a, k)[v[0]] = v[1]
        else:
            setattr(a, k, v)
    return a


TP_ARGUMENT_CASES = [
    (dict(world=0), BADSHAPE), (dict(world=9), BADSHAPE),
    (dict(rank=2), BADSHAPE), (dict(rank=-1), BADSHAPE),
    (dict(S=0), BADSHAPE), (dict(H=60), BADSHAPE), (dict(H=0), BADSHAPE),
    (dict(epoch=0), BADSHAPE),
    (dict(part_mc=A16), BADSHAPE),                              # multicast part without multicast xout / stats
    (dict(part_mc=A16, xout_mc=A16), BADSHAPE),
    (dict(part=(1, None)), BADSHAPE), (dict(xout=(1, None)), BADSHAPE), (dict(stats=(1, None)), BADSHAPE),
    (dict(pads=(1, None)), BADSHAPE),
    (dict(part=(1, MIS)), BADALIGN), (dict(xout=(0, MIS)), BADALIGN),
]


def test_tp_allreduce_argument_validation_without_gpu(lib):
    """vl2_tp_allreduce_stats refuses, before any CUDA call: a world outside 1..8, a rank outside the world, S or H not
    positive, H % 8 != 0, epoch 0 (the pads start at 0: nothing would wait), a multicast part address without the other
    two, a missing buffer of a rank in the world (VL2_E_BADSHAPE), and a part or xout buffer that is not 16-byte aligned
    (VL2_E_BADALIGN), each with a message naming the call."""
    for kw, code in TP_ARGUMENT_CASES:
        a = _tp_args(**kw)
        assert lib.vl2_tp_allreduce_stats(ctypes.byref(a), None) == code, (kw, lib.vl2_last_error())
        assert lib.vl2_last_error().startswith(b"vl2_tp_allreduce_stats: "), kw
    assert lib.vl2_tp_allreduce_stats(None, None) == BADSHAPE


def test_ops_refuse_cpu_tensors():
    import torch
    from videollama2_b200 import ops
    from videollama2_b200._lib import Vl2Error
    x = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(Vl2Error):
        ops.gemm(x, x)
    with pytest.raises(Vl2Error):
        ops.layernorm(x, x[0], x[0], 1e-5)


C_CONSUMER = r"""
#include <stdio.h>
#include <string.h>
#include "vl2.h"
/* A plain C99 consumer of the C-ABI: no torch, no C++.  Prints the struct sizes the Python binding must agree with and
 * checks that argument validation happens before any CUDA call (so it also runs on a box without a GPU). */
int main(void) {
  vl2_gemm_args g;
  vl2_attn_args a;
  vl2_preprocess_args pp;
  memset(&g, 0, sizeof g); memset(&a, 0, sizeof a); memset(&pp, 0, sizeof pp);
  printf("%d %zu %zu %zu\n", vl2_version(), sizeof g, sizeof a, sizeof pp);
  g.M = 4; g.N = 8; g.K = 12;                       /* K %% 8 != 0 */
  int rc = vl2_gemm_bf16(&g, NULL);
  printf("%d %s\n", rc, vl2_last_error());
  rc = vl2_attention(NULL, NULL);
  printf("%d\n", rc);
  rc = vl2_preprocess_frames(&pp, NULL);
  printf("%d\n", rc);
  printf("%zu %zu\n", vl2_attention_decode_workspace(32, 8, 128), vl2_preprocess_workspace(&pp));
  return 0;
}
"""


def test_plain_c_consumer_links_and_validates(lib, tmp_path):
    """include/vl2.h is valid C99, a C program links against libvl2.so with nothing but the header, the struct sizes
    match the ctypes mirrors, and bad arguments are rejected with VL2_E_* codes before any device work."""
    import shutil
    import subprocess
    from videollama2_b200 import _lib, preprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "consumer.c"
    src.write_text(C_CONSUMER)
    exe = tmp_path / "consumer"
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                    "-o", str(exe), "-L", libdir, "-l:libvl2.so", f"-Wl,-rpath,{libdir}"], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    ver, sz_gemm, sz_attn, sz_pp = out[0].split()
    assert int(ver) == 100
    assert int(sz_gemm) == ctypes.sizeof(_lib.GemmArgs) and int(sz_attn) == ctypes.sizeof(_lib.AttnArgs)
    assert int(sz_pp) == ctypes.sizeof(preprocess.PreprocessArgs)
    assert out[1].startswith("-") and "multiples of 8" in out[1]          # VL2_E_BADSHAPE + message
    assert int(out[2]) < 0 and int(out[3]) < 0
    ws_attn, ws_pp = out[4].split()
    assert int(ws_attn) == 32 * (296 // 8) * 130 * 4 and int(ws_pp) == 0


def test_gemm_plan_for_the_path_shapes(lib):
    """vl2_gemm_plan is host logic only: the tile the cost model picks and how many rounds the persistent grid runs for
    the GEMMs of config 2 (132 SMs, an H100 SXM, assumed without a device).  Pins the scheduler against accidental changes."""
    def plan(M, N, K):
        out = (ctypes.c_int32 * 6)()
        assert lib.vl2_gemm_plan(M, N, K, 0, out) == 0
        return dict(zip(("bn", "pair", "tiles", "slots", "rounds", "sms"), out))
    gate_up = plan(1776, 28672, 4096)            # decoder gate/up: the 256 x 256 two-CTA tile, 784 tiles on 66 pairs
    assert (gate_up["bn"], gate_up["pair"], gate_up["tiles"], gate_up["slots"], gate_up["rounds"]) == (256, 1, 784, 66, 12)
    for M, N, K in [(1776, 6144, 4096), (1776, 4096, 4096), (1776, 4096, 14336), (9232, 3072, 1024), (9232, 4096, 1024),
                    (9232, 1024, 4096), (11664, 1152, 1152)]:
        p = plan(M, N, K)
        assert p["pair"] == 1 and p["bn"] in (192, 224, 256) and p["sms"] == 132
        tile_m = 256
        assert p["tiles"] == -(-M // tile_m) * -(-N // p["bn"]) and p["rounds"] == -(-p["tiles"] // p["slots"])
    o_proj, down = plan(1776, 4096, 4096), plan(1776, 4096, 14336)   # 7 x 16 tiles: two rounds of the 66 pairs
    assert (o_proj["bn"], o_proj["rounds"], down["bn"], down["rounds"]) == (256, 2, 256, 2)
    assert plan(1776, 6144, 4096)["bn"] == 224 and plan(9232, 1024, 1024)["bn"] == 224
    small = plan(300, 520, 256)                  # a small matrix gets a narrow single-CTA tile
    assert small["pair"] == 0 and small["bn"] <= 128 and small["rounds"] == 1
    out = (ctypes.c_int32 * 6)()
    assert lib.vl2_gemm_plan(0, 8, 8, 0, out) < 0


def test_ops_validate_out_and_inv_freq_before_launch(monkeypatch):
    """attention / attention_decode refuse an `out` of another type than the operands (a bf16 or fp32 buffer would be
    filled with fp16 bit patterns) or of the wrong shape, and decode_rope_append an inv_freq that is not fp32 [D / 2],
    before anything is launched: the device check and the library are replaced by stand-ins, and a launch fails."""
    import torch
    from videollama2_b200 import ops

    class Launched(Exception):
        pass

    def no_launch(t):
        raise Launched("a kernel was launched")

    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ops, "_L", no_launch)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "decode_workspace", lambda *a: torch.zeros(16))
    B, S, Hq, Hkv, D = 1, 8, 4, 2, 64
    h = torch.float16
    q, k, v = torch.zeros(B * S, Hq * D, dtype=h), torch.zeros(B * S, Hkv * D, dtype=h), torch.zeros(B * S, Hkv * D, dtype=h)
    kw = dict(B=B, S=S, Hq=Hq, Hkv=Hkv, D=D, causal=True, scale=0.125)
    for bad in (torch.bfloat16, torch.float32):
        with pytest.raises(TypeError):
            ops.attention(q, k, v, out=torch.zeros(B * S, Hq * D, dtype=bad), **kw)
    with pytest.raises(AssertionError):
        ops.attention(q, k, v, out=torch.zeros(B * S, Hq * D - 8, dtype=h), **kw)
    with pytest.raises(Launched):
        ops.attention(q, k, v, out=torch.zeros(B * S, Hq * D, dtype=h), **kw)
    qd, cache = torch.zeros(Hq * D, dtype=h), torch.zeros(16, (Hq + 2 * Hkv) * D, dtype=h)
    kc, vc = cache[:, Hq * D:(Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:]
    kw = dict(n_pos=16, Hq=Hq, Hkv=Hkv, D=D, scale=0.125)
    for bad in (torch.bfloat16, torch.float32):
        with pytest.raises(TypeError):
            ops.attention_decode(qd, kc, vc, out=torch.zeros(1, Hq * D, dtype=bad), **kw)
    with pytest.raises(AssertionError):
        ops.attention_decode(qd, kc, vc, out=torch.zeros(1, Hq * D // 2, dtype=h), **kw)
    with pytest.raises(Launched):
        ops.attention_decode(qd, kc, vc, out=torch.zeros(1, Hq * D, dtype=h), **kw)
    row, pos = torch.zeros(1, (Hq + 2 * Hkv) * D, dtype=h), torch.zeros(1, dtype=torch.int32)
    for inv in (torch.zeros(D // 2, dtype=torch.float64), torch.zeros(D // 2, dtype=h), torch.zeros(D, dtype=torch.float32)):
        with pytest.raises(AssertionError):
            ops.decode_rope_append(row, cache, pos, Hq, Hkv, D, inv)
    with pytest.raises(Launched):
        ops.decode_rope_append(row, cache, pos, Hq, Hkv, D, torch.zeros(D // 2, dtype=torch.float32))

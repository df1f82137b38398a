"""The GEMM's specialised epilogue variants against its generic epilogue, bit for bit.

vl2_gemm_bf16 picks one epilogue variant per launch from the arguments that are set (bias, bias + activation, bias +
residual, residual + sums of squares, RoPE, SwiGLU, none); everything else takes the generic epilogue. A variant does
the generic epilogue's fp32 operations in the same order, so the two must give the same bits. `generic_epilogue=True`
forces the generic one in the same process (the kernel's trace shows which of the two ran). Every variant runs at every
forced tile width (single CTA and pair) on both storage types, with M tails (M % 128 != 0 and M < 128) and N tails
inside a tile. Outputs are compared as raw 16-bit patterns, so a NaN-filled guard around a strided output view is
checked too."""
import pytest
import torch

from videollama2_b200 import ops

pytestmark = pytest.mark.gpu

STORAGE_TYPES = (torch.bfloat16, torch.float16)
DT_IDS = {torch.bfloat16: "bf16", torch.float16: "fp16"}
WIDTHS = [64, 96, 128, 160, 192, 224, 256] + [1000 + b for b in (128, 160, 192, 224, 256)]
K = 192
D_HEAD = 64


@pytest.fixture(autouse=True)
def _needs_device(cuda):
    return cuda


def _bits(t):
    return t.view(torch.int16) if t.dtype != torch.float32 else t.view(torch.int32)


def _operands(M, N, dt, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(dt).cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(dt).cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).to(dt).cuda()
    rms = (torch.rand(M, 4, generator=g) * K * 0.5 + 1.0).cuda()
    return a, w, bias, res, rms


def _case(variant, M, N, dt, seed=0):
    """ops.gemm keyword arguments of one epilogue variant (without `out`), and the output width."""
    a, w, bias, res, rms = _operands(M, N, dt, seed)
    if variant == "none":
        return a, w, {}, N
    if variant == "rms":
        return a, w, {"rms_in": rms, "rms_eps": 1e-5}, N
    if variant == "bias":
        return a, w, {"bias": bias}, N
    if variant.startswith("bias_act"):
        act = {"quick_gelu": ops.ACT_QUICK_GELU, "silu": ops.ACT_SILU, "gelu_erf": ops.ACT_GELU_ERF,
               "gelu_tanh": ops.ACT_GELU_TANH}[variant[len("bias_act_"):]]
        return a, w, {"bias": bias, "act": act}, N
    if variant == "bias_res":
        return a, w, {"bias": bias, "residual": res}, N
    if variant == "res_sumsq":
        return a, w, {"residual": res, "sumsq_out": None}, N
    if variant in ("rope", "bias_rope"):
        tab = ops.rope_table(5 + M + 1, D_HEAD, 1e6, "cuda", dt)
        kw = {"rms_in": rms, "rms_eps": 1e-5, "rope": (tab, 5, D_HEAD, max(D_HEAD, (N // 2 // D_HEAD) * D_HEAD))}
        if variant == "bias_rope":
            kw["bias"] = bias
        return a, w, kw, N
    if variant == "swiglu":
        return a, w, {"act": ops.ACT_SWIGLU, "rms_in": rms, "rms_eps": 1e-5}, N // 2
    raise ValueError(variant)


VARIANTS = ["none", "rms", "bias", "bias_act_quick_gelu", "bias_act_silu", "bias_act_gelu_erf", "bias_act_gelu_tanh",
            "bias_res", "res_sumsq", "rope", "bias_rope", "swiglu"]


def _run(a, w, kw, n_out, bn, generic, out=None, trace=False):
    kw = dict(kw)
    M = a.shape[0]
    if out is None:
        out = torch.full((M, n_out), float("nan"), device="cuda", dtype=a.dtype)
    sq = None
    if "sumsq_out" in kw:
        sq = torch.full((M, w.shape[0] // 32), float("nan"), device="cuda")
        kw["sumsq_out"] = sq
    ops.gemm(a, w, out=out, bn=bn, generic_epilogue=generic, trace=trace, **kw)
    return out, sq


def _assert_same(a, w, kw, n_out, bn):
    fast, sq_fast = _run(a, w, kw, n_out, bn, False)
    slow, sq_slow = _run(a, w, kw, n_out, bn, True)
    torch.cuda.synchronize()
    assert not torch.isnan(slow.float()).any(), "the generic epilogue left outputs unwritten"
    assert torch.equal(_bits(fast), _bits(slow))
    if sq_fast is not None:
        assert torch.equal(_bits(sq_fast), _bits(sq_slow))


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", [64, 1256])
@pytest.mark.parametrize("variant", VARIANTS)
def test_both_epilogues_run(variant, bn, dt):
    """The comparisons below compare two different code paths: the kernel's trace (first consumer thread of CTA 0)
    records the generic epilogue's first-slot points 1 and 2 as clocks and a variant's as -1; point 3 (first slot
    stored) is written by both."""
    a, w, kw, n_out = _case(variant, 300, 352, dt, seed=0)
    for generic in (False, True):
        _run(a, w, kw, n_out, bn, generic, trace=True)
        t = ops.gemm_trace(dt)
        assert t[0] >= 1 and t[3] >= t[5] > 0, t[:8]
        if generic:
            assert t[5] <= t[1] <= t[2] <= t[3], t[:8]
        else:
            assert t[1] == -1 and t[2] == -1, t[:8]


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
def test_uncovered_launch_takes_the_generic_epilogue(dt):
    """An fp32 output has no variant: the launch runs the generic epilogue without being forced to."""
    a, w, _, _ = _case("none", 300, 352, dt)
    ops.gemm(a, w, out_dtype=torch.float32, bn=1256, trace=True)
    t = ops.gemm_trace(dt)
    assert t[0] >= 1 and t[5] <= t[1] <= t[2] <= t[3], t[:8]


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_variant_matches_generic(variant, bn, dt):
    # M = 300: a 128-row and a 256-row tile tail; N = 352: a partial last tile at every width (N % BN != 0 but 256)
    a, w, kw, n_out = _case(variant, 300, 352, dt, seed=VARIANTS.index(variant))
    _assert_same(a, w, kw, n_out, bn)


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", [128, 256, 1128, 1256])
@pytest.mark.parametrize("variant", VARIANTS)
def test_variant_matches_generic_small_m(variant, bn, dt):
    # M < 128 (a single, partial tile) and N = 96: less than one tile wide at these widths
    a, w, kw, n_out = _case(variant, 77, 96, dt, seed=7)
    _assert_same(a, w, kw, n_out, bn)


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", [64, 224, 256, 1224, 1256])
def test_residual_aliasing_output(bn, dt):
    for variant in ("bias_res", "res_sumsq"):
        a, w, kw, n_out = _case(variant, 300, 352, dt, seed=3)
        got = []
        for generic in (False, True):
            x = kw["residual"].clone()
            k2 = dict(kw, residual=x)
            _, sq = _run(a, w, k2, n_out, bn, generic, out=x)
            got.append((x, sq))
        torch.cuda.synchronize()
        assert torch.equal(_bits(got[0][0]), _bits(got[1][0])), variant
        if got[0][1] is not None:
            assert torch.equal(_bits(got[0][1]), _bits(got[1][1])), variant
        # and it is the result without aliasing
        ref, _ = _run(a, w, kw, n_out, bn, True)
        assert torch.equal(_bits(got[0][0]), _bits(ref)), variant


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", [96, 256, 1160, 1256])
@pytest.mark.parametrize("variant", ["bias", "bias_act_gelu_erf", "bias_res", "res_sumsq", "rope", "swiglu"])
def test_strided_output_view_keeps_its_guard(variant, bn, dt):
    """out= is a view with ldc > N inside a NaN-filled buffer: the columns past N and the rows past M stay NaN."""
    M, N = 300, 352
    a, w, kw, n_out = _case(variant, M, N, dt, seed=11)
    bufs = []
    for generic in (False, True):
        buf = torch.full((M + 5, n_out + 40), float("nan"), device="cuda", dtype=dt)
        _run(a, w, kw, n_out, bn, generic, out=buf[:M, :n_out])
        bufs.append(buf)
    torch.cuda.synchronize()
    assert torch.equal(_bits(bufs[0]), _bits(bufs[1]))
    assert torch.isnan(bufs[0][:, n_out:].float()).all() and torch.isnan(bufs[0][M:].float()).all()
    assert not torch.isnan(bufs[0][:M, :n_out].float()).any()

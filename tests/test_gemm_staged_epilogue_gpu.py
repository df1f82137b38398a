"""The GEMM's staged epilogue variants across the tiles of a persistent CTA, bit for bit against the generic epilogue.

A variant takes its row factors from a shared-memory double buffer, its residual or RoPE table entries from a two-slot
shared-memory ring filled by TMA, and writes each slot through a per-warp pair of staging tiles stored by TMA.  At the
small shapes of test_gemm_epilogue_gpu.py a CTA gets at most one tile, so the buffers' phases never wrap.  Here every
CTA runs several tiles (M = 4096 + 77, N = 3072 + 96: M and N tails), with K = 64 (one k-block: the operand ring and the
staging tiles turn over faster than the k-loop) and K = 1024."""
import pytest
import torch

from test_gemm_epilogue_gpu import DT_IDS, STORAGE_TYPES, VARIANTS, WIDTHS, _bits, _run
from videollama2_b200 import ops

pytestmark = pytest.mark.gpu

M, N = 4096 + 77, 3072 + 96
D_HEAD = 64


@pytest.fixture(autouse=True)
def _needs_device(cuda):
    return cuda


def _case(variant, K, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, generator=g, device="cuda").to(dt)
    w = (torch.randn(N, K, generator=g, device="cuda") * K ** -0.5).to(dt)
    bias = torch.randn(N, generator=g, device="cuda")
    res = torch.randn(M, N, generator=g, device="cuda").to(dt)
    rms = torch.rand(M, 4, generator=g, device="cuda") * K * 0.5 + 1.0
    kw, n_out = {}, N
    if variant == "rms":
        kw = {"rms_in": rms, "rms_eps": 1e-5}
    elif variant == "bias":
        kw = {"bias": bias}
    elif variant.startswith("bias_act"):
        act = {"quick_gelu": ops.ACT_QUICK_GELU, "silu": ops.ACT_SILU, "gelu_erf": ops.ACT_GELU_ERF,
               "gelu_tanh": ops.ACT_GELU_TANH}[variant[len("bias_act_"):]]
        kw = {"bias": bias, "act": act}
    elif variant == "bias_res":
        kw = {"bias": bias, "residual": res}
    elif variant == "res_sumsq":
        kw = {"residual": res, "sumsq_out": None}
    elif variant in ("rope", "bias_rope"):
        tab = ops.rope_table(5 + M + 1, D_HEAD, 1e6, "cuda", dt)
        kw = {"rms_in": rms, "rms_eps": 1e-5, "rope": (tab, 5, D_HEAD, (N // 2 // D_HEAD) * D_HEAD)}
        if variant == "bias_rope":
            kw["bias"] = bias
    elif variant == "swiglu":
        kw, n_out = {"act": ops.ACT_SWIGLU, "rms_in": rms, "rms_eps": 1e-5}, N // 2
    else:
        assert variant == "none"
    return a, w, kw, n_out


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("K", [64, 1024])
@pytest.mark.parametrize("bn", WIDTHS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_variant_matches_generic_over_many_tiles(variant, bn, K, dt):
    a, w, kw, n_out = _case(variant, K, dt, seed=VARIANTS.index(variant) + K)
    fast, sq_fast = _run(a, w, kw, n_out, bn, False)
    slow, sq_slow = _run(a, w, kw, n_out, bn, True)
    torch.cuda.synchronize()
    assert not torch.isnan(slow.float()).any(), "the generic epilogue left outputs unwritten"
    assert torch.equal(_bits(fast), _bits(slow))
    if sq_fast is not None:
        assert torch.equal(_bits(sq_fast), _bits(sq_slow))


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=DT_IDS.get)
@pytest.mark.parametrize("bn", [96, 1256])
def test_residual_aliasing_output_over_many_tiles(bn, dt):
    """The residual is the output buffer itself: each tile's residual slots reach shared memory before its stores."""
    for variant in ("bias_res", "res_sumsq"):
        a, w, kw, n_out = _case(variant, 64, dt, seed=5)
        x = kw["residual"].clone()
        _, sq = _run(a, w, dict(kw, residual=x), n_out, bn, False, out=x)
        ref, sq_ref = _run(a, w, kw, n_out, bn, True)
        torch.cuda.synchronize()
        assert torch.equal(_bits(x), _bits(ref)), variant
        if sq is not None:
            assert torch.equal(_bits(sq), _bits(sq_ref)), variant

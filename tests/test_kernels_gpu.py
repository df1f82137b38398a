"""Kernel-level parity on the GPU: every libvl2 entry point against a plain PyTorch fp32 restatement of the same op
(inputs bf16-rounded, math fp32).  Tolerances are written per test; integer/index work is exact."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def relerr(a, b):
    a = a.float()
    b = b.float()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def rnd(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).to(dev)


ACTS = {
    0: lambda x: x,
    1: lambda x: x * torch.sigmoid(1.702 * x),
    2: torch.nn.functional.silu,
    3: lambda x: torch.nn.functional.gelu(x),
    5: lambda x: torch.nn.functional.gelu(x, approximate="tanh"),
}


@pytest.mark.parametrize("M,N,K", [
    (128, 256, 64), (128, 128, 128), (256, 64, 192), (200, 264, 136), (1, 8, 8), (577, 1024, 1024),
    (1776, 4096, 1024), (1521, 512, 2048), (333, 3072, 640),
])
def test_gemm_plain(cuda, M, N, K):
    from videollama2_b200 import ops
    a = rnd((M, K), cuda, seed=1)
    w = rnd((N, K), cuda, 0.05, seed=2)
    out = ops.gemm(a, w)
    ref = a.float() @ w.float().t()
    assert relerr(out, ref) < 6e-3, (M, N, K)


@pytest.mark.parametrize("bn", [64, 96, 128, 160, 192, 224, 256])
def test_gemm_every_tile_width(cuda, bn):
    """Each instantiated tile width, multi-tile persistent loop (tiles > SMs for the narrow ones), M/N/K tails."""
    from videollama2_b200 import ops
    M, N, K = 1100, 2072, 328
    a = rnd((M, K), cuda, seed=40)
    w = rnd((N, K), cuda, 0.06, seed=41)
    bias = torch.randn(N, device=cuda)
    res = rnd((M, N), cuda, seed=42)
    out = ops.gemm(a, w, bias=bias, act=ops.ACT_SILU, residual=res, bn=bn)
    ref = torch.nn.functional.silu(a.float() @ w.float().t() + bias) + res.float()
    assert relerr(out, ref) < 6e-3, bn


@pytest.mark.parametrize("bn", [128, 160, 192, 224, 256])
@pytest.mark.parametrize("M,N,K", [(1100, 2072, 328), (100, 512, 64), (130, 264, 136), (256, 256, 64), (9232, 1024, 192)])
def test_gemm_cta_pair_kernel(cuda, bn, M, N, K):
    """Two-CTA cluster kernel (two CTAs per 256 x BN tile, B tile multicast to both): every width; persistent multi-tile
    loops; M tails where the peer CTA's half is partly or entirely out of bounds; N/K tails."""
    from videollama2_b200 import ops
    a = rnd((M, K), cuda, seed=60)
    w = rnd((N, K), cuda, 0.06, seed=61)
    bias = torch.randn(N, device=cuda)
    res = rnd((M, N), cuda, seed=62)
    out = ops.gemm(a, w, bias=bias, act=ops.ACT_QUICK_GELU, residual=res, bn=1000 + bn)
    x = a.float() @ w.float().t() + bias
    ref = x * torch.sigmoid(1.702 * x) + res.float()
    assert relerr(out, ref) < 6e-3, (bn, M, N, K)


def test_gemm_cta_pair_swiglu_and_f32(cuda):
    from videollama2_b200 import ops
    M, I, K = 1776, 640, 256
    a = rnd((M, K), cuda, seed=63)
    gate, up = rnd((I, K), cuda, 0.1, seed=64), rnd((I, K), cuda, 0.1, seed=65)
    w = torch.stack([gate, up], dim=1).reshape(2 * I, K).contiguous()
    out = ops.gemm(a, w, act=ops.ACT_SWIGLU, bn=1256)
    ref = torch.nn.functional.silu(a.float() @ gate.float().t()) * (a.float() @ up.float().t())
    assert relerr(out, ref) < 8e-3
    o32 = ops.gemm(a, gate, out_dtype=torch.float32, bn=1224)
    assert relerr(o32, a.float() @ gate.float().t()) < 2e-3


@pytest.mark.parametrize("act", [0, 1, 2, 3, 5])
@pytest.mark.parametrize("with_res", [False, True])
def test_gemm_epilogue(cuda, act, with_res):
    from videollama2_b200 import ops
    M, N, K = 300, 520, 256
    a = rnd((M, K), cuda, seed=3)
    w = rnd((N, K), cuda, 0.08, seed=4)
    bias = torch.randn(N, device=cuda)
    res = rnd((M, N), cuda, seed=5) if with_res else None
    rs = torch.rand(M, device=cuda) + 0.5
    out = ops.gemm(a, w, bias=bias, act=act, residual=res, row_scale=rs)
    ref = ACTS[act]((a.float() @ w.float().t()) * rs[:, None] + bias)
    if with_res:
        ref = ref + res.float()
    assert relerr(out, ref) < 6e-3
    out32 = ops.gemm(a, w, bias=bias, act=act, residual=res, row_scale=rs, out_dtype=torch.float32)
    assert out32.dtype == torch.float32 and relerr(out32, ref) < 2e-3


@pytest.mark.parametrize("M,N,K,bn,kind", [
    (1776, 4096, 4096, 0, "res_sumsq"),      # decoder o_proj: 112 pair tiles on 66 pairs -> 46 tiles split
    (1776, 6144, 4096, 0, "bias"),           # decoder QKV: 196 pair tiles on 66 pairs -> 64 tiles split
    (1776, 4096, 1024, 1256, "plain"),       # short K: 16 k-blocks -> 2 slices of 8
    (1200, 4096, 2048, 256, "res_sumsq"),    # single-CTA tiles: 160 tiles on 132 SMs -> 28 tiles split in 4
    (1776, 28672, 512, 0, "swiglu"),         # SwiGLU epilogue on an owner tile
    (300, 520, 256, 0, "bias"),              # one round, short K: nothing to split
    (1154, 1024, 4096, 0, "res_sumsq"),      # ViT fc2 of a 2-frame shard: one partial round of pair tiles
    (1776, 4096, 14336, 0, "res_sumsq"),     # decoder down_proj
])
@pytest.mark.parametrize("slices", [2, 3, 4])
def test_gemm_splitk_tail(cuda, M, N, K, bn, kind, slices):
    """The last, partial round of the persistent grid is cut into K-slices (fp32 partials through the workspace, owner
    CTA adds them in a fixed order; `slices` = 2..4 K-slices per remaining tile, forced through the test hook; off by default in production): same result as the unsplit kernel up to fp32 summation order, bit-identical from
    launch to launch (the arrival counters re-arm themselves), and equal to the fp32 reference."""
    from videollama2_b200 import ops
    a = rnd((M, K), cuda, seed=11)
    w = rnd((N, K), cuda, K ** -0.5, seed=12)
    kw = {}
    n_out = N
    if kind == "bias":
        kw["bias"] = torch.randn(N, device=cuda)
    elif kind == "res_sumsq":
        kw["residual"] = rnd((M, N), cuda, seed=13)
        kw["sumsq_out"] = torch.empty((M, N // 32), device=cuda, dtype=torch.float32)
    elif kind == "swiglu":
        kw["act"] = ops.ACT_SWIGLU
        n_out = N // 2
    ref = a.float() @ w.float().t()
    if kind == "bias":
        ref = ref + kw["bias"]
    elif kind == "res_sumsq":
        ref = ref + kw["residual"].float()
    elif kind == "swiglu":
        ref = torch.nn.functional.silu(ref[:, 0::2]) * ref[:, 1::2]
    outs = []
    for _ in range(3):
        outs.append(ops.gemm(a, w, bn=bn, splitk=slices, **kw).clone())
        if kind == "res_sumsq":
            ss = kw["sumsq_out"].sum(1)
            assert relerr(ss, outs[-1].float().pow(2).sum(1)) < 1e-3
    assert outs[0].shape == (M, n_out)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    assert relerr(outs[0], ref) < 6e-3
    if kind == "res_sumsq":
        kw["sumsq_out"] = torch.empty((M, N // 32), device=cuda, dtype=torch.float32)
    unsplit = ops.gemm(a, w, bn=bn, splitk=False, **kw)
    assert relerr(outs[0], unsplit.float()) < 2e-3


def test_gemm_swiglu_and_strided(cuda):
    from videollama2_b200 import ops
    M, I, K = 260, 384, 128
    a_full = rnd((M, K + 64), cuda, seed=6)
    a = a_full[:, 32:32 + K]  # strided view, 64-byte aligned start
    gate = rnd((I, K), cuda, 0.1, seed=7)
    up = rnd((I, K), cuda, 0.1, seed=8)
    w = torch.stack([gate, up], dim=1).reshape(2 * I, K).contiguous()
    out = ops.gemm(a, w, act=ops.ACT_SWIGLU)
    ref = torch.nn.functional.silu(a.float() @ gate.float().t()) * (a.float() @ up.float().t())
    assert out.shape == (M, I) and relerr(out, ref) < 8e-3


def test_gemm_rejects_bad_args(cuda):
    from videollama2_b200 import ops
    a = rnd((16, 12), cuda)
    w = rnd((8, 12), cuda)
    with pytest.raises(ValueError):
        ops.gemm(a, w)  # K % 8 != 0


@pytest.mark.parametrize("B,S,Hq,Hkv,D,causal", [
    (2, 577, 4, 4, 64, False), (1, 128, 2, 2, 64, False), (3, 45, 2, 2, 64, False),
    (1, 300, 4, 2, 128, True), (1, 1776, 8, 2, 128, True), (1, 128, 2, 1, 128, True), (2, 260, 2, 2, 64, True),
    # head widths between the native 64 / 128 (SigLIP-so400m: 16 heads x 72): heads packed at their true width
    (3, 729, 16, 16, 72, False), (2, 25, 2, 2, 72, False), (1, 200, 4, 2, 96, True), (2, 130, 3, 3, 40, False),
    (1, 77, 2, 2, 8, False),
    # Qwen2-7B geometry: 28 query heads over 4 kv heads (GQA group 7), full config-3 sequence length
    (1, 1776, 28, 4, 128, True), (1, 300, 14, 2, 128, True), (2, 130, 7, 1, 64, False),
])
def test_attention(cuda, B, S, Hq, Hkv, D, causal):
    from videollama2_b200 import ops
    qkv = rnd((B * S, (Hq + 2 * Hkv) * D), cuda, 1.0, seed=9)
    q = qkv[:, : Hq * D]
    k = qkv[:, Hq * D: (Hq + Hkv) * D]
    v = qkv[:, (Hq + Hkv) * D:]
    scale = 1.0 / math.sqrt(D)
    out = ops.attention(q, k, v, B=B, S=S, Hq=Hq, Hkv=Hkv, D=D, causal=causal, scale=scale)
    qf = q.float().view(B, S, Hq, D).transpose(1, 2)
    kf = k.float().view(B, S, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    vf = v.float().view(B, S, Hkv, D).transpose(1, 2).repeat_interleave(Hq // Hkv, dim=1)
    s = (qf @ kf.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(S, S, device=cuda, dtype=torch.bool).triu(1), float("-inf"))
    ref = (torch.softmax(s, dim=-1) @ vf).transpose(1, 2).reshape(B * S, Hq * D)
    assert relerr(out, ref) < 8e-3, (B, S, Hq, Hkv, D, causal)


@pytest.mark.parametrize("rows,C", [(9232, 1024), (1521, 4096), (7, 128), (33, 3584)])
@pytest.mark.parametrize("act,with_res", [(0, False), (2, False), (2, True)])
def test_layernorm(cuda, rows, C, act, with_res):
    from videollama2_b200 import ops
    x = rnd((rows, C), cuda, 2.0, seed=10) + 0.5
    g = rnd((C,), cuda, 0.1, seed=11) + 1.0
    b = rnd((C,), cuda, 0.1, seed=12)
    res = rnd((rows, C), cuda, seed=13) if with_res else None
    y = ops.layernorm(x, g, b, 1e-5, act=act, residual=res)
    ref = torch.nn.functional.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)
    if with_res:
        ref = ref + res.float()
    if act == 2:
        ref = torch.nn.functional.silu(ref)
    assert relerr(y, ref) < 4e-3


@pytest.mark.parametrize("rows,C", [(1776, 4096), (5, 128), (64, 3584)])
def test_rmsnorm(cuda, rows, C):
    from videollama2_b200 import ops
    x = rnd((rows, C), cuda, 3.0, seed=14)
    g = rnd((C,), cuda, 0.1, seed=15) + 1.0
    y = ops.rmsnorm(x, g, 1e-5)
    xf = x.float()
    ref = g.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))
    assert relerr(y, ref) < 4e-3


@pytest.mark.parametrize("F,H,P,C", [(2, 336, 14, 1024), (3, 56, 14, 64)])
def test_patch_embed_path(cuda, F, H, P, C):
    from videollama2_b200 import ops
    px = rnd((F, 3, H, H), cuda, seed=16)
    wconv = rnd((C, 3, P, P), cuda, 0.05, seed=17)
    K = 3 * P * P
    Kpad = (K + 63) // 64 * 64
    A = ops.patch_im2col(px, P, Kpad)
    ref_A = torch.nn.functional.unfold(px.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, K)
    assert torch.equal(A[:, :K].float(), ref_A) and A[:, K:].abs().max().item() == 0  # pure data movement: exact
    wpad = torch.zeros((C, Kpad), device=cuda, dtype=torch.bfloat16)
    wpad[:, :K] = wconv.reshape(C, K)
    patch = ops.gemm(A, wpad)
    ref_patch = torch.nn.functional.conv2d(px.float(), wconv.float(), stride=P).flatten(2).transpose(1, 2).reshape(-1, C)
    assert relerr(patch, ref_patch) < 6e-3
    np_ = (H // P) ** 2
    cls = rnd((C,), cuda, seed=18)
    pos = rnd((np_ + 1, C), cuda, seed=19)
    g = rnd((C,), cuda, 0.1, seed=20) + 1
    b = rnd((C,), cuda, 0.1, seed=21)
    tok = ops.clip_embed_finish(patch, cls, pos, g, b, F, 1e-5)
    emb = torch.cat([cls.float().expand(F, 1, C), patch.float().view(F, np_, C)], 1) + pos.float()
    ref_tok = torch.nn.functional.layer_norm(emb, (C,), g.float(), b.float(), 1e-5).reshape(-1, C)
    assert relerr(tok, ref_tok) < 4e-3


@pytest.mark.parametrize("F,H,W,C", [(2, 24, 24, 4096), (3, 13, 13, 512), (1, 4, 5, 64), (2, 13, 13, 8192), (1, 6, 7, 8192),
                                     (1, 24, 24, 6144)])
def test_dwconv_ln_silu_pool_scale(cuda, F, H, W, C):
    from videollama2_b200 import ops
    x = rnd((F, H, W, C), cuda, seed=22)
    wd = rnd((C, 1, 3, 3), cuda, 0.3, seed=23)
    g = rnd((C,), cuda, 0.1, seed=24) + 1
    b = rnd((C,), cuda, 0.1, seed=25)
    w9c = wd.reshape(C, 9).t().contiguous()
    y, pooled = ops.dwconv3x3_ln_silu(x, w9c, g, b, 1e-5)
    conv = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wd.float(), padding=1, groups=C).permute(0, 2, 3, 1)
    ref = torch.nn.functional.silu(torch.nn.functional.layer_norm(conv, (C,), g.float(), b.float(), 1e-5))
    assert relerr(y, ref) < 5e-3
    assert relerr(pooled, y.float().mean(dim=(1, 2))) < 1e-5  # pooling of what was written: fp32-exact up to order
    s = torch.rand((F, C), device=cuda)
    y2 = ops.se_scale(y.clone(), s)
    assert relerr(y2, y.float() * s[:, None, None, :]) < 4e-3


@pytest.mark.parametrize("pad", [1, 0])
@pytest.mark.parametrize("T,H,W,C", [(4, 6, 6, 64), (16, 24, 24, 128), (3, 5, 7, 8)])
def test_conv3d_path(cuda, pad, T, H, W, C):
    from videollama2_b200 import ops
    x = rnd((T, H, W, C), cuda, seed=26)
    wc = rnd((C, C, 2, 2, 2), cuda, 0.1, seed=27)
    bias = torch.randn(C, device=cuda)
    A = ops.conv3d_im2col(x, pad)
    wk = wc.permute(0, 2, 3, 4, 1).reshape(C, 8 * C).contiguous()
    out = ops.gemm(A, wk, bias=bias, act=ops.ACT_SILU)
    ref = torch.nn.functional.conv3d(x.float().permute(3, 0, 1, 2)[None], wc.float(), bias, stride=2, padding=pad)
    ref = torch.nn.functional.silu(ref)[0].permute(1, 2, 3, 0).reshape(-1, C)
    assert out.shape == ref.shape and relerr(out, ref) < 6e-3


def test_skinny_gemm(cuda):
    from videollama2_b200 import ops
    a = torch.randn((16, 4096), device=cuda)
    w = rnd((1024, 4096), cuda, 0.05, seed=28)
    bias = torch.randn(1024, device=cuda)
    for act, fn in ((ops.ACT_NONE, lambda t: t), (ops.ACT_SILU, torch.nn.functional.silu), (ops.ACT_SIGMOID, torch.sigmoid)):
        out = ops.gemm_skinny(a, w, bias=bias, act=act)
        # fp32 A is staged as bf16 (the reference's own activation dtype): compare against the bf16-rounded input
        assert relerr(out, fn(a.bfloat16().float() @ w.float().t() + bias)) < 1e-4
    ab = rnd((1, 4096), cuda, seed=29)
    out = ops.gemm_skinny(ab, w, out_dtype=torch.bfloat16)
    assert relerr(out, ab.float() @ w.float().t()) < 4e-3


def test_rope(cuda):
    from videollama2_b200 import ops
    S, Hq, Hkv, D = 300, 4, 2, 128
    qkv = rnd((S, (Hq + 2 * Hkv) * D), cuda, seed=30)
    orig = qkv.clone()
    inv_freq = 1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    ops.rope_inplace(qkv, S, Hq, Hkv, D, 0, Hq * D, 7, inv_freq.to(cuda))
    pos = torch.arange(7, 7 + S, dtype=torch.float32)
    fr = torch.outer(pos, inv_freq)
    emb = torch.cat([fr, fr], -1)
    cos, sin = emb.cos().to(cuda), emb.sin().to(cuda)

    def rot(x):
        return torch.cat([-x[..., D // 2:], x[..., : D // 2]], -1)

    qk = orig[:, : (Hq + Hkv) * D].float().view(S, Hq + Hkv, D)
    ref = qk * cos[:, None, :] + rot(qk) * sin[:, None, :]
    assert relerr(qkv[:, : (Hq + Hkv) * D], ref.reshape(S, -1)) < 5e-3
    assert torch.equal(qkv[:, (Hq + Hkv) * D:], orig[:, (Hq + Hkv) * D:])  # V untouched: exact


def test_embed_splice_exact(cuda):
    from videollama2_b200 import ops
    V, H = 1000, 256
    table = rnd((V, H), cuda, seed=31)
    ids = torch.tensor([5, 999, -201, 0, 17], dtype=torch.int64, device=cuda)
    dst = torch.tensor([0, 1, 2, 50, 51], dtype=torch.int32, device=cuda)
    out = torch.full((52, H), 7.0, device=cuda, dtype=torch.bfloat16)
    ops.embed_splice(ids, dst, table, out)
    torch.cuda.synchronize()
    assert torch.equal(out[0], table[5]) and torch.equal(out[1], table[999])
    assert torch.equal(out[50], table[0]) and torch.equal(out[51], table[17])
    assert (out[2:50] == 7.0).all()  # placeholder row and untouched rows stay as they were


def test_skinny_gemm_residual_swiglu_out(cuda):
    from videollama2_b200 import ops
    x = rnd((1, 512), cuda, seed=50)
    w = rnd((256, 512), cuda, 0.05, seed=51)
    res = rnd((1, 256), cuda, seed=52)
    out = ops.gemm_skinny(x, w, residual=res, out_dtype=torch.bfloat16)
    assert relerr(out, x.float() @ w.float().t() + res.float()) < 4e-3
    gate, up = rnd((96, 512), cuda, 0.05, seed=53), rnd((96, 512), cuda, 0.05, seed=54)
    wgu = torch.stack([gate, up], 1).reshape(192, 512).contiguous()
    h = ops.gemm_skinny(x, wgu, act=ops.ACT_SWIGLU, out_dtype=torch.bfloat16)
    ref = torch.nn.functional.silu(x.float() @ gate.float().t()) * (x.float() @ up.float().t())
    assert h.shape == (1, 96) and relerr(h, ref) < 5e-3
    buf = torch.zeros((3, 256), device=cuda, dtype=torch.bfloat16)
    ops.gemm_skinny(x, w, out=buf[1:2])
    assert relerr(buf[1], (x.float() @ w.float().t())[0]) < 4e-3 and buf[0].abs().max() == 0 and buf[2].abs().max() == 0


@pytest.mark.parametrize("N,K", [(4096, 4096), (1000, 328), (28672, 4096), (4096, 14336), (37, 8), (152064, 3584)])
@pytest.mark.parametrize("mode", ["plain", "rms_bias", "swiglu_rms", "residual", "f32out"])
def test_gemv(cuda, N, K, mode):
    """M = 1 weight-streaming GEMV with the fused RMSNorm scale / bias / SwiGLU / residual epilogues."""
    from videollama2_b200 import ops
    if mode == "swiglu_rms" and N % 2:
        pytest.skip("SwiGLU needs even N")
    x = rnd((1, K), cuda, 1.5, seed=91)
    w = rnd((N, K), cuda, K ** -0.5, seed=92)
    xf, wf = x.float(), w.float()
    eps = 1e-5
    s = torch.rsqrt((xf * xf).mean() + eps)
    if mode == "plain":
        out, ref = ops.gemv(x, w), xf @ wf.t()
    elif mode == "rms_bias":
        b = rnd((N,), cuda, 0.1, seed=93).float()
        out, ref = ops.gemv(x, w, bias=b, rms_eps=eps), s * (xf @ wf.t()) + b
    elif mode == "swiglu_rms":
        out = ops.gemv(x, w, act=ops.ACT_SWIGLU, rms_eps=eps)
        y = s * (xf @ wf.t())
        ref = torch.nn.functional.silu(y[:, 0::2]) * y[:, 1::2]
    elif mode == "residual":
        r = rnd((1, N), cuda, 1.0, seed=94)
        out, ref = ops.gemv(x, w, residual=r), xf @ wf.t() + r.float()
    else:
        out, ref = ops.gemv(x, w, out_dtype=torch.float32), xf @ wf.t()
        assert out.dtype == torch.float32
    assert out.shape == ref.shape
    assert relerr(out, ref) < (2e-5 if mode == "f32out" else 4e-3)
    # M = 1 through the skinny entry point takes the same kernel
    if mode == "plain":
        assert torch.equal(ops.gemm_skinny(x, w, out_dtype=torch.bfloat16), out)


@pytest.mark.parametrize("n_pos,Hq,Hkv,D", [(1, 4, 2, 128), (37, 4, 2, 128), (1777, 32, 8, 128), (300, 4, 4, 64), (5000, 2, 1, 128),
                                            (128, 8, 8, 128), (129, 28, 4, 128), (1607, 28, 4, 128), (9000, 16, 2, 64),
                                            (40000, 8, 1, 128)])
def test_attention_decode(cuda, n_pos, Hq, Hkv, D):
    from videollama2_b200 import ops
    width = (Hq + 2 * Hkv) * D
    cache = rnd((n_pos + 3, width), cuda, seed=55)
    q = cache[n_pos - 1, : Hq * D].contiguous()
    k = cache[:, Hq * D: (Hq + Hkv) * D]
    v = cache[:, (Hq + Hkv) * D:]
    out = ops.attention_decode(q, k, v, n_pos=n_pos, Hq=Hq, Hkv=Hkv, D=D, scale=D ** -0.5)
    qf = q.float().view(Hq, 1, D)
    kf = k[:n_pos].float().view(n_pos, Hkv, D).permute(1, 0, 2).repeat_interleave(Hq // Hkv, 0)
    vf = v[:n_pos].float().view(n_pos, Hkv, D).permute(1, 0, 2).repeat_interleave(Hq // Hkv, 0)
    ref = (torch.softmax(qf @ kf.transpose(1, 2) * D ** -0.5, -1) @ vf).reshape(1, Hq * D)
    assert relerr(out, ref) < 6e-3
    # graph-replayable variant (position read from device memory) is bit-identical
    pos_dev = torch.tensor([n_pos - 1], device=cuda, dtype=torch.int32)
    out2 = torch.empty_like(out)
    ops.attention_decode_dyn(q, k, v, pos_dev, Hq=Hq, Hkv=Hkv, D=D, scale=D ** -0.5, out=out2)
    assert torch.equal(out, out2)


def test_decode_rope_append_matches_eager(cuda):
    from videollama2_b200 import ops
    Hq, Hkv, D, pos = 8, 2, 128, 77
    width = (Hq + 2 * Hkv) * D
    row = rnd((1, width), cuda, seed=61)
    inv = (1.0 / (1e6 ** (torch.arange(0, D, 2).float() / D))).to(cuda)
    eager = row.clone()
    ops.rope_inplace(eager, 1, Hq, Hkv, D, 0, Hq * D, pos, inv)
    cache = torch.zeros((100, width), device=cuda, dtype=torch.bfloat16)
    stage = row.clone()
    ops.decode_rope_append(stage, cache, torch.tensor([pos], device=cuda, dtype=torch.int32), Hq, Hkv, D, inv)
    assert torch.equal(stage, eager) and torch.equal(cache[pos:pos + 1], eager)
    assert int(cache[:pos].abs().sum()) == 0 and int(cache[pos + 1:].abs().sum()) == 0


@pytest.mark.parametrize("bn", [0, 1256, 224])
def test_gemm_folded_rmsnorm(cuda, bn):
    """rmsnorm(x; g) W^T through the GEMM: gains folded into W, 1/rms applied per row in the epilogue, the output's
    sums of squares written as per-32-column partials (deterministic: no atomics)."""
    from videollama2_b200 import ops
    M, N, K = 700, 1056, 512
    x = rnd((M, K), cuda, 2.0, seed=70)
    g = rnd((K,), cuda, 0.1, seed=71) + 1.0
    w = rnd((N, K), cuda, 0.05, seed=72)
    res = rnd((M, N), cuda, seed=73)
    wf = (w.float() * g.float()[None, :]).to(torch.bfloat16)
    ss = ops.row_sumsq(x)
    assert ss.shape == (M, 1) and relerr(ss[:, 0], x.float().pow(2).sum(-1)) < 1e-5
    parts = torch.full((M, N // 32), 7.0, device=cuda)
    out = ops.gemm(x, wf, residual=res, rms_in=ss, rms_eps=1e-5, sumsq_out=parts, bn=bn)
    xf = x.float()
    ref = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * g.float()) @ w.float().t() + res.float()
    assert relerr(out, ref) < 8e-3
    assert relerr(parts.sum(-1), out.float().pow(2).sum(-1)) < 1e-4
    # chained: the partials feed the next folded norm
    w2 = rnd((64, N), cuda, 0.03, seed=74)
    y = ops.gemm(out, w2, rms_in=parts, rms_eps=1e-5, bn=bn)
    of = out.float()
    assert relerr(y, (of * torch.rsqrt(of.pow(2).mean(-1, keepdim=True) + 1e-5)) @ w2.float().t()) < 8e-3


@pytest.mark.parametrize("M,N,K,bn", [(1154, 3072, 1024, 0), (9232, 4096, 1024, 0), (300, 288, 288, 0), (577, 256, 128, 64),
                                      (1154, 1024, 1024, 1128), (260, 2304, 1152, 224)])
@pytest.mark.parametrize("stats_from", ["row_kernel", "gemm_epilogue"])
def test_gemm_folded_layernorm(cuda, M, N, K, bn, stats_from):
    """LayerNorm folded into the consuming GEMM (vl2_gemm_args.ln_sum_in / ln_colsum): rstd * (x W'^T - mu * colsum) + b'
    against layer_norm + linear in fp32; the row statistics come from vl2_row_stats or from the producing GEMM's epilogue
    (rowsum_out / sumsq_out), which must equal the sums of the bf16 outputs."""
    from videollama2_b200 import ops
    g = (rnd((K,), cuda, 0.1, seed=71) + 1.0).float()
    beta = rnd((K,), cuda, 0.2, seed=72).float()
    w = rnd((N, K), cuda, K ** -0.5, seed=73)
    b = rnd((N,), cuda, 0.1, seed=74).float()
    if stats_from == "row_kernel":
        x = rnd((M, K), cuda, 1.5, seed=75) + 0.75                   # mean well away from zero: mu * colsum matters
        stats = ops.row_stats(x)
    else:
        if K % 32:
            pytest.skip("epilogue statistics need N % 32 == 0")
        a0 = rnd((M, 64), cuda, seed=76)
        w0 = rnd((K, 64), cuda, 0.2, seed=77)
        res = rnd((M, K), cuda, 1.0, seed=78) + 0.5
        stats = (torch.empty((M, K // 32), device=cuda, dtype=torch.float32), torch.empty((M, K // 32), device=cuda, dtype=torch.float32))
        x = ops.gemm(a0, w0, residual=res, rowsum_out=stats[0], sumsq_out=stats[1])
        assert relerr(stats[0].sum(-1), x.float().sum(-1)) < 1e-5 and relerr(stats[1].sum(-1), x.float().pow(2).sum(-1)) < 1e-5
    wf = (w.float() * g[None, :]).to(torch.bfloat16)
    out = ops.gemm(x, wf, bias=(b + w.float() @ beta).contiguous(), ln_in=stats, ln_colsum=wf.float().sum(1).contiguous(),
                   rms_eps=1e-5, bn=bn)
    ref = torch.nn.functional.layer_norm(x.float(), (K,), g, beta, 1e-5) @ w.float().t() + b
    assert relerr(out, ref) < 8e-3


@pytest.mark.parametrize("pad", [1, 0])
@pytest.mark.parametrize("T,H,W,C,N,bn", [(16, 24, 24, 4096, 512, 0), (4, 6, 6, 64, 64, 0), (8, 27, 27, 128, 256, 0), (3, 5, 7, 64, 96, 0),
                                          (16, 24, 24, 256, 512, 1256), (16, 24, 24, 256, 512, 128), (2, 30, 30, 64, 64, 0)])
def test_conv3d_implicit_gemm(cuda, T, H, W, C, N, bn, pad):
    """The Conv3d(k=s=2) front end of vl2_gemm_bf16 (TMA gathers the taps from x, out-of-bounds = zero padding) equals the
    explicit tap-gather + GEMM BIT FOR BIT (same K order) and nn.functional.conv3d within bf16 tolerance."""
    from videollama2_b200 import ops
    if (W % 2 == 1 or H % 2 == 1) and pad == 1:
        pytest.skip("odd H / W with padding is not a configuration of the path")
    x = rnd((T, H, W, C), cuda, seed=81)
    wt = rnd((N, C, 2, 2, 2), cuda, (8 * C) ** -0.5, seed=82)
    b = rnd((N,), cuda, 0.1, seed=83).float()
    wk = wt.permute(0, 2, 3, 4, 1).reshape(N, 8 * C).contiguous()
    out = ops.conv3d_k2s2(x, wk, bias=b, act=ops.ACT_SILU, pad=pad, bn=bn)
    explicit = ops.gemm(ops.conv3d_im2col(x, pad), wk, bias=b, act=ops.ACT_SILU)
    assert torch.equal(out, explicit)
    ref = torch.nn.functional.conv3d(x.float().permute(3, 0, 1, 2)[None], wt.float(), b, stride=2, padding=pad)
    ref = torch.nn.functional.silu(ref)[0].permute(1, 2, 3, 0).reshape(-1, N)
    assert out.shape == ref.shape and relerr(out, ref) < 8e-3


def test_conv3d_implicit_gemm_rejects_bad_shapes(cuda):
    from videollama2_b200 import ops
    x = rnd((4, 40, 40, 64), cuda)                                   # 21 output columns > 16 per padded line
    with pytest.raises((ValueError, NotImplementedError)):
        ops.conv3d_k2s2(x, rnd((64, 512), cuda), pad=1)
    with pytest.raises(ValueError):
        ops.conv3d_k2s2(rnd((4, 8, 8, 64), cuda), rnd((64, 256), cuda), pad=1)     # K != 8*C


@pytest.mark.parametrize("S,Hq,Hkv,D,pos0,bn", [(1776, 8, 2, 128, 0, 0), (300, 28, 4, 128, 5, 0), (130, 4, 2, 64, 0, 64),
                                               (260, 2, 1, 128, 17, 1256), (77, 4, 4, 32, 3, 0)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_gemm_rope_epilogue(cuda, S, Hq, Hkv, D, pos0, bn, with_bias):
    """RoPE fused into the QKV GEMM epilogue on permuted (adjacent-pair) columns == HF apply_rotary_pos_emb
    (rotate-half pairing, HF:mistral/modeling_mistral.py:51-82) on the un-permuted projection, up to the column
    permutation; v columns untouched; vl2_rope_inplace(interleaved=1) reproduces the epilogue's layout."""
    from videollama2_b200 import ops
    K = 256
    nqk, nv = (Hq + Hkv) * D, Hkv * D
    x = rnd((S, K), cuda, seed=91)
    w = rnd((nqk + nv, K), cuda, K ** -0.5, seed=92)
    b = rnd((nqk + nv,), cuda, 0.1, seed=93).float() if with_bias else None
    perm = torch.cat([ops.rope_interleave_rows(Hq + Hkv, D), torch.arange(nqk, nqk + nv)]).to(cuda)
    tab = ops.rope_table(pos0 + S + 3, D, 1e6, cuda)
    out = ops.gemm(x, w[perm].contiguous(), bias=None if b is None else b[perm].contiguous(), rope=(tab, pos0, D, nqk), bn=bn)
    # reference: plain projection, HF rotation, then the same permutation
    y = x.float() @ w.float().t() + (0 if b is None else b)
    inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, device=cuda).float() / D))
    ang = torch.outer(torch.arange(pos0, pos0 + S, device=cuda).float(), inv)
    cos = torch.cat([ang, ang], -1).cos().to(torch.bfloat16).float()
    sin = torch.cat([ang, ang], -1).sin().to(torch.bfloat16).float()
    qk = y[:, :nqk].view(S, Hq + Hkv, D)
    rot = torch.cat([-qk[..., D // 2:], qk[..., :D // 2]], -1)
    ref = torch.cat([(qk * cos[:, None] + rot * sin[:, None]).reshape(S, nqk), y[:, nqk:]], 1)[:, perm]
    assert relerr(out, ref) < 6e-3
    assert relerr(out[:, nqk:], y[:, nqk:]) < 6e-3
    # the stand-alone kernel in interleaved mode on the un-rotated projection gives the same layout
    plain = ops.gemm(x, w[perm].contiguous(), bias=None if b is None else b[perm].contiguous(), bn=bn)
    inv_dev = inv.contiguous()
    ops.rope_inplace(plain, S, Hq, Hkv, D, 0, Hq * D, pos0, inv_dev, interleaved=True)
    assert relerr(plain, ref) < 8e-3


@pytest.mark.parametrize("F,H,P,C", [(2, 336, 14, 1024), (3, 56, 14, 128), (1, 112, 14, 256), (16, 336, 14, 1024)])
def test_patch_embed_fused_clip(cuda, F, H, P, C):
    """vl2_patch_embed (patch gather -> wgmma conv -> + position -> class row -> pre-LayerNorm in ONE kernel) against
    conv2d + cat(cls) + position + layer_norm in fp32, and against the three-kernel explicit path it replaces."""
    from videollama2_b200 import ops
    px = rnd((F, 3, H, H), cuda, seed=16)
    wconv = rnd((C, 3, P, P), cuda, 0.05, seed=17)
    K = 3 * P * P
    Kpad = (K + 63) // 64 * 64
    wpad = torch.zeros((C, Kpad), device=cuda, dtype=torch.bfloat16)
    wpad[:, :K] = wconv.reshape(C, K)
    np_ = (H // P) ** 2
    cls = rnd((C,), cuda, seed=18)
    pos = rnd((np_ + 1, C), cuda, seed=19)
    g = rnd((C,), cuda, 0.1, seed=20) + 1
    b = rnd((C,), cuda, 0.1, seed=21)
    tok = ops.patch_embed(px, wpad, pos, P, cls=cls, gamma=g, beta=b, eps=1e-5)
    patch = torch.nn.functional.conv2d(px.float(), wconv.float(), stride=P).flatten(2).transpose(1, 2)
    emb = torch.cat([cls.float().expand(F, 1, C), patch], 1) + pos.float()
    ref = torch.nn.functional.layer_norm(emb, (C,), g.float(), b.float(), 1e-5).reshape(-1, C)
    assert tok.shape == ref.shape and relerr(tok, ref) < 5e-3
    explicit = ops.clip_embed_finish(ops.gemm(ops.patch_im2col(px, P, Kpad), wpad), cls, pos, g, b, F, 1e-5)
    assert relerr(tok, explicit.float()) < 3e-3
    assert torch.equal(tok.view(F, np_ + 1, C)[0, 0], tok.view(F, np_ + 1, C)[F - 1, 0])      # class rows identical


@pytest.mark.parametrize("F,H,P,C", [(2, 384, 14, 1152), (3, 70, 14, 288)])
def test_patch_embed_fused_siglip(cuda, F, H, P, C):
    """SigLIP form: conv + bias + position rows, no class token, no LayerNorm (27 x 27 patches out of 384 pixels: 6 unused)."""
    from videollama2_b200 import ops
    px = rnd((F, 3, H, H), cuda, seed=26)
    wconv = rnd((C, 3, P, P), cuda, 0.05, seed=27)
    K = 3 * P * P
    Kpad = (K + 63) // 64 * 64
    wpad = torch.zeros((C, Kpad), device=cuda, dtype=torch.bfloat16)
    wpad[:, :K] = wconv.reshape(C, K)
    np_ = (H // P) ** 2
    pos = rnd((np_, C), cuda, seed=29)
    bias = rnd((C,), cuda, 0.2, seed=30).float()
    tok = ops.patch_embed(px, wpad, pos, P, bias=bias)
    patch = torch.nn.functional.conv2d(px.float(), wconv.float(), bias, stride=P).flatten(2).transpose(1, 2)
    ref = (patch + pos.float()).reshape(-1, C)
    assert tok.shape == ref.shape and relerr(tok, ref) < 4e-3


@pytest.mark.parametrize("bn", [64, 96, 128, 160, 192, 224, 256, 1128, 1160, 1192, 1224, 1256])
@pytest.mark.parametrize("kind", ["bias_act_res", "rms_stats", "swiglu", "plain_tail", "inplace_strided"])
def test_gemm_epilogue_kinds_agree_across_tiles(cuda, bn, kind):
    """Every epilogue family on a forced tile (single-CTA widths and two-CTA pair tiles) against the tile the cost model
    picks on the same launch: same arithmetic per output element, so the outputs agree up to FMA contraction and the
    k-block order of the accumulation, and both against the fp32 restatement.  M / N tails, several tiles per CTA, an
    output that aliases the residual inside a wider buffer (nothing outside the slice may be written)."""
    from videollama2_b200 import ops
    M, N, K = (9232, 1048, 192) if kind == "plain_tail" else (2100, 2080, 328)
    a = rnd((M, K), cuda, seed=70)
    w = rnd((N, K), cuda, 0.06, seed=71)
    kw, ref = {}, a.float() @ w.float().t()
    stats = None
    if kind == "bias_act_res":
        bias = torch.randn(N, device=cuda)
        res = rnd((M, N), cuda, seed=72)
        kw = dict(bias=bias, act=ops.ACT_QUICK_GELU, residual=res)
        ref = ACTS[1](ref + bias) + res.float()
    elif kind == "rms_stats":
        rms_in = (a.float() ** 2).view(M, 8, K // 8).sum(-1).contiguous()
        res = rnd((M, N), cuda, seed=73)
        stats = [(torch.empty((M, N // 32), device=cuda), torch.empty((M, N // 32), device=cuda)) for _ in range(2)]
        kw = dict(rms_in=rms_in, rms_eps=1e-5, residual=res)
        ref = ref * torch.rsqrt((a.float() ** 2).mean(-1, keepdim=True) + 1e-5) + res.float()
    elif kind == "swiglu":
        ref = torch.nn.functional.silu(ref[:, 0::2]) * ref[:, 1::2]
        kw = dict(act=ops.ACT_SWIGLU)
    outs = []
    for i, tile in enumerate((bn, 0)):
        k2 = dict(kw)
        if stats is not None:
            k2.update(sumsq_out=stats[i][0], rowsum_out=stats[i][1])
        if kind == "inplace_strided":
            # out aliases the residual (the residual stream updated in place) and both are column slices of a wider buffer
            buf = rnd((M, N + 64), cuda, seed=74)
            view = buf[:, 32:32 + N]
            if i == 0:
                ref = ref + view.float()
            outs.append(ops.gemm(a, w, residual=view, out=view, bn=tile).clone())
            assert torch.equal(buf[:, :32], rnd((M, N + 64), cuda, seed=74)[:, :32]), "store outside the output slice"
            assert torch.equal(buf[:, 32 + N:], rnd((M, N + 64), cuda, seed=74)[:, 32 + N:]), "store outside the output slice"
        else:
            outs.append(ops.gemm(a, w, bn=tile, **k2))
    assert relerr(outs[0], ref) < 6e-3 and relerr(outs[1], ref) < 6e-3, (kind, bn)
    diff = (outs[0].float() - outs[1].float()).abs()
    assert (diff > 0).float().mean().item() < 1e-3 and relerr(outs[0], outs[1]) < 1e-4, (kind, bn, diff.max().item())
    if stats is not None:
        o = outs[0].float()
        for (sq, sm) in stats:
            assert torch.allclose(sq.sum(1), (o ** 2).sum(1), rtol=2e-3, atol=1e-2)
            assert torch.allclose(sm.sum(1), o.sum(1), rtol=2e-3, atol=0.5)

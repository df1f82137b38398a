"""The tensor-core kernels (wgmma GEMM with its pair tiles, split-K and Conv3d front end; FlashAttention; split-KV decode
attention; fused patch embedding) checked bit for bit where the right answer is known exactly, and element by element
against a bound derived from the kernel's own roundings where it is not.  Every test runs on both builds of the library,
bf16 storage (libvl2.so) and IEEE fp16 storage (libvl2_f16.so, the same sources with other conversion instructions and
wgmma / TMA types): the `dt` parameter; the bf16 cases keep their original ids, the fp16 ones are [fp16-...] (a test
without other parameters has an fp16 sibling named ..._fp16).

A whole-tensor relL2 dilutes a fault confined to one row, one tile or one k-block below the 16-bit noise floor; the
checks here do not: every element is compared on its own (see test_exact_checker.py for the faults each check rejects).

Exact sections
  * GEMM: small-integer operands make every product and partial sum an integer far below 2^24, so the fp32 accumulation
    is exact in any order and the output equals the fp64 product (fp32) or its round-to-nearest-even (bf16 / fp16).  In
    fp16 integers above 2048 round too; that is still one rounding of an fp32-exact value (to_storage_exact).  Nothing
    reaches 65504 by construction in the random tests only because the random sums stay small, which each fp16 test
    that could overflow (|acc| <= 4K, row_scale up to 2) asserts on its data.
  * Attention: queries and keys built from digit codes route every query row to one target key with a logit gap of
    >= 64 in log2 units; the softmax is one-hot far below 16-bit resolution and the output IS the target's value row.
    In bf16 the other keys' P (<= 2^-64) enters the P V MMA as a tiny normal number; in fp16 it underflows to exactly
    0.  Poison keys (a higher logit than the target) sit just past the causal boundary and in the next batch's rows; in
    fp16, whose largest finite value is 65504, the poison logit 2^21 is split as 2^15 * 2^6 over query and key.

Where the exactness premise had to be narrowed, the test says so: the RoPE table is quantised to multiples of 2^-8, the
routing tests use a softmax scale whose product with log2(e) is exactly 2^-3 (decode: scale 1/8).  The production
table and the production scale 1 / sqrt(D) are covered by the bounded sections.

Bounded sections: check_elementwise() against the bound each test derives; the rounding into the storage type is
storage_bound: 2^-8 |x| for bf16, 2^-11 |x| + 2^-25 (half the subnormal spacing) for fp16.  attention_bound has, for
fp16, a subnormal term 2^-25 sum_j |v_j|: the unnormalised P (<= 1) loses up to 2^-25 per key when it is rounded to fp16
for the P V MMA.  Worst measured error / bound on one H100 80GB HBM3 (700 W power limit), bf16 / fp16: activation
epilogues 0.98 / 0.91 (SwiGLU 0.95 / 0.80), production QKV epilogue 0.96 / 0.83, folded LayerNorm with row means of
+-20..40 0.88 / 0.64, attention with logit std 1 / 4 / 16 0.77 / 0.85 / 0.79 and 0.71 / 0.67 / 0.52, patch embedding
(CLIP form) 0.97 / 0.95.  In bf16 the worst elements are those whose final rounding error is close to half an ulp just
above a power of two, where the rounding term of the bound is tight and the fp32 terms add little; at fp16's 2^-11 the
fp32 terms (accumulation, ex2, rsqrt) are a larger share of the bound, which the ratios stay clear of.

fp16 only (section 4): the top of the range - 65504 stays, 65504 < x < 65520 becomes 65504, x >= 65520 becomes inf,
as torch rounds, in the GEMM epilogue on single-CTA and pair tiles, with split-K and with a residual, and sumsq_out of
an overflowed slot is inf; results in the subnormal range are the correctly rounded subnormals; subnormal operands
enter the wgmma GEMM and attention (as V) unflushed."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
F32_U = 2.0 ** -24       # fp32 unit roundoff
FP16_MAX = 65504.0       # largest finite fp16; fp16 rounding sends |x| >= 65520 to inf

# The two storage types the library builds for (libvl2.so, libvl2_f16.so).  Round-to-nearest into the type:
# |rnd(x) - x| <= STORAGE_REL |x| + STORAGE_ABS, the absolute term being half the smallest subnormal spacing (fp16:
# subnormals below 2^-14 are spaced 2^-24 apart; bf16 has the exponent range of fp32, so none arise in these tests).
STORAGE_TYPES = (torch.bfloat16, torch.float16)
STORAGE_BITS = {torch.bfloat16: 8, torch.float16: 11}                    # significant bits
STORAGE_REL = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
STORAGE_ABS = {torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}


def _default_id(v, argname, idx):
    """The id pytest gives parameter value v of argname at index idx when no ids are passed."""
    if v is None or isinstance(v, (bool, int, float, str)):
        return str(v)
    return f"{argname}{idx}"


def storage_params(argnames, values):
    """parametrize over the storage type `dt` (first) and `argnames` / `values`.  The bf16 cases keep the
    ids pytest gives `values` alone - the ids these tests had when they ran on bf16 only - and the fp16 cases are
    'fp16-<that id>'."""
    names = [n.strip() for n in argnames.split(",")]
    cases = []
    for dt in STORAGE_TYPES:
        for i, v in enumerate(values):
            vs = tuple(v) if len(names) > 1 else (v,)
            vid = "-".join(_default_id(x, n, i) for x, n in zip(vs, names))
            cases.append(pytest.param(dt, *vs, id=vid if dt == torch.bfloat16 else f"fp16-{vid}"))
    return pytest.mark.parametrize(",".join(["dt"] + names), cases)


def tag(dt) -> str:
    """Prefix of the printed section names: none for bf16 (the names they always had), 'fp16 ' for fp16."""
    return "" if dt == torch.bfloat16 else "fp16 "


# ---------------------------------------------------------------------------------------------------------------------
# element-wise checker and the bounds it is used with (device-agnostic: the CPU self-tests use them too)
# ---------------------------------------------------------------------------------------------------------------------
def error_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    """|out - ref| / bound per element (fp64); a NaN output counts as an infinite error."""
    o = out.double()
    r = (o - ref.double()).abs() / bound.double()
    return torch.where(torch.isnan(o), torch.full_like(r, math.inf), r)


def check_elementwise(out, ref, bound, what="", tile=(128, 128)) -> float:
    """Every element of `out` within `bound` of the fp64 `ref`.  On failure names the worst element's (row, column) and
    the (row, column) of the output tile of size `tile` it lies in.  Returns the worst error / bound ratio."""
    r = error_ratio(out, ref, bound)
    r2 = r.reshape(r.shape[0], -1) if r.dim() > 1 else r.reshape(1, -1)
    worst = float(r2.max())
    if not worst <= 1.0:
        idx = int(torch.argmax(torch.nan_to_num(r2, nan=math.inf)))
        row, col = divmod(idx, r2.shape[1])
        o = float(out.reshape(r2.shape)[row, col])
        f = float(ref.reshape(r2.shape)[row, col])
        b = float(bound.reshape(r2.shape)[row, col])
        raise AssertionError(f"{what}: worst element (row {row}, col {col}) in tile ({row // tile[0]}, {col // tile[1]}): "
                             f"out {o:.6g}, ref {f:.6g}, |err| {abs(o - f):.3g} > bound {b:.3g} (ratio {worst:.3g})")
    print(f"worst error/bound {what}: {worst:.3f}")
    return worst


def gemm_acc_bound(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Bound on |fp32 tensor-core accumulation - exact| of a[M,K] w[N,K]^T: the MMA adds the exact products of a k16
    step to the fp32 accumulator, aligning and truncating at fp32 precision at most a few times per step.  Allow four
    units of 2^-23 per step, relative to the running sum of |products| <= (|a| |w|^T)."""
    K = a.shape[1]
    return math.ceil(K / 16) * 2.0 ** -21 * (a.double().abs() @ w.double().abs().t())


def storage_bound(ref: torch.Tensor, acc_err: torch.Tensor, dt) -> torch.Tensor:
    """A result of storage type dt: the fp32 errors carried into the final rounding plus that rounding (2^-8 of the
    value for bf16; 2^-11 of the value plus 2^-25, half the fp16 subnormal spacing, for fp16)."""
    u = STORAGE_REL[dt]
    return u * ref.double().abs() + (1 + u) * acc_err + STORAGE_ABS[dt] + 1e-30


def attention_bound(ref, p, v_abs, ds_max, s_abs_max, n_kv_tiles, dt, v_abs_sum=None) -> torch.Tensor:
    """Bound on one attention output element o = sum_j p_j v_j (p the exact softmax) of the wgmma kernel:
      * P enters the P V MMA rounded to the storage type while l sums the fp32 values: <= u sum p|v| (u = 2^-8 / 2^-11);
        in fp16 every unnormalised p_j (<= 1, scaled by factors <= 1 afterwards, divided by l >= 1) may in addition lose
        up to 2^-25 to a subnormal or zero: <= 2^-25 sum_j |v_j| over the visible keys (v_abs_sum);
      * logit errors ds (fp32 Q K^T, scaled) move every p by a relative <= 2 max ds: <= 2 ds_max sum p|v|;
      * ex2.approx and the fp32 rounding of its argument s * scale_log2 - m: relative <= 2^-21 (1 + |s scale_log2|);
      * fp32 accumulation of P V over the key tiles (8 k16 steps each): <= 8 n_kv 2^-21 sum p|v|;
      * the output rounding into the storage type."""
    u = STORAGE_REL[dt]
    pv = p @ v_abs
    rel = u + 2 * ds_max + 2.0 ** -21 * (1 + s_abs_max) + 8 * n_kv_tiles * 2.0 ** -21
    bound = u * ref.abs() + (1 + u) * rel * pv + 1e-30
    if STORAGE_ABS[dt]:
        bound = bound + (1 + u) * STORAGE_ABS[dt] * v_abs_sum + STORAGE_ABS[dt]
    return bound


def attention_reference(q, k, v, causal, scale, dt):
    """fp64 attention of q [H, S, D], k / v [H, S, D] (GQA already expanded) with everything attention_bound needs."""
    q, k, v = q.double(), k.double(), v.double()
    S, D = q.shape[1], q.shape[2]
    s = (q @ k.transpose(1, 2)) * scale
    ds = math.ceil(D / 16) * 2.0 ** -21 * (q.abs() @ k.abs().transpose(1, 2)) * scale
    visible = torch.ones(S, S, dtype=torch.float64, device=q.device)
    if causal:
        mask = torch.ones(S, S, dtype=torch.bool, device=q.device).triu(1)
        s = s.masked_fill(mask, -math.inf)
        ds = ds.masked_fill(mask, 0.0)
        visible = visible.masked_fill(mask, 0.0)
    p = torch.softmax(s, -1)
    ref = p @ v
    s_abs = torch.nan_to_num(s.abs(), posinf=0.0).amax(-1, keepdim=True) * LOG2E
    bound = attention_bound(ref, p, v.abs(), ds.amax(-1, keepdim=True), s_abs, math.ceil(S / 128), dt,
                            v_abs_sum=visible @ v.abs())
    return ref, bound


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def ints(shape, lo, hi, seed, dev, dtype):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device=dev).to(dtype)


def rnd(shape, dev, scale=1.0, seed=0, *, dtype):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).to(dev)


def to_storage_exact(ref64: torch.Tensor, dt) -> torch.Tensor:
    """Round an fp64 result that fp32 holds exactly to the storage type dt (nearest even; fp16: subnormals kept, +-inf
    from 65520 on), as the kernels' pack_bf16 / __float2bfloat16_rn do in the build for dt."""
    r32 = ref64.float()
    assert torch.equal(r32.double(), ref64), "exactness premise: the fp64 result must be fp32-exact"
    return r32.to(dt)


def storage_ulp(v: torch.Tensor, dt) -> torch.Tensor:
    """The spacing of dt's values at |v| (fp16: at least the subnormal spacing 2^-24)."""
    ulp = torch.ldexp(torch.ones_like(v), torch.frexp(v.float())[1].to(torch.int32) - STORAGE_BITS[dt])
    return ulp if dt == torch.bfloat16 else ulp.clamp(min=2.0 ** -24)


def assert_nan(t: torch.Tensor, what: str) -> None:
    assert t.numel() == 0 or bool(torch.isnan(t.float()).all()), f"store outside the output: {what}"


def exact_softmax_scale():
    """(scale, scale * log2 e) with the kernel's fp32 product scale * float(log2 e) exactly a power of two: logits that are
    integers then give exact exp2 arguments, and the target's own probability is exactly 1."""
    l2e = np.float32(LOG2E)
    t = np.float32(0.125)
    s = np.float32(t / l2e)
    for _ in range(64):
        prod = np.float32(s * l2e)
        if prod == t:
            return float(s), float(t)
        s = np.nextafter(s, np.float32(np.inf) if prod < t else np.float32(-np.inf), dtype=np.float32)
    raise AssertionError("no fp32 scale with an exact scale_log2")


# ---------------------------------------------------------------------------------------------------------------------
# 1. GEMM on exact-arithmetic operands
# ---------------------------------------------------------------------------------------------------------------------
TILES = [0, 64, 96, 128, 160, 192, 224, 256, 1128, 1160, 1192, 1224, 1256]   # 0 = the cost model's choice; 1000 + BN = pair


def _edge_cases(bn):
    w = bn % 1000 if bn else 128
    # M: 1, the 128-row boundary, the 256-row (pair) boundary, several persistent rounds (4100 x ~4 tiles > 132 CTAs);
    # N: 8, BN +- 8, multiples of BN +- 8; K: one partial k-block, the 64 boundary, the decoder's down_proj depth
    return [(1, 8, 8), (127, w - 8, 56), (129, w + 8, 64), (255, 2 * w - 8, 72), (257, w, 200), (4100, 4 * w + 8, 136),
            (130, w + 8, 14336)]


def _assert_fp16_range(ref: torch.Tensor, what) -> None:
    """Premise of the fp16 instances of the exact tests: no output reaches fp16's overflow threshold."""
    assert float(ref.abs().max()) < FP16_MAX, f"{what}: the random data reaches the fp16 range"


@storage_params("bn", TILES)
def test_gemm_exact_every_tile_and_edge(cuda, dt, bn):
    """Operands in {-2..2} (|acc| <= 4K <= 57344): exact fp32 accumulation, so the output is the fp64 product rounded once.
    Per tile shape and edge case: (a) 16-bit output written into a column slice of a NaN-filled wider, taller buffer
    from a row-strided A (lda > K), integer bias and power-of-two row_scale; (b) the output aliasing an integer residual
    in such a buffer; (c) fp32 output.  Nothing outside the output slice may change.  In fp16, integers above 2048 round
    (still one rounding of an fp32-exact value), and |acc| row_scale + bias could reach 2 * 57344 + 8 by construction;
    the random sums have a standard deviation of 2 sqrt(K) <= 240 and stay far below 65504, which is asserted."""
    from videollama2_b200 import ops
    for ci, (M, N, K) in enumerate(_edge_cases(bn)):
        seed = 1000 * bn + 10 * ci
        a_full = ints((M, K + 16), -2, 2, seed, cuda, dt)
        a = a_full[:, 8:8 + K]
        w = ints((N, K), -2, 2, seed + 1, cuda, dt)
        bias = ints((N,), -8, 8, seed + 2, cuda, torch.float32)
        rs = (2.0 ** torch.randint(-2, 2, (M,), generator=torch.Generator().manual_seed(seed + 3))).float().to(cuda)
        acc = a.double() @ w.double().t()
        tag_ = (bn, M, N, K)
        # (a)
        buf = torch.full((M + 3, N + 32), float("nan"), device=cuda, dtype=dt)
        out = buf[:M, 16:16 + N]
        ops.gemm(a, w, bias=bias, row_scale=rs, out=out, bn=bn)
        ref = acc * rs.double()[:, None] + bias.double()
        if dt == torch.float16:
            _assert_fp16_range(ref, tag_)
        assert torch.equal(out, to_storage_exact(ref, dt)), ("bias/row_scale", tag_)
        assert_nan(buf[:, :16], f"left guard {tag_}")
        assert_nan(buf[:, 16 + N:], f"right guard {tag_}")
        assert_nan(buf[M:], f"rows past M {tag_}")
        # (b)
        buf = torch.full((M + 3, N + 32), float("nan"), device=cuda, dtype=dt)
        view = buf[:M, 16:16 + N]
        view.copy_(ints((M, N), -8, 8, seed + 4, cuda, dt))
        ref = acc + view.double()
        ops.gemm(a, w, residual=view, out=view, bn=bn)
        assert torch.equal(view, to_storage_exact(ref, dt)), ("aliased residual", tag_)
        assert_nan(buf[:, :16], f"left guard (aliased) {tag_}")
        assert_nan(buf[:, 16 + N:], f"right guard (aliased) {tag_}")
        assert_nan(buf[M:], f"rows past M (aliased) {tag_}")
        # (c)
        o32 = ops.gemm(a.contiguous(), w, out_dtype=torch.float32, bn=bn)
        assert torch.equal(o32.double(), acc), ("fp32 output", tag_)


@storage_params("M,N,K,bn", [
    (1776, 4096, 14336, 0),     # decoder down_proj
    (1776, 6144, 4096, 0),      # decoder QKV
    (1200, 4096, 2048, 256),    # single-CTA tiles: 160 tiles on 132 SMs
    (1154, 1024, 4096, 1128),   # ViT fc2 of a 2-frame shard on pair tiles
    (1776, 4096, 1024, 1256),   # short K: 16 k-blocks
])
def test_gemm_splitk_bit_identical_to_unsplit(cuda, dt, M, N, K, bn):
    """With exact arithmetic the split-K partials add the same products as the unsplit kernel: forced 2, 3 and 4 K-slices
    are bit-identical to it, and to the fp64 product (fp16: the sums stay below 2048 + 8 * 2 sqrt(K) or so, far below
    65504, asserted)."""
    from videollama2_b200 import ops
    a = ints((M, K), -2, 2, 21, cuda, dt)
    w = ints((N, K), -2, 2, 22, cuda, dt)
    res = ints((M, N), -8, 8, 23, cuda, dt)
    ref64 = a.double() @ w.double().t() + res.double()
    if dt == torch.float16:
        _assert_fp16_range(ref64, (M, N, K))
    ref = to_storage_exact(ref64, dt)
    unsplit = ops.gemm(a, w, residual=res, bn=bn, splitk=False)
    assert torch.equal(unsplit, ref)
    for s in (2, 3, 4):
        assert torch.equal(ops.gemm(a, w, residual=res, bn=bn, splitk=s), unsplit), s


@storage_params("bn", [0, 64, 96, 160, 256, 1128, 1192, 1256])
def test_gemm_statistics_exact(cuda, dt, bn):
    """sumsq_out / rowsum_out on operands in {-1, 0, 1}: outputs are integers <= 200 (exact in both storage types) and
    the per-32-column sums of squares stay below 2^24, so both statistics equal the fp64 sums exactly."""
    from videollama2_b200 import ops
    M, N, K = 700, 1056, 192
    a = ints((M, K), -1, 1, 31, cuda, dt)
    w = ints((N, K), -1, 1, 32, cuda, dt)
    res = ints((M, N), -8, 8, 33, cuda, dt)
    sq = torch.full((M, N // 32), float("nan"), device=cuda)
    sm = torch.full((M, N // 32), float("nan"), device=cuda)
    out = ops.gemm(a, w, residual=res, sumsq_out=sq, rowsum_out=sm, bn=bn)
    ref = a.double() @ w.double().t() + res.double()
    assert torch.equal(out, to_storage_exact(ref, dt))
    assert torch.equal(sq.double(), (ref ** 2).view(M, N // 32, 32).sum(-1))
    assert torch.equal(sm.double(), ref.view(M, N // 32, 32).sum(-1))


def rope_table_bits(c: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """ops.rope_table's layout from 16-bit cos / sin tensors: cos in the low half, sin in the high half of an int32."""
    return (c.view(torch.int16).to(torch.int32) & 0xFFFF) | (s.view(torch.int16).to(torch.int32) << 16)


def _rope_table_quantised(n_pos, D, theta, dev, dt):
    """A RoPE table in the layout of ops.rope_table with cos / sin rounded to multiples of 2^-8 (exact in bf16 and
    fp16).  The production table's tiny sines (down to ~2^-20) would make x0 cos - x1 sin span more than fp32's 24
    bits; on this grid the products of integers with the table's 8-bit mantissas AND their sums are fp32-exact,
    whatever the compiler contracts."""
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).double() / D))
    ang = torch.outer(torch.arange(n_pos, dtype=torch.float64), inv)
    c = (torch.round(ang.cos() * 256) / 256).to(dt)
    s = (torch.round(ang.sin() * 256) / 256).to(dt)
    assert torch.equal(c.double(), torch.round(ang.cos() * 256) / 256)
    return rope_table_bits(c, s).contiguous().to(dev), c.double().to(dev), s.double().to(dev)


@storage_params("bn", [0, 64, 128, 1256])
def test_gemm_rope_epilogue_exact(cuda, dt, bn):
    """Integer projection + integer bias, rotated by a 16-bit cos / sin table on adjacent column pairs (2i, 2i+1) of
    every q / k head, v columns untouched: bit-exact against the fp64 rotation (|rotated| <= 2 * 264 on the 2^-8 grid:
    fp32-exact, one rounding into fp16)."""
    from videollama2_b200 import ops
    S, Hq, Hkv, D, pos0, K = 300, 4, 2, 128, 5, 64
    nqk, N = (Hq + Hkv) * D, (Hq + 2 * Hkv) * D
    x = ints((S, K), -2, 2, 41, cuda, dt)
    w = ints((N, K), -2, 2, 42, cuda, dt)
    b = ints((N,), -8, 8, 43, cuda, torch.float32)
    tab, c, s = _rope_table_quantised(pos0 + S + 2, D, 1e6, cuda, dt)
    out = ops.gemm(x, w, bias=b, rope=(tab, pos0, D, nqk), bn=bn)
    y = x.double() @ w.double().t() + b.double()
    qk = y[:, :nqk].view(S, Hq + Hkv, D // 2, 2)
    co, sn = c[pos0:pos0 + S][:, None, :], s[pos0:pos0 + S][:, None, :]
    rot = torch.stack([qk[..., 0] * co - qk[..., 1] * sn, qk[..., 1] * co + qk[..., 0] * sn], -1).reshape(S, nqk)
    assert torch.equal(out, to_storage_exact(torch.cat([rot, y[:, nqk:]], 1), dt))


@pytest.mark.parametrize("pad", [1, 0])
@storage_params("T,H,W,C,N,bn", [(16, 24, 24, 4096, 512, 0), (4, 6, 6, 64, 64, 0), (8, 27, 27, 128, 256, 0),
                                 (3, 5, 7, 64, 96, 0), (16, 24, 24, 256, 512, 1256), (16, 24, 24, 256, 512, 128),
                                 (2, 30, 30, 64, 64, 0)])
def test_conv3d_implicit_gemm_exact(cuda, dt, T, H, W, C, N, bn, pad):
    """The Conv3d(k = s = 2) front end on integer x / weights / bias (|acc| <= 4 * 8C <= 131072 by construction; the
    random sums have a standard deviation of 2 sqrt(8C) <= 362, asserted below 65504 for fp16): bit-exact against fp64
    conv3d, including the zero-padded border taps and the padded output lines."""
    from videollama2_b200 import ops
    if (W % 2 == 1 or H % 2 == 1) and pad == 1:
        pytest.skip("odd H / W with padding is not a configuration of the path")
    x = ints((T, H, W, C), -2, 2, 51, cuda, dt)
    wt = ints((N, C, 2, 2, 2), -2, 2, 52, cuda, dt)
    b = ints((N,), -8, 8, 53, cuda, torch.float32)
    wk = wt.permute(0, 2, 3, 4, 1).reshape(N, 8 * C).contiguous()
    out = ops.conv3d_k2s2(x, wk, bias=b, pad=pad, bn=bn)
    ref = torch.nn.functional.conv3d(x.double().permute(3, 0, 1, 2)[None], wt.double(), b.double(), stride=2, padding=pad)
    ref = ref[0].permute(1, 2, 3, 0).reshape(-1, N)
    if dt == torch.float16:
        _assert_fp16_range(ref, (T, H, W, C, N))
    assert torch.equal(out, to_storage_exact(ref, dt))


# ---------------------------------------------------------------------------------------------------------------------
# 2. attention routing, bit-exact
# ---------------------------------------------------------------------------------------------------------------------
L_CODE = 512.0          # query amplitude on its target's code: the target beats any other key by >= 512 logit units
R_RAMP = 512.0          # logit step per key position of the ramp heads
L_POISON = 2.0 ** 21    # poison logit: beats every legitimate logit (<= 512 * 1776)


def poison_split(dt):
    """(query, key) values of a poison channel with product L_POISON: bf16 holds 2^21 itself; fp16's largest finite value
    is 65504, so there the query carries 2^15 and the key 2^6."""
    return (L_POISON, 1.0) if dt == torch.bfloat16 else (2.0 ** 15, 2.0 ** 6)


def _digits(u: torch.Tensor, nd: int) -> torch.Tensor:
    return torch.stack([(u // 4 ** i) % 4 for i in range(nd)], -1)


def _code_onehot(u: torch.Tensor, nd: int) -> torch.Tensor:
    """Base-4 digit code u as nd concatenated one-hots of width 4: two codes' dot product = their matching digits."""
    return torch.nn.functional.one_hot(_digits(u, nd), 4).flatten(-2).double()


def _routing_problem(B, S, Hq, Hkv, D, causal, dt):
    """q / k / v [B, S, H, D] (fp64, exact in the storage type dt) and the target key of every (batch, row, query head).

    Layout of the D columns: [nd base-4 digit one-hots | ramp (2) | poison channels (B - 1) | zero].
      * Targets: up to 12 key positions spread over the first, middle and last key tiles, each with its own code.  A code
        head of row i carries L_CODE times its target's code and picks among the targets it can see; other targets
        match at most nd - 1 digits, the remaining keys have no code (logit 0).
      * Ramp heads (odd heads, causal only): logit = R_RAMP * key position, so the target is the diagonal key and every
        key past the boundary, i + 1 first, is a poison with a higher logit; the row maximum arrives in the last tile.
      * Batch poison: the first rows of batch b + 1 - those the TMA box of batch b's tail tile would reach in memory -
        carry channel b, which every query of batch b weights so that the logit is L_POISON (poison_split)."""
    nd = (D - 2 - (B - 1)) // 4
    rb, pb = 4 * nd, 4 * nd + 2
    pq, pk = poison_split(dt)
    n_t = min(4 ** nd, S, 12)
    tpos = torch.unique(torch.linspace(0, S - 1, n_t).round().long())
    n_t = tpos.numel()
    q = torch.zeros(B, S, Hq, D, dtype=torch.float64)
    k = torch.zeros(B, S, Hkv, D, dtype=torch.float64)
    i = torch.arange(S)[None, :, None]
    h = torch.arange(Hq)[None, None, :]
    bb = torch.arange(B)[:, None, None]
    n_vis = (tpos[None, :] <= torch.arange(S)[:, None]).sum(1) if causal else torch.full((S,), n_t)
    u = (i * 7 + h * 5 + bb * 3) % n_vis[None, :, None]                       # [B, S, Hq] index into tpos
    ramp = ((h % 2 == 1) & bool(causal)).expand(B, S, Hq)
    q[..., :rb] = L_CODE * _code_onehot(u, nd) * (~ramp)[..., None]
    q[..., rb] = 64 * R_RAMP * ramp
    q[..., rb + 1] = R_RAMP * ramp
    for b in range(B - 1):
        q[b, ..., pb + b] = pq
    target = torch.where(ramp, i.expand(B, S, Hq), tpos[u])
    k[:, tpos, :, :rb] = _code_onehot(torch.arange(n_t), nd)[None, :, None, :]
    j = torch.arange(S, dtype=torch.float64)
    k[..., rb] = (j // 64)[None, :, None]
    k[..., rb + 1] = (j % 64)[None, :, None]
    n_pad = min(S, -S % 128)
    for b in range(1, B):
        k[b, :n_pad, :, pb + b - 1] = pk
    v = torch.randn(B, S, Hkv, D, generator=torch.Generator().manual_seed(B * S + D)).to(dt).double()
    for t in (q, k):
        assert torch.equal(t.to(dt).double(), t)
    return q, k, v, target


def _run_routing(cuda, dt, B, S, Hq, Hkv, D, causal, v=None):
    """Run a routing problem (optionally with other value rows v [B, S, Hkv, D]) and check out == the target's row."""
    from videollama2_b200 import ops
    q, k, v0, target = _routing_problem(B, S, Hq, Hkv, D, causal, dt)
    v = v0 if v is None else v
    scale, _ = exact_softmax_scale()
    qkv = torch.cat([q.reshape(B * S, Hq * D), k.reshape(B * S, Hkv * D), v.reshape(B * S, Hkv * D)], 1)
    qkv = qkv.to(dt).to(cuda)
    buf = torch.full((B * S, Hq * D + 16), float("nan"), device=cuda, dtype=dt)
    out = buf[:, 8:8 + Hq * D]
    ops.attention(qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:], B=B, S=S, Hq=Hq, Hkv=Hkv, D=D,
                  causal=causal, scale=scale, out=out)
    kvh = torch.arange(Hq) // (Hq // Hkv)
    want = v[torch.arange(B)[:, None, None], target, kvh[None, None, :]]            # [B, S, Hq, D]
    got = out.view(B, S, Hq, D).cpu()
    bad = (got.double() != want).any(-1)
    assert not bad.any(), f"{int(bad.sum())} (batch, row, head) outputs differ; first at {bad.nonzero()[0].tolist()}"
    assert_nan(buf[:, :8], "left guard")
    assert_nan(buf[:, 8 + Hq * D:], "right guard")


@storage_params("B,S,Hq,Hkv,D,causal", [
    (1, 1, 2, 2, 64, False), (1, 1, 2, 1, 128, True), (3, 2, 2, 2, 64, True), (3, 2, 4, 2, 8, False),
    (1, 127, 4, 2, 128, True), (3, 127, 2, 2, 72, False), (1, 128, 2, 2, 64, False), (3, 128, 14, 2, 128, True),
    (3, 129, 4, 4, 40, False), (1, 129, 28, 4, 128, True), (1, 255, 2, 1, 96, True), (3, 255, 4, 2, 64, False),
    (3, 256, 7, 1, 64, True), (1, 256, 16, 16, 72, False), (3, 257, 28, 4, 128, True), (1, 257, 2, 2, 8, False),
    (3, 45, 2, 2, 8, True), (3, 300, 6, 3, 40, True), (1, 1776, 28, 4, 128, True), (3, 1776, 8, 8, 64, False),
    (1, 1776, 4, 2, 96, False), (3, 729, 16, 16, 72, False),
])
def test_attention_routing_exact(cuda, dt, B, S, Hq, Hkv, D, causal):
    """out[b, i, h] == v[b, target(b, i, h), h // group] bit for bit, with poison keys past the causal boundary and in
    the next batch's rows, targets in the first / middle / last key tile (the online-softmax rescale runs whenever a
    later tile raises the maximum), and the output written with ldo > Hq * D between NaN guard columns.  In fp16 the
    other keys' P (<= 2^-64) underflows to exactly 0 when it is rounded for the P V MMA, where bf16 keeps it; l sums
    the fp32 values (1 + <= 2^-64 * S == 1), so the output is the target's row in both types."""
    _run_routing(cuda, dt, B, S, Hq, Hkv, D, causal)


@pytest.mark.parametrize("D", [64, 128])
@storage_params("causal", [False, True])
def test_attention_equal_top_logits_exact(cuda, dt, D, causal):
    """Two keys with equal top logits in different key tiles (positions 5 and 260): out = (v_a + v_b) / 2, bit for bit
    (values are integers of equal parity, so the mean is exact); causal rows 5..259 see only v_a (rows before 5 see no
    coded key and are not checked)."""
    from videollama2_b200 import ops
    S, Hq, Hkv = 300, 2, 1
    pa, pb = 5, 260
    scale, _ = exact_softmax_scale()
    q = torch.zeros(S, Hq * D, dtype=torch.float64)
    k = torch.zeros(S, Hkv * D, dtype=torch.float64)
    q[:, :4] = L_CODE
    q[:, D:D + 4] = L_CODE
    k[pa, :4] = 1.0
    k[pb, :4] = 1.0
    v = torch.randint(-100, 101, (S, Hkv * D), generator=torch.Generator().manual_seed(7)).double()
    v[pb] -= (v[pa] + v[pb]) % 2
    qkv = torch.cat([q, k, v], 1).to(dt).to(cuda)
    out = ops.attention(qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:], B=1, S=S, Hq=Hq,
                        Hkv=Hkv, D=D, causal=causal, scale=scale)
    want = ((v[pa] + v[pb]) / 2).repeat(Hq)[None, :].expand(S, Hq * D).clone()
    if causal:
        want[:pb] = v[pa].repeat(Hq)
    assert torch.equal(out.cpu().double()[pa:], want[pa:])


def _decode_nsplit(Hkv):
    return max(1, min(64, (2 * 148) // Hkv))      # decode.cu decode_nsplit: only used to place targets in every split


@storage_params("n_pos,Hq,Hkv,D", [(1, 4, 2, 128), (127, 8, 8, 64), (128, 28, 4, 128), (129, 32, 8, 128),
                                   (5000, 14, 2, 128), (40000, 8, 1, 128), (40000, 16, 4, 64)])
def test_attention_decode_routing_exact(cuda, dt, n_pos, Hq, Hkv, D):
    """Split-KV decode attention routes each query head to its target key bit for bit: targets at position 0, at the last
    position and inside every split, a poison row at n_pos (one past the last visible position) and beyond; the graph
    variant reading the position from device memory is bit-identical.  (fp16: the other keys' weights underflow to 0,
    as in test_attention_routing_exact.)"""
    from videollama2_b200 import ops
    nd = (D - 1) // 4
    pq, pk = poison_split(dt)
    n_tiles = (n_pos + 127) // 128
    tpos = {0, n_pos - 1}
    for s in range(min(_decode_nsplit(Hkv), n_tiles)):
        tpos.add(min(n_pos - 1, s * 128 + (37 * s) % 128))
    tpos = torch.tensor(sorted(tpos))
    n_t = tpos.numel()
    assert n_t <= 4 ** nd
    width = (Hq + 2 * Hkv) * D
    cache = torch.zeros(n_pos + 3, width, dtype=dt, device=cuda)
    kc = cache[:, Hq * D:(Hq + Hkv) * D].view(n_pos + 3, Hkv, D)
    kc[tpos.to(cuda), :, :4 * nd] = _code_onehot(torch.arange(n_t), nd)[:, None, :].to(cuda, dt)
    kc[n_pos:, :, D - 1] = pk                                                   # poison: past the last position
    g = torch.Generator().manual_seed(n_pos + Hq)
    cache[:, (Hq + Hkv) * D:] = torch.randn(n_pos + 3, Hkv * D, generator=g).to(dt).to(cuda)
    k, v = cache[:, Hq * D:(Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:]
    vv = v.view(n_pos + 3, Hkv, D)
    pos_dev = torch.tensor([n_pos - 1], device=cuda, dtype=torch.int32)
    group = Hq // Hkv
    for call in range((n_t + Hq - 1) // Hq):
        u = (call * Hq + torch.arange(Hq)) % n_t
        q = torch.zeros(Hq, D, dtype=torch.float64)
        q[:, :4 * nd] = L_CODE * _code_onehot(u, nd)
        q[:, D - 1] = pq
        qd = q.reshape(-1).to(dt).to(cuda)
        out = ops.attention_decode(qd, k, v, n_pos=n_pos, Hq=Hq, Hkv=Hkv, D=D, scale=0.125)
        want = vv[tpos[u].to(cuda), (torch.arange(Hq) // group).to(cuda)].reshape(1, Hq * D)
        bad = (out != want).view(Hq, D).any(-1).cpu()
        assert not bad.any(), f"heads {bad.nonzero().flatten().tolist()} (targets {tpos[u][bad].tolist()}) differ"
        out2 = torch.empty_like(out)
        ops.attention_decode_dyn(qd, k, v, pos_dev, Hq=Hq, Hkv=Hkv, D=D, scale=0.125, out=out2)
        assert torch.equal(out, out2)


def test_attention_decode_equal_top_logits_exact(cuda):
    """Two keys with equal top logits in different decode splits: the combine step returns (v_a + v_b) / 2 exactly."""
    _decode_equal_top_logits(cuda, torch.bfloat16)


def test_attention_decode_equal_top_logits_exact_fp16(cuda):
    """test_attention_decode_equal_top_logits_exact on the fp16 build."""
    _decode_equal_top_logits(cuda, torch.float16)


def _decode_equal_top_logits(cuda, dt):
    from videollama2_b200 import ops
    n_pos, Hq, Hkv, D = 5000, 8, 2, 128
    pa, pb = 70, 128 * 5 + 3                          # tiles 0 and 5: different splits
    width = (Hq + 2 * Hkv) * D
    cache = torch.zeros(n_pos, width, dtype=torch.float64)
    cache[pa, Hq * D:(Hq + Hkv) * D] = 1.0
    cache[pb, Hq * D:(Hq + Hkv) * D] = 1.0
    vals = torch.randint(-100, 101, (n_pos, Hkv * D), generator=torch.Generator().manual_seed(3)).double()
    vals[pb] -= (vals[pa] + vals[pb]) % 2
    cache[:, (Hq + Hkv) * D:] = vals
    cd = cache.to(dt).to(cuda)
    # logit 64 * 128 * scale = 1024 nats over the zero keys: their exp underflows to exactly 0
    q = torch.full((Hq * D,), 64.0, device=cuda, dtype=dt)
    out = ops.attention_decode(q, cd[:, Hq * D:(Hq + Hkv) * D], cd[:, (Hq + Hkv) * D:], n_pos=n_pos, Hq=Hq, Hkv=Hkv, D=D,
                               scale=0.125)
    want = ((vals[pa] + vals[pb]) / 2).view(Hkv, D).repeat_interleave(Hq // Hkv, 0).reshape(1, -1)
    assert torch.equal(out.cpu().double(), want)


# ---------------------------------------------------------------------------------------------------------------------
# 3. element-wise error bounds
# ---------------------------------------------------------------------------------------------------------------------
ACT64 = {
    1: lambda x: x * torch.sigmoid(1.702 * x),
    2: torch.nn.functional.silu,
    3: lambda x: torch.nn.functional.gelu(x),
    5: lambda x: torch.nn.functional.gelu(x, approximate="tanh"),
}
ACT_SLOPE = 1.2              # max |f'| of quick_gelu / silu / gelu (1.13 for gelu, 1.10 for silu)


def _act_rel(x):
    """Relative error of the epilogue's activation: ex2.approx (2^-22) on an argument rounded to fp32 (|k x| 2^-24),
    1 + e rounded, __fdividef (2 ulp): <= 2^-20 + 2^-22 |x| of the result."""
    return 2.0 ** -20 + 2.0 ** -22 * x.abs()


@pytest.mark.parametrize("bn", [64, 160, 256, 1128, 1224])
@storage_params("act", [1, 2, 3, 5, 4])   # 4 = SwiGLU
def test_gemm_activation_epilogues_bounded(cuda, dt, bn, act):
    """Every activation and SwiGLU on single-CTA and pair tiles, each element within its bound: the accumulation
    (gemm_acc_bound, times the row scale and the activation's slope), the fp32 bias add, the activation's own
    approximation, the output rounding."""
    from videollama2_b200 import ops
    M, N, K = 600, 528, 320
    a = rnd((M, K), cuda, seed=61, dtype=dt)
    w = rnd((N, K), cuda, 0.08, seed=62, dtype=dt)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(63)).to(cuda)
    acc = a.double() @ w.double().t()
    e_acc = gemm_acc_bound(a, w)
    if act == ops.ACT_SWIGLU:
        out = ops.gemm(a, w, bias=bias, act=act, bn=bn)
        x = acc + bias.double()
        ex = e_acc + F32_U * x.abs()
        g, u, eg, eu = x[:, 0::2], x[:, 1::2], ex[:, 0::2], ex[:, 1::2]
        sg = torch.nn.functional.silu(g)
        ref = sg * u
        err = ACT_SLOPE * eg * u.abs() + (sg.abs() + ACT_SLOPE * eg) * eu + (_act_rel(g) + F32_U) * ref.abs()
    else:
        rs = (torch.rand(M, generator=torch.Generator().manual_seed(64)) + 0.5).to(cuda)
        out = ops.gemm(a, w, bias=bias, act=act, row_scale=rs, bn=bn)
        x = acc * rs.double()[:, None] + bias.double()
        ex = e_acc * rs.double()[:, None] + 2 * F32_U * (x.abs() + bias.double().abs())
        ref = ACT64[act](x)
        err = ACT_SLOPE * ex + _act_rel(x) * ref.abs()
    check_elementwise(out, ref, storage_bound(ref, err, dt), f"{tag(dt)}act {act} bn {bn}",
                      tile=(256 if bn > 1000 else 128, bn % 1000))


@storage_params("bn", [0, 64, 1256])
def test_gemm_qkv_production_epilogue_bounded(cuda, dt, bn):
    """The decoder's QKV projection as it runs (decoder._layer): folded RMSNorm (rms_in from row_sumsq) + bias + RoPE with
    the production table of the storage type, in one epilogue; element-wise against fp64."""
    from videollama2_b200 import ops
    S, Hq, Hkv, D, K, pos0 = 300, 4, 2, 128, 512, 17
    nqk, N = (Hq + Hkv) * D, (Hq + 2 * Hkv) * D
    x = rnd((S, K), cuda, 2.0, seed=71, dtype=dt)
    w = rnd((N, K), cuda, K ** -0.5, seed=72, dtype=dt)
    b = rnd((N,), cuda, 0.5, seed=73, dtype=torch.float32)
    tab = ops.rope_table(pos0 + S, D, 1e6, cuda, dt)
    ss = ops.row_sumsq(x)
    out = ops.gemm(x, w, bias=b, rms_in=ss, rms_eps=1e-5, rope=(tab, pos0, D, nqk), bn=bn)
    xd = x.double()
    rs = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-5)
    acc = xd @ w.double().t()
    y = acc * rs + b.double()
    # rs: fp32 sum of squares (<= K 2^-24 relative, any order), rsqrtf (2 ulp): relative <= K 2^-25 + 2^-21
    ey = gemm_acc_bound(x, w) * rs + (K * 2.0 ** -25 + 2.0 ** -21) * (acc * rs).abs() + 2 * F32_U * (y.abs() + b.double().abs())
    tv = tab.cpu()
    c = (tv & 0xFFFF).to(torch.int16).view(dt).double()[pos0:pos0 + S].to(cuda)
    s = (tv >> 16).to(torch.int16).view(dt).double()[pos0:pos0 + S].to(cuda)
    yq, eq = y[:, :nqk].view(S, Hq + Hkv, D // 2, 2), ey[:, :nqk].view(S, Hq + Hkv, D // 2, 2)
    co, sn = c[:, None, :], s[:, None, :]
    r0 = yq[..., 0] * co - yq[..., 1] * sn
    r1 = yq[..., 1] * co + yq[..., 0] * sn
    e_rot = co.abs() * (eq[..., 0] + eq[..., 1]) + sn.abs() * (eq[..., 0] + eq[..., 1]) \
        + 2 * F32_U * (yq[..., 0].abs() + yq[..., 1].abs())
    ref = torch.cat([torch.stack([r0, r1], -1).reshape(S, nqk), y[:, nqk:]], 1)
    err = torch.cat([torch.stack([e_rot, e_rot], -1).reshape(S, nqk), ey[:, nqk:]], 1)
    check_elementwise(out, ref, storage_bound(ref, err, dt), f"{tag(dt)}qkv bn {bn}")


@storage_params("bn", [0, 64, 1128])
def test_gemm_folded_layernorm_large_mean_bounded(cuda, dt, bn):
    """Folded LayerNorm rstd * (x W'^T - mu * colsum) + b' on rows with mean and std ~ 30 (the outlier channels of CLIP
    residual streams): the cancellation in acc - mu * colsum and in E[x^2] - mu^2 must stay within the bound built from
    the accumulation (which scales with |x|, i.e. with the mean), the fp32 row statistics and the fp32 column sums."""
    from videollama2_b200 import ops
    M, K, N = 577, 1024, 1024
    g = torch.Generator().manual_seed(81)
    mu_row = (torch.rand(M, 1, generator=g) * 20 + 20) * torch.where(torch.rand(M, 1, generator=g) < 0.5, -1.0, 1.0)
    x = (mu_row + 30 * torch.randn(M, K, generator=g)).to(dt).to(cuda)
    wf = rnd((N, K), cuda, K ** -0.5, seed=82, dtype=dt)
    colsum = wf.double().sum(1)
    bias = rnd((N,), cuda, 0.2, seed=83, dtype=torch.float32)
    stats = ops.row_stats(x)
    out = ops.gemm(x, wf, bias=bias, ln_in=stats, ln_colsum=colsum.float().contiguous(), rms_eps=1e-5, bn=bn)
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = xd.var(-1, unbiased=False, keepdim=True)
    rstd = torch.rsqrt(var + 1e-5)
    acc = xd @ wf.double().t()
    cen = acc - mu * colsum[None, :]
    ref = rstd * cen + bias.double()
    # row statistics: fp32 sums of K terms in any order (<= K 2^-24 of the sums of |terms|)
    d_mu = K * F32_U * xd.abs().mean(-1, keepdim=True)
    d_var = K * F32_U * xd.pow(2).mean(-1, keepdim=True) + 2 * mu.abs() * d_mu + 2 * F32_U * (2 * mu * mu + var)
    d_rstd = d_var / (2 * (var + 1e-5)) + 2.0 ** -21                                  # relative, rsqrtf 2 ulp
    e_cen = gemm_acc_bound(x, wf) + (mu.abs() * F32_U + d_mu) * colsum.abs()[None, :] + F32_U * (acc.abs() + (mu * colsum).abs())
    err = rstd * e_cen + d_rstd * (rstd * cen).abs() + 2 * F32_U * (ref.abs() + bias.double().abs())
    check_elementwise(out, ref, storage_bound(ref, err, dt), f"{tag(dt)}folded LN bn {bn}")


@pytest.mark.parametrize("sigma", [1.0, 4.0, 16.0])
@storage_params("B,S,Hq,Hkv,D,causal", [(2, 577, 4, 4, 64, False), (1, 1776, 8, 2, 128, True), (3, 300, 6, 2, 72, True)])
def test_attention_peaky_logits_bounded(cuda, dt, sigma, B, S, Hq, Hkv, D, causal):
    """Logit standard deviation sigma (q, k ~ N(0, sqrt(sigma)), production scale 1 / sqrt(D)); causal rows get a ramp
    of 3 sigma over the key positions, so the row maximum tends to arrive in a late key tile and the running maximum is
    raised tile after tile.  Every output element within attention_bound.  sigma = 16 puts most of P below 2^-14, i.e.
    into fp16's subnormal range, where the subnormal term of attention_bound is the one that counts."""
    from videollama2_b200 import ops
    amp = math.sqrt(sigma)
    qkv = rnd((B * S, (Hq + 2 * Hkv) * D), cuda, amp, seed=int(sigma) * 7 + D, dtype=dt)
    if causal:
        qkv[:, :Hq * D].view(B * S, Hq, D)[:, :, 0] = math.sqrt(D)
        ramp = (3 * sigma * torch.arange(S, device=cuda) / S).repeat(B)
        qkv[:, Hq * D:(Hq + Hkv) * D].view(B * S, Hkv, D)[:, :, 0] = ramp[:, None].to(dt)
    scale = D ** -0.5
    q, k, v = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    out = ops.attention(q, k, v, B=B, S=S, Hq=Hq, Hkv=Hkv, D=D, causal=causal, scale=scale)
    G = Hq // Hkv
    worst = 0.0
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        qf = q[rows].view(S, Hq, D).transpose(0, 1)
        kf = k[rows].view(S, Hkv, D).transpose(0, 1).repeat_interleave(G, 0)
        vf = v[rows].view(S, Hkv, D).transpose(0, 1).repeat_interleave(G, 0)
        ref, bound = attention_reference(qf, kf, vf, causal, scale, dt)
        got = out[rows].view(S, Hq, D).transpose(0, 1)
        for h in range(Hq):
            worst = max(worst, check_elementwise(got[h], ref[h], bound[h], f"{tag(dt)}sigma {sigma} batch {b} head {h}",
                                                 tile=(128, D)))
    print(f"worst error/bound {tag(dt)}attention sigma {sigma} {(B, S, Hq, Hkv, D, causal)}: {worst:.3f}")


def _ln_rows_bound(x, d_x, gamma, beta):
    """fp64 LayerNorm of rows x [R, C] (gamma, beta [C]) and a bound on the kernel's fp32 result given per-element input
    errors d_x: fp32 row sums (<= C 2^-24 of the sums of |terms|), E[x^2] - mu^2, rsqrtf, the normalise-scale-shift.
    The rounding into the storage type is storage_bound's."""
    C = x.shape[1]
    mu = x.mean(-1, keepdim=True)
    var = x.var(-1, unbiased=False, keepdim=True)
    rstd = torch.rsqrt(var + 1e-5)
    y = (x - mu) * rstd * gamma + beta
    d_mu = d_x.mean(-1, keepdim=True) + C * F32_U * x.abs().mean(-1, keepdim=True)
    d_var = 2 * (x.abs() * d_x).mean(-1, keepdim=True) + C * F32_U * x.pow(2).mean(-1, keepdim=True) \
        + 2 * mu.abs() * d_mu + 2 * F32_U * (2 * mu * mu + var)
    d_rstd = d_var / (2 * (var + 1e-5)) + 2.0 ** -21
    err = gamma.abs() * rstd * (d_x + d_mu) + gamma.abs() * (x - mu).abs() * rstd * (d_rstd + 4 * F32_U) + F32_U * y.abs()
    return y, err


@storage_params("F,H,P,C", [(2, 56, 14, 128), (3, 112, 14, 256), (16, 336, 14, 1024), (2, 336, 14, 1024)])
def test_patch_embed_clip_rowwise_bounded(cuda, dt, F, H, P, C):
    """CLIP form (conv rounded to the storage type -> + position -> pre-LayerNorm, as in HF; class row LN(cls + pos[0])
    in every frame) checked row by row at C = 128 / 256 / 1024, i.e. clusters of 1, 2, 4 and 8 CTAs sharing a row's
    LayerNorm statistics over distributed shared memory.  Where the fp32 conv sum may round to the other side of a
    rounding midpoint of the storage type than the exact sum, one ulp of input error is allowed for that element."""
    from videollama2_b200 import ops
    px = rnd((F, 3, H, H), cuda, seed=91, dtype=dt)
    wconv = rnd((C, 3, P, P), cuda, 0.05, seed=92, dtype=dt)
    K = 3 * P * P
    Kpad = (K + 63) // 64 * 64
    wpad = torch.zeros((C, Kpad), device=cuda, dtype=dt)
    wpad[:, :K] = wconv.reshape(C, K)
    npch = (H // P) ** 2
    cls = rnd((C,), cuda, seed=93, dtype=dt)
    pos = rnd((npch + 1, C), cuda, seed=94, dtype=dt)
    g = rnd((C,), cuda, 0.1, seed=95, dtype=dt) + 1
    b = rnd((C,), cuda, 0.1, seed=96, dtype=dt)
    tok = ops.patch_embed(px, wpad, pos, P, cls=cls, gamma=g, beta=b, eps=1e-5)
    A = torch.nn.functional.unfold(px.double(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, K)
    conv = A @ wconv.reshape(C, K).double().t()
    e_conv = math.ceil(Kpad / 16) * 2.0 ** -21 * (A.abs() @ wconv.reshape(C, K).double().abs().t())
    conv_b = conv.float().to(dt).double()
    ulp = storage_ulp(conv, dt)
    mid_dist = ((conv - conv_b).abs() - ulp / 2).abs()                           # distance to the nearest rounding midpoint
    d_conv = torch.where(mid_dist <= e_conv, ulp, torch.zeros_like(ulp))
    x = torch.cat([(cls.double() + pos[0].double()).expand(F, 1, C),
                   conv_b.view(F, npch, C) + pos[1:].double()], 1).reshape(-1, C)
    d_x = torch.cat([torch.zeros(F, 1, C, device=cuda, dtype=torch.float64), d_conv.view(F, npch, C)], 1).reshape(-1, C) \
        + F32_U * x.abs()
    ref, err = _ln_rows_bound(x, d_x, g.double(), b.double())
    check_elementwise(tok, ref, storage_bound(ref, err, dt), f"{tag(dt)}patch embed C {C} F {F}", tile=(npch + 1, C))


@storage_params("F,H,P,C", [(2, 384, 14, 1152), (3, 70, 14, 288)])
def test_patch_embed_siglip_exact(cuda, dt, F, H, P, C):
    """SigLIP form on integer pixels, weights, bias and positions (|acc| <= 4 * 588): conv + bias + position is exact in
    fp32, so the output is the fp64 result rounded once, bit for bit."""
    from videollama2_b200 import ops
    px = ints((F, 3, H, H), -2, 2, 101, cuda, dt)
    wconv = ints((C, 3, P, P), -2, 2, 102, cuda, dt)
    K = 3 * P * P
    Kpad = (K + 63) // 64 * 64
    wpad = torch.zeros((C, Kpad), device=cuda, dtype=dt)
    wpad[:, :K] = wconv.reshape(C, K)
    npch = (H // P) ** 2
    pos = ints((npch, C), -8, 8, 103, cuda, dt)
    bias = ints((C,), -8, 8, 104, cuda, torch.float32)
    tok = ops.patch_embed(px, wpad, pos, P, bias=bias)
    patch = torch.nn.functional.conv2d(px.double(), wconv.double(), bias.double(), stride=P).flatten(2).transpose(1, 2)
    assert torch.equal(tok, to_storage_exact((patch + pos.double()).reshape(-1, C), dt))


# ---------------------------------------------------------------------------------------------------------------------
# 4. fp16 only: the top of the range and the subnormals
# ---------------------------------------------------------------------------------------------------------------------
H16 = torch.float16
# fp32 biases at the top of fp16's range: bias + (an integer accumulator of a few tens) crosses 65504 (kept), 65504..65520
# (rounds down to 65504, e.g. 65519.75), 65520 (the midpoint to the next binade: +inf) and beyond, at both signs
OVERFLOW_BIAS = [65504.0, 65504.75, 65496.25, 65520.0, 65536.0, 1.0e5, 65472.0, 0.0]


def assert_overflow_classes(ref64: torch.Tensor) -> None:
    """The fp64 results of an overflow test contain every case at both signs: exactly 65504, strictly between 65504 and
    65520 (rounds to 65504), and >= 65520 (rounds to inf)."""
    for sgn in (1.0, -1.0):
        r = ref64 * sgn
        assert bool((r == FP16_MAX).any()), "no result of exactly 65504"
        assert bool(((r > FP16_MAX) & (r < 65520.0)).any()), "no result in (65504, 65520)"
        assert bool((r >= 65520.0).any()), "no result >= 65520"


@pytest.mark.parametrize("bn,splitk,residual", [(128, False, False), (1256, False, False), (128, 2, False),
                                                (128, False, True), (1256, False, True), (0, 4, True)])
def test_fp16_gemm_overflow_rounds_like_torch(cuda, bn, splitk, residual):
    """Results at the top of fp16's range leave the epilogue (pack_bf16 = __floats2half2_rn in the fp16 build) as torch
    rounds the fp64 result: 65504 stays, 65519.75 becomes 65504, 65520 and more become +-inf; no saturation, no NaN.
    Integer accumulators in [-48, 48] plus fp32 biases of OVERFLOW_BIAS (or, with a residual, bias 0.75 and residuals
    of +-65504 / +-65472) make every fp64 result fp32-exact.  Single-CTA and pair tiles, forced split-K, residual.  The
    per-32-column sumsq_out of a slot holding an infinity is +inf, because the statistics are taken from the rounded
    value the consumer reads, and finite otherwise."""
    from videollama2_b200 import ops
    M, N, K = 300, 256, 256
    a = ints((M, K), -1, 1, 201, cuda, H16)
    w = ints((N, K), -1, 1, 202, cuda, H16)
    acc = a.double() @ w.double().t()
    col = torch.arange(N)
    big = (col // 32) % 2 == 0              # even 32-column slots reach the top of the range, odd ones stay moderate
    sgn = torch.where(col % 2 == 0, 1.0, -1.0).double()
    if residual:
        bias = torch.where((col // 4) % 2 == 0, 0.0, 0.75).double()
        res = sgn * torch.where(big, torch.tensor([FP16_MAX, 65472.0]).double()[(col // 2) % 2], 1000.0)
        res = res[None, :].expand(M, N).to(H16).to(cuda).contiguous()
        ref = acc + bias.to(cuda) + res.double()
    else:
        bias = sgn * torch.where(big, torch.tensor(OVERFLOW_BIAS).double()[(col // 2) % len(OVERFLOW_BIAS)], 1000.25)
        res = None
        ref = acc + bias.to(cuda)
    assert_overflow_classes(ref)
    sq = torch.full((M, N // 32), float("nan"), device=cuda)
    out = ops.gemm(a, w, bias=bias.float().to(cuda), residual=res, sumsq_out=sq, bn=bn, splitk=splitk or False)
    want = to_storage_exact(ref, H16)
    assert not bool(torch.isnan(out).any()) and not bool(torch.isnan(sq).any())
    assert torch.equal(out, want)
    slot_inf = torch.isinf(want).view(M, N // 32, 32).any(-1)
    assert torch.equal(torch.isinf(sq), slot_inf) and bool(slot_inf.any()) and bool((~slot_inf).any())
    assert bool((sq[slot_inf] > 0).all())


@pytest.mark.parametrize("bn", [128, 1256])
def test_fp16_gemm_subnormal_results_rounded(cuda, bn):
    """row_scale 2^-20 .. 2^-28 on integer accumulators: acc * row_scale (fp32-exact) lands in fp16's subnormal range
    [2^-24, 2^-14) and below; the output must be torch's correctly rounded fp16 subnormal (round to nearest even on the
    2^-24 grid), not zero and not a truncation."""
    from videollama2_b200 import ops
    M, N, K = 300, 256, 128
    a = ints((M, K), -2, 2, 211, cuda, H16)
    w = ints((N, K), -2, 2, 212, cuda, H16)
    rs = (2.0 ** -torch.arange(20, 29)[torch.arange(M) % 9]).float().to(cuda)
    acc = a.double() @ w.double().t()
    ref = acc * rs.double()[:, None]
    out = ops.gemm(a, w, row_scale=rs, bn=bn)
    want = to_storage_exact(ref, H16)
    sub = (want != 0) & (want.abs() < 2.0 ** -14)
    assert int(sub.sum()) > 1000 and bool((want.double() != ref).any())      # subnormal results, many of them rounded
    assert torch.equal(out, want)


def subnormals(shape, kmax, seed, dev):
    """fp16 subnormals k 2^-24, k in [-kmax, kmax] (zero included; kmax < 1024), as an fp16 tensor."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-kmax, kmax + 1, shape, generator=g).double() * 2.0 ** -24).to(H16).to(dev)


@pytest.mark.parametrize("bn", [128, 1256])
def test_fp16_gemm_subnormal_operands_exact(cuda, bn):
    """Both wgmma operands fp16 subnormals (k 2^-24, |k| <= 63): their products k k' 2^-48 and sums (|sum k k'| <
    192 * 2^12 < 2^24) are fp32-exact normals; row_scale 2^40 scales them to multiples of 2^-8 (fp32 output: exact),
    2^24 to multiples of 2^-24 (fp16 output: one rounding, the smallest ones subnormal).  A flushed operand would give
    zeros."""
    from videollama2_b200 import ops
    M, N, K = 300, 256, 192
    a = subnormals((M, K), 63, 221, cuda)
    w = subnormals((N, K), 63, 222, cuda)
    assert bool((a != 0).any()) and float(a.abs().max()) < 2.0 ** -14
    acc = a.double() @ w.double().t()
    rs = torch.full((M,), 2.0 ** 40, device=cuda)
    o32 = ops.gemm(a, w, row_scale=rs, out_dtype=torch.float32, bn=bn)
    assert torch.equal(o32.double(), acc * 2.0 ** 40)
    o16 = ops.gemm(a, w, row_scale=torch.full((M,), 2.0 ** 24, device=cuda), bn=bn)
    assert torch.equal(o16, to_storage_exact(acc * 2.0 ** 24, H16))


def test_fp16_attention_subnormal_values_exact(cuda):
    """Value rows of fp16 subnormals through the routing problem: P is one-hot (1 on the target, 0 after the fp16
    rounding elsewhere), so the output is the target's subnormal value row bit for bit; a flushed V operand or a flushed
    output would give zeros."""
    B, S, Hq, Hkv, D = 3, 300, 6, 3, 40
    g = torch.Generator().manual_seed(231)
    v = torch.randint(-1023, 1024, (B, S, Hkv, D), generator=g).double() * 2.0 ** -24
    _run_routing(cuda, H16, B, S, Hq, Hkv, D, True, v=v)

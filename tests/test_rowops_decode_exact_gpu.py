"""The row, decode and glue kernels (rowops.cu, decode.cu) checked element by element: bit for bit where small-integer
operands keep fp32 exact, and against a bound derived from the kernel's own roundings where they do not.  Every test
runs on the bf16 and the fp16 build of the library (the `dt` parameter, as in test_kernels_exact_gpu.py).

Covered: the decode GEMV (both row-per-warp variants, RMS scale, every activation, bias / residual, both output types, K
across the bulk-copy ring), the mma.sync skinny GEMM (both A types, every activation, M on both sides of the second
16-row pass, ragged N and K), the RoPE cos / sin of the decode kernels against the host table of the prefill GEMM out to
position 32768, the decode RoPE-append, LayerNorm / RMSNorm on every dispatch branch, row statistics, the STC
connector's depthwise conv + LN + SiLU with its SE pooling and scaling, the CLIP embedding finish and the im2col gathers
and embedding splice.  Outputs go into NaN-filled buffers wherever the API lets the caller place them, and the NaN
guards around them must survive.

Exactness premises
  * GEMV / skinny GEMM: operands in {-2..2}, integer bias and residual; the fp32 A of the skinny GEMM holds rounding
    ties of the storage type (bf16: (2k+1) 2^-8 in [1, 2) and (2k+1) 2^-9 in [0.5, 1); fp16: (2k+1) 2^-11 in [1, 2)
    and (2k+1) 2^-12 in [0.5, 1)).  Staged, those are multiples of 2^-8 (bf16) or 2^-11 (fp16), so every partial sum is
    a multiple of that, bounded by sum_k |a_k| |w_k|; it is fp32-exact below 2^16 (bf16) or 2^13 (fp16).  For fp16 the
    skinny weights are in {-1..1} to keep sum |a| |w| (about 0.76 K) below 2^13 up to the SE MLP's K = 8192; each run
    asserts the premise on its data.  The GEMV's |result| stays below 4K + 16 < 65504 (SwiGLU excepted, see
    _past_fp16_range).
  * RoPE: a (1, 0) pair makes the kernel write its 16-bit (cos, sin); bf16 x bf16 and fp16 x fp16 products are
    fp32-exact, so a rotated row is x0 c - x1 s rounded to fp32 once and then to the storage type.
  * Constant LayerNorm rows have an exact mean: the output is the storage type's rounding of beta + residual.

Bounded sections use check_elementwise() from test_kernels_exact_gpu.py and print their worst error / bound ratio.
Worst measured on one H100 80GB HBM3 (700 W power limit), bf16 / fp16: GEMV 0.995 / 0.998, skinny GEMM 0.996 / 0.999,
LayerNorm 0.994 / 0.994, RMSNorm 0.988 / 0.999, depthwise conv + LN + SiLU 0.983 / 0.958, SE pooling 0.164 / 0.171,
CLIP embedding finish 0.974 / 0.934; the final rounding dominates.  The device RoPE cos / sin differ from
ops.rope_table in bf16 in 16 of 4194304 values (D = 128) and 9 of 2097152 (D = 64), in fp16 in 99 of 4194304 and 48 of
2097152, all one ulp next to a rounding midpoint; the bf16 host table differs from the correctly rounded one in 3 of
4194304.

fp16 only (section h): the GEMV, skinny GEMM (both A types, including fp32 A values of 65504, 65519, 65519.99, 65520
and beyond being staged), LayerNorm (large beta, large gamma) and RMSNorm (large gamma) stores round like torch at the
top of the range: 65504 stays, (65504, 65520) becomes 65504, >= 65520 becomes inf, no NaN; subnormal GEMV results are
correctly rounded, and subnormal operands enter the GEMV, the skinny GEMM and LayerNorm unflushed."""
import itertools
import math

import pytest
import torch

from test_kernels_exact_gpu import (ACT_SLOPE, F32_U, FP16_MAX, STORAGE_BITS, STORAGE_TYPES, _act_rel, _ln_rows_bound,
                                    assert_nan, check_elementwise, ints, rnd, storage_bound, storage_params, storage_ulp,
                                    subnormals, tag, to_storage_exact)

pytestmark = pytest.mark.gpu

NAN = float("nan")
ACT_NONE, ACT_SILU, ACT_SWIGLU, ACT_SIGMOID = 0, 2, 4, 100      # videollama2_b200._lib
RMS_REL = 2.0 ** -22 + 2.0 ** -23     # rsqrtf (2 ulp) of an argument rounded twice (the division by K, + eps)


def _report(section: str, worst: float) -> None:
    print(f"worst error/bound {section}: {worst:.3f}")


def _abi(dt, name: str, *args) -> None:
    """Call a C-ABI entry point of the build for storage type dt directly (for outputs the torch front end allocates
    itself) on the current stream."""
    from videollama2_b200 import _lib
    _lib.check(getattr(_lib.load(dt), name)(*args, torch.cuda.current_stream().cuda_stream), name)


# ---------------------------------------------------------------------------------------------------------------------
# epilogue of the GEMV and the skinny GEMM: act(acc * s + bias) (+ residual)
# ---------------------------------------------------------------------------------------------------------------------
def _epilogue(acc, s, rel_s, bias, act, res):
    """fp64 result and fp32 error bound of act(acc * s + bias) (+ residual) for an exact accumulator `acc` and a row
    scale s with relative error rel_s: the fp32 multiply and bias add, the activation (slope and its own
    approximation, _act_rel), the residual add.  SwiGLU pairs interleaved (gate, up) columns."""
    x = acc * s
    ex = acc.abs() * s * rel_s + F32_U * x.abs()
    if bias is not None:
        x = x + bias
        ex = ex + F32_U * x.abs()
    if act == ACT_SWIGLU:
        g, u, eg, eu = x[..., 0::2], x[..., 1::2], ex[..., 0::2], ex[..., 1::2]
        sg = torch.nn.functional.silu(g)
        ref = sg * u
        return ref, ACT_SLOPE * eg * u.abs() + (sg.abs() + ACT_SLOPE * eg) * eu + (_act_rel(g) + F32_U) * ref.abs()
    if act == ACT_SILU:
        ref = torch.nn.functional.silu(x)
        err = ACT_SLOPE * ex + _act_rel(x) * ref.abs()
    elif act == ACT_SIGMOID:
        ref = torch.sigmoid(x)
        err = ACT_SLOPE * ex + _act_rel(x) * ref.abs()
    else:
        ref, err = x, ex
    if res is not None:
        ref = ref + res
        err = err + F32_U * ref.abs()
    return ref, err


def _check_epilogue(out, ref, err, exact, what):
    """Exact: torch.equal with the fp64 result rounded once.  Otherwise element-wise; returns the worst ratio."""
    if exact:
        want = to_storage_exact(ref, out.dtype) if out.dtype in STORAGE_TYPES else ref.float()
        assert torch.equal(out.reshape(want.shape), want), what
        return 0.0
    out = out.reshape(ref.shape)
    if out.dtype == torch.float16:
        out, ref = _past_fp16_range(out, ref, err, what)
    bound = storage_bound(ref, err, out.dtype) if out.dtype in STORAGE_TYPES else err + F32_U * ref.abs() + 1e-30
    return check_elementwise(out, ref, bound, what)


def _past_fp16_range(out, ref, err, what):
    """fp16 results beyond the range (SwiGLU multiplies two accumulators: up to ~1e5 on the integer operands): where the
    fp32 value, ref +- err, is >= 65520 for sure, the output must be inf of ref's sign; where it may lie on either side
    of 65520, +-65504 or +-inf.  Returns (out, ref) with those elements set to 0 for the element-wise check."""
    o = out.double()
    sure = ref.abs() - err >= 65520.0
    maybe = (ref.abs() + err >= 65520.0) & ~sure
    assert torch.equal(o[sure], torch.copysign(torch.full_like(ref[sure], math.inf), ref[sure])), f"{what}: overflow"
    m = o[maybe]
    assert bool((((m.abs() == FP16_MAX) | m.isinf()) & (torch.sign(m) == torch.sign(ref[maybe]))).all()), what
    past = sure | maybe
    return out.masked_fill(past, 0.0), ref.masked_fill(past, 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# a. GEMV (M = 1)
# ---------------------------------------------------------------------------------------------------------------------
# N: warps past N leave early (1, 3, 5); one row per warp below 8192 (4095, 8191); two rows per warp from 8192, the last
# one clamped for odd N (8193).  K: one partial chunk (8), a partial last 2 KB chunk (1016, 1032), fewer chunks than and
# exactly the 3-stage ring (2048, 3072), 4096, and 14 chunks (14336): the ring wraps four times (three with the 4-stage
# ring of R = 2) and the mbarrier parity flips each time.
GEMV_SHAPES = [(N, K) for N in (1, 3, 5) for K in (8, 1032, 14336)] + \
              [(N, K) for N in (4095, 8191, 8192, 8193) for K in (8, 1016, 1024, 1032, 2048, 3072, 4096, 14336)]


def _run_gemv_variants(cuda, dt, N, K, seed, acts, dtypes, eps=1e-5):
    from videollama2_b200 import ops
    w = ints((N, K), -2, 2, seed, cuda, dt)
    x = ints((K,), -2, 2, seed + 1, cuda, dt)
    bias = ints((N,), -8, 8, seed + 2, cuda, torch.float32)
    acc = w.double() @ x.double()
    s_rms = 1.0 / math.sqrt(float(x.double().pow(2).sum()) / K + eps)
    worst = 0.0
    for rms, act, use_bias, use_res, odt in itertools.product((False, True), acts, (False, True), (False, True), dtypes):
        if act == ACT_SWIGLU and (N % 2 or use_res):
            continue
        n_out = N // 2 if act == ACT_SWIGLU else N
        res = ints((n_out,), -8, 8, seed + 3, cuda, dt) if use_res else None
        cache = torch.full((4, n_out), NAN, device=cuda, dtype=odt)       # the decode step writes one row of the cache
        row = cache[2:3]
        ops.gemv(x, w, bias=bias if use_bias else None, act=act, residual=res, out=row, rms_eps=eps if rms else 0.0)
        what = f"{tag(dt)}gemv N {N} K {K} rms {rms} act {act} bias {use_bias} res {use_res} {odt}"
        assert_nan(cache[:2], what)
        assert_nan(cache[3:], what)
        ref, err = _epilogue(acc, s_rms if rms else 1.0, RMS_REL if rms else 0.0, bias.double() if use_bias else None,
                             act, res.double() if use_res else None)
        worst = max(worst, _check_epilogue(row[0], ref, err, not rms and act == ACT_NONE, what))
    return worst


@storage_params("N,K", GEMV_SHAPES)
def test_gemv_exact_and_bounded(cuda, dt, N, K):
    """Every variant (RMS scale or not, act none / SiLU / sigmoid / SwiGLU, with and without bias and residual, 16-bit
    and fp32 output) written into one row of a NaN cache: bit-exact without RMS scale and activation, else element-wise.
    fp16 range: |w x| <= 4K by construction, and with the RMS scale too (sum |w_k x_k| s <= 2 sum |x_k| sqrt(K / sum
    x_k^2) <= 2K), so |result| <= 4 * 14336 + 16 < 65504 - except SwiGLU, silu(g) u, which reaches ~1e5 at K >= 3072
    and must then be +-inf, as torch's fp16 rounding gives (_past_fp16_range)."""
    worst = _run_gemv_variants(cuda, dt, N, K, 7 * N + K, (ACT_NONE, ACT_SILU, ACT_SIGMOID, ACT_SWIGLU),
                               (dt, torch.float32))
    _report(f"{tag(dt)}gemv N {N} K {K}", worst)


@storage_params("N,K,act,dtype", [(28672, 4096, ACT_SWIGLU, torch.bfloat16),     # Mistral gate/up
                                  (37888, 3584, ACT_SWIGLU, torch.bfloat16),     # Qwen2 gate/up
                                  (152064, 3584, ACT_NONE, torch.float32),      # Qwen2 lm_head
                                  (32000, 4096, ACT_NONE, torch.float32)])      # Mistral lm_head
def test_gemv_decoder_shapes(cuda, dt, N, K, act, dtype):
    """The decode step's widest GEMVs at their real shapes (K = 3584 ends in half a chunk); `dtype` is the output type
    of the bf16 build, 16-bit (the storage type dt) for the MLP and fp32 for the lm_head."""
    odt = dt if dtype == torch.bfloat16 else dtype
    _report(f"{tag(dt)}gemv decoder N {N} K {K}", _run_gemv_variants(cuda, dt, N, K, N + K, (act,), (odt,)))


# ---------------------------------------------------------------------------------------------------------------------
# b. skinny GEMM (mma.sync m16n8k16), M <= 32
# ---------------------------------------------------------------------------------------------------------------------
def _storage_ties(shape, seed, dev, dt):
    """fp32 values exactly halfway between two neighbours of the storage type, either sign, mixed with small integers:
    bf16 (2k+1) 2^-8 in [1, 2) and (2k+1) 2^-9 in [0.5, 1); fp16 (2k+1) 2^-11 in [1, 2) and (2k+1) 2^-12 in [0.5, 1).
    Staging them to the storage type must round to nearest even, as torch's .to() does; truncation or round-half-up
    would move half of them."""
    bits = STORAGE_BITS[dt]
    g = torch.Generator().manual_seed(seed)
    odd = 2 * torch.randint(0, 2 ** bits // 2, shape, generator=g) + 1
    tie = (2 ** bits + odd).double() * 2.0 ** -bits * 2.0 ** -torch.randint(0, 2, shape, generator=g).double()
    tie = tie * (1 - 2 * torch.randint(0, 2, shape, generator=g)).double()
    small = torch.randint(-2, 3, shape, generator=g).double()
    a = torch.where(torch.rand(shape, generator=g) < 0.75, tie, small).float()
    assert not torch.equal(a.to(dt).float(), a)
    return a.to(dev)


def _run_skinny(cuda, dt, M, N, K, seed, acts=(ACT_NONE, ACT_SILU, ACT_SIGMOID, ACT_SWIGLU), a_types=(False, True)):
    from videollama2_b200 import ops
    w_max = 2 if dt == torch.bfloat16 else 1          # fp16: see the exactness premise in the module docstring
    w_all = ints((N + 1, K), -w_max, w_max, seed, cuda, dt)
    bias_all = ints((N + 1,), -8, 8, seed + 1, cuda, torch.float32)
    a_b = ints((M, K), -2, 2, seed + 2, cuda, dt)
    a_f = _storage_ties((M, K), seed + 3, cuda, dt)
    worst = 0.0
    for a_f32, act in itertools.product(a_types, acts):
        a = a_f if a_f32 else a_b
        n = N + N % 2 if act == ACT_SWIGLU else N                 # SwiGLU needs (gate, up) pairs: N + 1 for odd N
        w, bias = w_all[:n], bias_all[:n]
        acc = a.to(dt).double() @ w.double().t()
        # every partial sum is a multiple of 2^-(bits) (the staged ties in [0.5, 1)) bounded by sum |a| |w|: fp32-exact
        # below 2^(24 - bits), bias and residual (<= 8 each) included
        assert float((a.to(dt).double().abs() @ w.double().abs().t()).max()) + 16 < 2.0 ** (24 - STORAGE_BITS[dt])
        n_out = n // 2 if act == ACT_SWIGLU else n
        for (use_bias, use_res), odt in itertools.product(((False, False), (True, True)), (torch.float32, dt)):
            use_res = use_res and act != ACT_SWIGLU
            res = ints((M, n_out), -8, 8, seed + 4, cuda, dt) if use_res else None
            buf = torch.full((M * n_out + 64,), NAN, device=cuda, dtype=odt)
            out = buf[32:32 + M * n_out].view(M, n_out)
            ops.gemm_skinny(a, w, bias=bias if use_bias else None, act=act, residual=res, out=out)
            what = f"{tag(dt)}skinny M {M} N {n} K {K} a_f32 {a_f32} act {act} bias {use_bias} res {use_res} {odt}"
            assert_nan(buf[:32], what)
            assert_nan(buf[32 + M * n_out:], what)
            ref, err = _epilogue(acc, 1.0, 0.0, bias.double() if use_bias else None, act,
                                 res.double() if use_res else None)
            worst = max(worst, _check_epilogue(out, ref, err, act == ACT_NONE, what))
    return worst


@storage_params("M", [2, 15, 16, 17, 31, 32])
def test_gemm_skinny_exact_and_bounded(cuda, dt, M):
    """M on both sides of the second 16-row pass (17..32 reuse red[]); N with clamped columns of a 16-column CTA (1, 7,
    17, 1027) and K with k-blocks dropped by the kernel's okk mask (8, 24, 40, 1032): exact for act none, element-wise
    for SiLU / sigmoid / SwiGLU; fp32 A staged on rounding ties of the storage type; NaN guards on both sides of the
    output."""
    worst = 0.0
    for N, K in itertools.product((1, 7, 17, 1000, 1027), (8, 24, 40, 1032, 4096)):
        worst = max(worst, _run_skinny(cuda, dt, M, N, K, 100 * M + 7 * N + K))
    _report(f"{tag(dt)}skinny M {M}", worst)


def _se_shapes():
    """(C, SE width) of the connector's RegStage blocks for each decoder width (timm SEModule rd = round(C / 4))."""
    from videollama2_b200 import presets
    return [(cfg["hidden_size"], int(round(cfg["hidden_size"] * 0.25)))
            for cfg in (presets.MISTRAL_7B, presets.QWEN2_7B, presets.QWEN2_72B)]


@storage_params("frames", [8, 16])
def test_gemm_skinny_se_mlp_shapes(cuda, dt, frames):
    """The SE excitation MLP as the connector runs it: fp32 pooled means (M = frames) -> C / 4 with SiLU -> C with sigmoid."""
    worst = 0.0
    for C, rd in _se_shapes():
        worst = max(worst, _run_skinny(cuda, dt, frames, rd, C, C + frames, acts=(ACT_NONE, ACT_SILU), a_types=(True,)))
        worst = max(worst, _run_skinny(cuda, dt, frames, C, rd, rd + frames, acts=(ACT_NONE, ACT_SIGMOID),
                                       a_types=(True,)))
    _report(f"{tag(dt)}skinny SE MLP frames {frames}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# c. RoPE: the decode kernels' device sincosf against the prefill GEMM's host table
# ---------------------------------------------------------------------------------------------------------------------
ROPE_THETA = 1e6
ROPE_POSITIONS = 32768      # max_position_embeddings of Mistral-7B-v0.2 and Qwen2-7B


def rope_inv_freq(D, theta=ROPE_THETA):
    """fp32 inverse frequencies, as the decoder builds them for the kernels and ops.rope_table builds them for its table."""
    return 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))


def rope_angles_fp32(n_pos, D, theta=ROPE_THETA):
    """fp32 angle pos * inv_freq[i]: one fp32 multiply, in the kernel and in ops.rope_table alike."""
    return torch.outer(torch.arange(n_pos, dtype=torch.float32), rope_inv_freq(D, theta))


def rope_table_parts(tab: torch.Tensor, dt):
    """(cos, sin) [n_pos, D/2] of storage type dt from an ops.rope_table(..., dt) int32 table."""
    c = (tab & 0xFFFF).to(torch.int16).view(dt)
    s = (tab >> 16).to(torch.int16).view(dt)
    return c, s


def rope_table_mismatches(cand_c, cand_s, tab_c, tab_s, ang32) -> int:
    """Number of (position, frequency) values where a candidate 16-bit (bf16 or fp16) cos / sin differs from the
    table's.  Each mismatch must be one ulp of the type with the exact cos / sin of the fp32 angle within 4 fp32 ulps of
    the midpoint between the two values, i.e. where two fp32 implementations accurate to 2 ulps may round to either
    neighbour."""
    a64 = ang32.double()
    total = 0
    for name, cand, tab, fn in (("cos", cand_c, tab_c, torch.cos), ("sin", cand_s, tab_s, torch.sin)):
        bad = cand.float() != tab.float()
        n = int(bad.sum())
        if n == 0:
            continue
        ci, ti = cand[bad], tab[bad]
        ub_c = ci.view(torch.int16).to(torch.int32) & 0xFFFF
        ub_t = ti.view(torch.int16).to(torch.int32) & 0xFFFF
        adjacent = ((ub_c >> 15) == (ub_t >> 15)) & ((ub_c - ub_t).abs() == 1)
        mid = (ci.double() + ti.double()) / 2
        exact = fn(a64[bad])
        ulp32 = torch.ldexp(torch.ones_like(mid), torch.frexp(mid.float())[1].to(torch.int32) - 24)
        ok = adjacent & ((exact - mid).abs() <= 4 * ulp32)
        if not bool(ok.all()):
            k = int(torch.nonzero(~ok)[0, 0])
            pos, i = torch.nonzero(bad)[k].tolist()
            raise AssertionError(f"{name} differs at position {pos}, frequency {i} ({n} mismatches): candidate "
                                 f"{float(ci[k]):.9g}, table {float(ti[k]):.9g}, exact {float(exact[k]):.9g}")
        total += n
    return total


def _rope_pattern(D, interleaved, dev):
    """One head whose rotation pairs are all (1, 0): the rotated head is (cos, sin) of every frequency."""
    if interleaved:
        return torch.tensor([1.0, 0.0], device=dev).repeat(D // 2)
    return torch.cat([torch.ones(D // 2, device=dev), torch.zeros(D // 2, device=dev)])


def _rope_split(heads, D, interleaved):
    return (heads[..., 0::2], heads[..., 1::2]) if interleaved else (heads[..., :D // 2], heads[..., D // 2:])


@pytest.mark.parametrize("D,Hq,Hkv", [(128, 64, 8), (64, 128, 8)])
@storage_params("interleaved", [True, False])
def test_rope_device_tables_match_host_table(cuda, dt, D, Hq, Hkv, interleaved):
    """vl2_rope_inplace over positions 0..32767 on (1, 0) pairs extracts the kernel's 16-bit cos / sin; they must equal
    ops.rope_table(..., dt) (what the prefill GEMM epilogue reads) up to near-midpoint roundings.  (Hq + Hkv) * D / 16 >
    512 threads, so the head loop wraps.  Then rows of N(0, 1) values at positions 0..299, 4000..4299 and 32468..32767:
    bit-exact against the fp64 rotation with the extracted cos / sin rounded to fp32 and then to the storage type.  V
    columns and the columns outside the q / k / v slices stay untouched."""
    from videollama2_b200 import ops
    S = ROPE_POSITIONS
    assert (Hq + Hkv) * D // 16 > 512
    width, nqk = (Hq + 2 * Hkv) * D, (Hq + Hkv) * D
    inv = rope_inv_freq(D).to(cuda)
    buf = torch.full((S, width + 16), NAN, device=cuda, dtype=dt)
    qkv = buf[:, 8:8 + width]
    qkv[:, :nqk] = _rope_pattern(D, interleaved, cuda).repeat(Hq + Hkv).to(dt)
    v = rnd((S, 2 * Hkv * D // 2), cuda, seed=D, dtype=dt)
    qkv[:, nqk:] = v
    ops.rope_inplace(qkv, S, Hq, Hkv, D, 0, Hq * D, 0, inv, interleaved=interleaved)
    assert_nan(buf[:, :8], "left guard")
    assert_nan(buf[:, 8 + width:], "right guard")
    assert torch.equal(qkv[:, nqk:], v), "V columns changed"
    c, s = _rope_split(qkv[:, :nqk].view(S, Hq + Hkv, D), D, interleaved)
    assert torch.equal(c, c[:, :1].expand_as(c)) and torch.equal(s, s[:, :1].expand_as(s)), "heads disagree"
    dev_c, dev_s = c[:, 0].cpu(), s[:, 0].cpu()
    tab_c, tab_s = rope_table_parts(ops.rope_table(S, D, ROPE_THETA, "cpu", dt), dt)
    n = rope_table_mismatches(dev_c, dev_s, tab_c, tab_s, rope_angles_fp32(S, D))
    print(f"rope mismatches {tag(dt)}device vs host table D {D} interleaved {interleaved}: {n} of {2 * S * D // 2}")
    del buf, qkv, c, s
    cd, sd = dev_c.double().to(cuda), dev_s.double().to(cuda)
    for pos0 in (0, 4000, S - 300):
        rows = 300
        buf = torch.full((rows, width + 16), NAN, device=cuda, dtype=dt)
        qkv = buf[:, 8:8 + width]
        qkv.copy_(rnd((rows, width), cuda, seed=pos0 + D, dtype=dt))
        orig = qkv.clone()
        ops.rope_inplace(qkv, rows, Hq, Hkv, D, 0, Hq * D, pos0, inv, interleaved=interleaved)
        x0, x1 = _rope_split(orig[:, :nqk].double().view(rows, Hq + Hkv, D), D, interleaved)
        co, sn = cd[pos0:pos0 + rows, None, :], sd[pos0:pos0 + rows, None, :]
        r0, r1 = x0 * co - x1 * sn, x1 * co + x0 * sn
        rot = torch.stack([r0, r1], -1) if interleaved else torch.cat([r0, r1], -1)
        want = rot.reshape(rows, nqk).float().to(dt)
        got = qkv[:, :nqk]
        bad = got.float() != want.float()
        assert not bad.any(), f"pos0 {pos0}: {int(bad.sum())} rotated values differ, first at {bad.nonzero()[0].tolist()}"
        assert torch.equal(qkv[:, nqk:], orig[:, nqk:]), "V columns changed"
        assert_nan(buf[:, :8], "left guard")
        assert_nan(buf[:, 8 + width:], "right guard")


@storage_params("interleaved", [True, False])
def test_decode_rope_append_matches_rope_inplace(cuda, dt, interleaved):
    """vl2_decode_rope_append at positions 0, 1, 4095, 32767 and the last row of a 40000-row cache: the stage row and
    cache[pos] are bit-identical to vl2_rope_inplace of the same row at that position; every other cache row, and the
    columns beside the cache in its row-strided buffer, stay NaN."""
    from videollama2_b200 import ops
    Hq, Hkv, D, cap = 64, 8, 128, 40000
    width = (Hq + 2 * Hkv) * D
    inv = rope_inv_freq(D).to(cuda)
    buf = torch.full((cap, width + 16), NAN, device=cuda, dtype=dt)
    cache = buf[:, 8:8 + width]
    for pos in (0, 1, 4095, 32767, cap - 1):
        row = rnd((1, width), cuda, seed=pos, dtype=dt)
        stage = row.clone()
        ops.decode_rope_append(stage, cache, torch.tensor([pos], device=cuda, dtype=torch.int32), Hq, Hkv, D, inv,
                               interleaved=interleaved)
        ref = row.clone()
        ops.rope_inplace(ref, 1, Hq, Hkv, D, 0, Hq * D, pos, inv, interleaved=interleaved)
        assert pos == 0 or not torch.equal(ref, row)        # position 0 rotates by the identity
        assert torch.equal(stage, ref), f"stage row at position {pos}"
        assert torch.equal(cache[pos:pos + 1], ref), f"cache row {pos}"
        cache[pos] = NAN
        assert_nan(buf, f"cache outside row {pos}")


# ---------------------------------------------------------------------------------------------------------------------
# d. LayerNorm / RMSNorm on every dispatch branch
# ---------------------------------------------------------------------------------------------------------------------
# warp kernel NV = 1 (C <= 256), 2 (<= 512), 4 (<= 1024), 6 (<= 1536, SigLIP's 1152), 16 (<= 4096); streaming above
LN_C = [8, 256, 264, 512, 520, 1024, 1032, 1152, 1536, 1544, 3584, 4096, 4104, 8192]
NORM_ROWS = [1, 7, 9, 1521]


def _ln_input(family, rows, C, seed, dev, dt):
    g = torch.Generator().manual_seed(seed)
    if family == "normal":
        x = torch.randn(rows, C, generator=g)
    else:
        mu = (torch.rand(rows, 1, generator=g) * 20 + 20) * torch.where(torch.rand(rows, 1, generator=g) < 0.5, -1.0, 1.0)
        x = mu + (torch.randn(rows, C, generator=g) if family == "large_mean" else torch.zeros(rows, C))
    return x.to(dt).to(dev)


@storage_params("C", LN_C)
def test_layernorm_every_branch_bounded(cuda, dt, C):
    """N(0, 1) rows, rows with mean +-20..40 and std 1 (the streaming kernel takes E[x^2] - mu^2 in one pass), constant
    rows (exact mean: the output is the storage type's rounding of beta + residual, bit for bit); with and without
    residual, act none and SiLU, written between NaN rows.  Bound: _ln_rows_bound, the residual add, SiLU, the rounding
    into the storage type."""
    from videollama2_b200 import ops
    gamma = rnd((C,), cuda, 0.1, seed=C, dtype=dt) + 1
    beta = rnd((C,), cuda, 0.5, seed=C + 1, dtype=dt)
    gd, bd = gamma.double(), beta.double()
    worst = 0.0
    for rows, family in itertools.product(NORM_ROWS, ("normal", "large_mean", "constant")):
        x = _ln_input(family, rows, C, rows * C + len(family), cuda, dt)
        y, err_y = _ln_rows_bound(x.double(), torch.zeros_like(x, dtype=torch.float64), gd, bd)
        for use_res, act in itertools.product((False, True), (ACT_NONE, ACT_SILU)):
            res = rnd((rows, C), cuda, seed=rows + C, dtype=dt) if use_res else None
            buf = torch.full((rows + 2, C), NAN, device=cuda, dtype=dt)
            out = buf[1:rows + 1]
            ops.layernorm(x, gamma, beta, 1e-5, act=act, residual=res, out=out)
            what = f"{tag(dt)}layernorm C {C} rows {rows} {family} res {use_res} act {act}"
            assert_nan(buf[0], what)
            assert_nan(buf[rows + 1], what)
            z, err = y, err_y
            if use_res:
                z = y + res.double()
                err = err + F32_U * z.abs()
            if family == "constant" and act == ACT_NONE:
                want = (beta.float() + (res.float() if use_res else 0.0)).to(dt).expand(rows, C)
                assert torch.equal(out, want), what
            ref = z
            if act == ACT_SILU:
                ref = torch.nn.functional.silu(z)
                err = ACT_SLOPE * err + _act_rel(z) * ref.abs()
            worst = max(worst, check_elementwise(out, ref, storage_bound(ref, err, dt), what))
    _report(f"{tag(dt)}layernorm C {C}", worst)


def rmsnorm_reference(x, gamma, dt):
    """fp64 HF RMSNorm gamma * dt(x * rstd) of rows x [R, C] of storage type dt and the fp32 error bound of the kernel's
    result before its final rounding: where x * rstd lies within the fp32 error of x * rstd (fp32 sum of squares, the
    division and + eps, rsqrtf) of a rounding midpoint of dt, the kernel may round to the other neighbour (one ulp)."""
    C = x.shape[1]
    xd = x.double()
    ms = xd.pow(2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(ms + 1e-5)
    rel = (C * F32_U * ms + 2 * F32_U * (ms + 1e-5)) / (2 * (ms + 1e-5)) + 2.0 ** -21
    t = xd * rstd
    e_t = t.abs() * (rel + F32_U)
    tb = t.float().to(dt).double()
    ulp = storage_ulp(t, dt)
    d_t = torch.where(((t - tb).abs() - ulp / 2).abs() <= e_t, ulp, torch.zeros_like(ulp))
    return gamma.double() * tb, gamma.double().abs() * d_t


@storage_params("C", [8, 256, 264, 512, 520, 1024, 1032, 4096, 8192])
def test_rmsnorm_every_branch_bounded(cuda, dt, C):
    """vl2_rmsnorm on the NV = 1 / 2 / 4 warp kernels and the streaming kernel, against HF's double rounding."""
    from videollama2_b200 import ops
    gamma = rnd((C,), cuda, 0.1, seed=C + 2, dtype=dt) + 1
    worst = 0.0
    for rows in NORM_ROWS:
        x = rnd((rows, C), cuda, 3.0, seed=rows + C, dtype=dt)
        buf = torch.full((rows + 2, C), NAN, device=cuda, dtype=dt)
        out = buf[1:rows + 1]
        ops.rmsnorm(x, gamma, 1e-5, out=out)
        assert_nan(buf[0], "row before")
        assert_nan(buf[rows + 1], "row after")
        ref, err = rmsnorm_reference(x, gamma, dt)
        worst = max(worst, check_elementwise(out, ref, storage_bound(ref, err, dt), f"{tag(dt)}rmsnorm C {C} rows {rows}"))
    _report(f"{tag(dt)}rmsnorm C {C}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# e. row statistics
# ---------------------------------------------------------------------------------------------------------------------
@storage_params("C", [8, 264, 4096, 8192, 14336])
def test_row_statistics_exact(cuda, dt, C):
    """Integers in {-3..3}: sums and sums of squares (<= 9 * 14336) are exact in fp32 in any order."""
    from videollama2_b200 import ops
    for rows in (1, 13, 1003):
        x = ints((rows, C), -3, 3, rows + C, cuda, dt)
        xd = x.double()
        assert torch.equal(ops.row_sumsq(x).double()[:, 0], xd.pow(2).sum(-1)), (rows, C)
        s, q = ops.row_stats(x)
        assert torch.equal(s.double()[:, 0], xd.sum(-1)), (rows, C)
        assert torch.equal(q.double()[:, 0], xd.pow(2).sum(-1)), (rows, C)


# ---------------------------------------------------------------------------------------------------------------------
# f. STC connector: depthwise 3x3 + LN + SiLU, SE pooling, SE scale
# ---------------------------------------------------------------------------------------------------------------------
@storage_params("F,H,W,C", [(1, 1, 1, 8), (1, 1, 1, 64), (1, 1, 2, 64), (1, 3, 5, 64), (3, 4, 7, 8), (3, 2, 3, 64),
                             (1, 5, 2, 4096), (3, 3, 5, 4096), (1, 1, 1, 4112), (3, 4, 3, 4112), (2, 3, 4, 6144),
                             (3, 2, 5, 8192), (1, 1, 2, 8192), (16, 4, 4, 512)])
def test_dwconv_ln_silu_pool_scale(cuda, dt, F, H, W, C):
    """Integer x and weights make the 3x3 depthwise conv exact; the LN + SiLU is bounded with _ln_rows_bound.  C = 8
    leaves one active thread, 4096 takes 512 threads, 4112 / 6144 / 8192 split a pixel row over a 2-CTA cluster.  With
    F > 1 the even frames hold a large constant, so a padding tap leaking across frames moves the border pixels of
    the odd frames far outside the bound.  pooled = fp64 mean of the 16-bit y as written, within (H W + 2) 2^-24 of
    mean |y|; vl2_se_scale is bit-identical to torch's fp32 multiply and rounding into the storage type."""
    from videollama2_b200 import ops
    x = ints((F, H, W, C), -2, 2, F * H * W + C, cuda, dt)
    if F > 1:
        x[0::2] = torch.tensor([48.0, -40.0], device=cuda).repeat(F)[:(F + 1) // 2, None, None, None].to(x.dtype)
    wd = ints((C, 1, 3, 3), -2, 2, C + 1, cuda, dt)
    w9c = wd.reshape(C, 9).t().contiguous()
    gamma = rnd((C,), cuda, 0.1, seed=C + 2, dtype=dt) + 1
    beta = rnd((C,), cuda, 0.5, seed=C + 3, dtype=dt)
    y, pooled = ops.dwconv3x3_ln_silu(x, w9c, gamma, beta, 1e-5)
    conv = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wd.double(), padding=1, groups=C)
    conv = conv.permute(0, 2, 3, 1).reshape(-1, C)
    assert torch.equal(conv.float().double(), conv)
    z, err = _ln_rows_bound(conv, torch.zeros_like(conv), gamma.double(), beta.double())
    ref = torch.nn.functional.silu(z)
    err = ACT_SLOPE * err + _act_rel(z) * ref.abs()
    what = f"{tag(dt)}dwconv F {F} H {H} W {W} C {C}"
    worst = check_elementwise(y.reshape(-1, C), ref, storage_bound(ref, err, dt), what, tile=(W, C))
    yd = y.double()
    pool_ref = yd.mean((1, 2))
    pool_bound = (H * W + 2) * F32_U * yd.abs().mean((1, 2)) + 1e-30
    worst_pool = check_elementwise(pooled, pool_ref, pool_bound, f"SE pooling {what}")
    s = torch.rand((F, C), generator=torch.Generator().manual_seed(C)).add(0.5).to(cuda)
    n = F * H * W * C
    buf = torch.full((n + 128,), NAN, device=cuda, dtype=dt)
    ys = buf[64:64 + n].view(F, H, W, C)
    ys.copy_(y)
    ops.se_scale(ys, s)
    assert torch.equal(ys, (y.float() * s[:, None, None, :]).to(dt)), f"se_scale {what}"
    assert_nan(buf[:64], "se_scale before")
    assert_nan(buf[64 + n:], "se_scale after")
    _report(f"dwconv+LN+SiLU {what}", worst)
    _report(f"SE pooling {what}", worst_pool)


# ---------------------------------------------------------------------------------------------------------------------
# g. glue: im2col gathers, embedding splice, CLIP embedding finish
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pad", [0, 1])
@storage_params("T,H,W,C", [(3, 5, 7, 8), (4, 6, 6, 64), (5, 9, 11, 16), (2, 3, 2, 4096), (16, 24, 24, 8)])
def test_conv3d_im2col_exact(cuda, dt, T, H, W, C, pad):
    """A[(t', h', w'), tap * C + c] = x[2t' - pad + dt, 2h' - pad + dh, 2w' - pad + dw, c], zero outside x, written into a
    NaN buffer (so the zero taps are stores, not leftovers): bit-exact."""
    x = rnd((T, H, W, C), cuda, seed=T * H * W + C, dtype=dt)
    To, Ho, Wo = (T + 2 * pad - 2) // 2 + 1, (H + 2 * pad - 2) // 2 + 1, (W + 2 * pad - 2) // 2 + 1
    M = To * Ho * Wo
    buf = torch.full((M * 8 * C + 16,), NAN, device=cuda, dtype=dt)
    A = buf[8:8 + M * 8 * C].view(M, 8 * C)
    _abi(dt, "vl2_conv3d_im2col", x.data_ptr(), A.data_ptr(), T, H, W, C, pad, To, Ho, Wo)
    xp = torch.nn.functional.pad(x, (0, 0, pad, pad, pad, pad, pad, pad))
    taps = [xp[dt:dt + 2 * To:2, dh:dh + 2 * Ho:2, dw:dw + 2 * Wo:2] for dt in (0, 1) for dh in (0, 1) for dw in (0, 1)]
    assert torch.equal(A, torch.stack(taps, 3).reshape(M, 8 * C))
    assert_nan(buf[:8], "before A")
    assert_nan(buf[8 + M * 8 * C:], "after A")


@storage_params("F,H,W,Kpad", [(2, 336, 336, 640), (1, 384, 384, 640), (3, 42, 70, 704), (2, 28, 14, 592)])
def test_patch_im2col_exact(cuda, dt, F, H, W, Kpad):
    """P = 14 (CLIP and SigLIP): A = unfold(pixels) bit for bit, columns K..Kpad zero; SigLIP's 384 px leaves 6 pixels of
    every row and column unused; non-square frames; written into a NaN buffer."""
    P = 14
    K = 3 * P * P
    px = rnd((F, 3, H, W), cuda, seed=H + W + F, dtype=dt)
    M = F * (H // P) * (W // P)
    buf = torch.full((M * Kpad + 16,), NAN, device=cuda, dtype=dt)
    A = buf[8:8 + M * Kpad].view(M, Kpad)
    _abi(dt, "vl2_patch_im2col", px.data_ptr(), A.data_ptr(), F, H, W, P, Kpad)
    ref = torch.nn.functional.unfold(px.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(M, K)
    assert torch.equal(A[:, :K].float(), ref)
    assert torch.equal(A[:, K:], torch.zeros_like(A[:, K:]))
    assert_nan(buf[:8], "before A")
    assert_nan(buf[8 + M * Kpad:], "after A")


@storage_params("H", [264, 4096])
def test_embed_splice_exact(cuda, dt, H):
    """ids -1 (placeholder), vocab (invalid), vocab - 1, 0 and duplicated ids: rows with a valid id are the table row bit
    for bit; rows with an invalid id and rows not listed stay NaN."""
    from videollama2_b200 import ops
    V = 1000
    table = rnd((V, H), cuda, seed=H, dtype=dt)
    ids_l = [-1, V, V - 1, 0, 5, 5, V - 1, 17, -201]
    dst_l = [0, 1, 2, 3, 4, 7, 8, 10, 11]
    out = torch.full((13, H), NAN, device=cuda, dtype=dt)
    ops.embed_splice(torch.tensor(ids_l, device=cuda), torch.tensor(dst_l, device=cuda, dtype=torch.int32), table, out)
    written = set()
    for i, d in zip(ids_l, dst_l):
        if 0 <= i < V:
            assert torch.equal(out[d], table[i]), (i, d)
            written.add(d)
    for d in range(13):
        if d not in written:
            assert_nan(out[d], f"row {d}")


@storage_params("C", [128, 1024, 8192, 16384])
def test_clip_embed_finish_bounded(cuda, dt, C):
    """[cls + pos[0]; patch + pos[1:]] per frame, then LayerNorm, row by row; C > 4096 holds several of a thread's
    kMaxVec vectors.  The fp32 sums are an input error of 2^-24 |x| for _ln_rows_bound."""
    from videollama2_b200 import ops
    F, npch = 3, 7
    patch = rnd((F * npch, C), cuda, seed=C, dtype=dt)
    cls = rnd((C,), cuda, seed=C + 1, dtype=dt)
    pos = rnd((npch + 1, C), cuda, 2.0, seed=C + 2, dtype=dt)
    gamma = rnd((C,), cuda, 0.1, seed=C + 3, dtype=dt) + 1
    beta = rnd((C,), cuda, 0.1, seed=C + 4, dtype=dt)
    tok = ops.clip_embed_finish(patch, cls, pos, gamma, beta, F, 1e-5)
    x = torch.cat([(cls.double() + pos[0].double()).expand(F, 1, C),
                   patch.double().view(F, npch, C) + pos[1:].double()], 1).reshape(-1, C)
    ref, err = _ln_rows_bound(x, F32_U * x.abs(), gamma.double(), beta.double())
    _report(f"{tag(dt)}clip embed finish C {C}",
            check_elementwise(tok, ref, storage_bound(ref, err, dt), f"{tag(dt)}clip embed finish C {C}",
                              tile=(npch + 1, C)))


# ---------------------------------------------------------------------------------------------------------------------
# h. fp16 only: the top of the range and the subnormals
# ---------------------------------------------------------------------------------------------------------------------
H16 = torch.float16


def _top_of_range_classes(ref64: torch.Tensor) -> None:
    """ref64 holds, at both signs, exactly 65504, values in (65504, 65520) (rounding to 65504) and values >= 65520
    (rounding to inf)."""
    for sgn in (1.0, -1.0):
        r = ref64 * sgn
        assert bool((r == FP16_MAX).any()) and bool(((r > FP16_MAX) & (r < 65520.0)).any()) and bool((r >= 65520.0).any())


def _pin_top_columns(w, bias, n_cols=64):
    """Columns 0..n_cols-1 of w [N, K] (16-bit) and bias [N] (fp32) such that result n is exactly +-65504 (A's column
    0, 65504, times w[n, 0] = +-1) plus an integer from -8 to 23: every case of _top_of_range_classes, at both signs."""
    n = torch.arange(n_cols)
    sgn = torch.where(n % 2 == 0, 1.0, -1.0)
    w[:n_cols, 1:] = 0
    w[:n_cols, 0] = sgn.to(w.device, w.dtype)
    bias[:n_cols] = (sgn * ((n // 2) % 32 - 8)).to(bias.device)


def test_fp16_gemv_overflow_rounds_like_torch(cuda):
    """GEMV (__float2half_rn store): x[0] = 65504 and x[1] = 32752 times w[n, 0] in {-2, -1, 1, 2} and w[n, 1] in
    {-2..2}, plus an integer sum of the remaining 62 terms, plus an fp32 bias with a fractional part of 0 or 0.75 and
    an integer residual (columns pinned by _pin_top_columns): every result fp32-exact, the 16-bit output torch's
    rounding (65504 kept, 65519.75 to 65504, >= 65520 to inf), the fp32 output the exact value; no NaN.  Both
    row-per-warp variants (N < 8192 and N >= 8192)."""
    from videollama2_b200 import ops
    K = 64
    for N in (4096, 8194):
        x = ints((K,), -2, 2, 301, cuda, H16)
        x[0] = FP16_MAX
        x[1] = 32752.0
        w = ints((N, K), -1, 1, 302, cuda, H16)
        g = torch.Generator().manual_seed(303)
        w[:, 0] = torch.tensor([-2.0, -1.0, 1.0, 2.0])[torch.randint(0, 4, (N,), generator=g)].to(cuda, H16)
        w[:, 1] = torch.randint(-2, 3, (N,), generator=g).to(cuda, H16)
        bias = (torch.randint(-40, 41, (N,), generator=g) + 0.75 * torch.randint(0, 2, (N,), generator=g)).float().to(cuda)
        res = ints((N,), -8, 8, 304, cuda, H16)
        _pin_top_columns(w, bias)
        res[:64] = 0
        ref = w.double() @ x.double() + bias.double() + res.double()
        _top_of_range_classes(ref)
        out = ops.gemv(x, w, bias=bias, residual=res)
        assert not bool(torch.isnan(out).any())
        assert torch.equal(out[0], to_storage_exact(ref, H16)), N
        o32 = ops.gemv(x, w, bias=bias, residual=res, out_dtype=torch.float32)
        assert torch.equal(o32[0].double(), ref), N


@pytest.mark.parametrize("a_f32", [False, True])
def test_fp16_skinny_overflow_and_staging(cuda, a_f32):
    """Skinny GEMM (mma.sync, __float2half_rn store) at the top of the range.  Column 0 of A holds 65504 (and, for the
    fp32 A, 65519 and 65519.99, which stage to 65504, and 65520 / -70000, which stage to +-inf); w[:, 0] in {-2, -1, 1,
    2}, the other columns are small integers, so a row's result is +-65504 or +-131008 plus an integer (+ a bias of 0 or
    0.75 + residual) - fp32-exact, or +-inf for the staged infinities (one infinite term per row, w[:, 0] never 0: no
    NaN).  Both output types; the reference stages A like torch's .to(float16)."""
    from videollama2_b200 import ops
    M, N, K = 7, 1000, 40
    g = torch.Generator().manual_seed(311 + a_f32)
    a = torch.randint(-2, 3, (M, K), generator=g).double()
    col0 = [FP16_MAX, -FP16_MAX, FP16_MAX, 32752.0, -32752.0, FP16_MAX, -FP16_MAX]
    if a_f32:
        col0 = [FP16_MAX, 65519.0, 65519.99, 65520.0, -70000.0, -65519.0, -FP16_MAX]
    a[:, 0] = torch.tensor(col0, dtype=torch.float64)
    a_dev = (a.float() if a_f32 else a.to(H16)).to(cuda)
    w = ints((N, K), -2, 2, 312, cuda, H16)
    w[:, 0] = torch.tensor([-2.0, -1.0, 1.0, 2.0])[torch.randint(0, 4, (N,), generator=g)].to(cuda, H16)
    bias = (torch.randint(-40, 41, (N,), generator=g) + 0.75 * torch.randint(0, 2, (N,), generator=g)).float().to(cuda)
    res = ints((M, N), -8, 8, 313, cuda, H16)
    _pin_top_columns(w, bias)
    res[:, :64] = 0
    staged = a_dev.cpu().to(H16).double().to(cuda)
    if a_f32:
        assert torch.equal(staged[:, 0].cpu(), torch.tensor([FP16_MAX, FP16_MAX, FP16_MAX, math.inf, -math.inf, -FP16_MAX,
                                                             -FP16_MAX], dtype=torch.float64))
    ref = staged @ w.double().t() + bias.double() + res.double()
    assert not bool(torch.isnan(ref).any())
    _top_of_range_classes(torch.nan_to_num(ref, posinf=0.0, neginf=0.0))
    for odt in (H16, torch.float32):
        out = ops.gemm_skinny(a_dev, w, bias=bias, residual=res, out_dtype=odt)
        assert not bool(torch.isnan(out).any()), odt
        want = ref.float().to(odt)
        assert torch.equal(out, want), odt


@pytest.mark.parametrize("C", [256, 1024, 4096, 8192])
def test_fp16_norms_overflow_rounds_like_torch(cuda, C):
    """LayerNorm and RMSNorm stores at the top of the range, on inputs where the fp32 result is exact:
      * large beta: constant rows (x - mu = 0 exactly) give beta + residual; beta = +-65504 / +-65472 with integer
        residuals crosses 65504, 65520 and beyond;
      * large gamma: rows of alternating +-1 (mu = 0, var = 1, eps = 0: rstd = 1) give +-gamma + beta with gamma up to
        65504 and beta in {0, 8, 15, 17, 32} - at least 0.5 away from 65520, so a 2-ulp rstd cannot move the rounding;
      * RMSNorm: rows [2, 0, 0, 0, ...] (mean square 1, eps = 0) give gamma * 2 with gamma in {16384, 32752, 32768,
        -32768, -32752}: 32768, 65504, +inf, -inf, -65504.
    Every 16-bit output equals torch's rounding of the fp64 value; no NaN."""
    from videollama2_b200 import ops
    rows = 24
    cc = torch.arange(C)
    g = torch.Generator().manual_seed(C)
    # large beta
    beta = torch.tensor([FP16_MAX, -FP16_MAX, 65472.0, -65472.0])[cc % 4].to(H16)
    gamma = torch.ones(C, dtype=H16)
    x = torch.full((rows, C), 3.0, dtype=H16)
    res = torch.randint(-40, 41, (rows, C), generator=g).to(H16)
    ref = beta.double() + res.double()
    _top_of_range_classes(ref)
    out = ops.layernorm(x.to(cuda), gamma.to(cuda), beta.to(cuda), 1e-5, residual=res.to(cuda))
    assert not bool(torch.isnan(out).any())
    assert torch.equal(out.cpu(), to_storage_exact(ref, H16)), "large beta"
    # large gamma
    gamma = torch.tensor([FP16_MAX, -FP16_MAX, 65472.0, 16.0])[cc % 4].to(H16)
    beta = torch.tensor([0.0, 8.0, 15.0, 17.0, 32.0, -8.0, -17.0, -32.0])[(cc // 4) % 8].to(H16)
    sgn = torch.where((cc + torch.arange(rows)[:, None]) % 2 == 0, 1.0, -1.0)
    x = sgn.to(H16)
    ref = sgn.double() * gamma.double() + beta.double()
    _top_of_range_classes(ref)
    out = ops.layernorm(x.to(cuda), gamma.to(cuda), beta.to(cuda), 0.0)
    assert not bool(torch.isnan(out).any())
    assert torch.equal(out.cpu(), to_storage_exact(ref, H16)), "large gamma"
    # RMSNorm
    gamma = torch.tensor([16384.0, 32752.0, 32768.0, -32768.0, -32752.0])[cc % 5].to(H16)
    x = torch.zeros(rows, C)
    x[torch.arange(rows)[:, None], (torch.arange(C // 4)[None, :] * 4 + torch.arange(rows)[:, None] % 4)] = 2.0
    ref = x.double() * gamma.double()
    out = ops.rmsnorm(x.to(H16).to(cuda), gamma.to(cuda), 0.0)
    assert not bool(torch.isnan(out).any())
    want = to_storage_exact(ref, H16)
    assert bool(torch.isinf(want).any()) and bool((want.abs() == FP16_MAX).any())
    assert torch.equal(out.cpu(), want), "rmsnorm"


def test_fp16_gemv_subnormals(cuda):
    """GEMV on fp16 subnormal x (k 2^-24, |k| <= 1023) and w in {-2..2} / 4: the products (multiples of 2^-26) and their
    sums are fp32-exact; the 16-bit output must be torch's rounding onto the 2^-24 subnormal grid (round to nearest
    even), the fp32 output the exact value.  Flushed inputs or outputs give zeros."""
    from videollama2_b200 import ops
    N, K = 4096, 1032
    x = subnormals((K,), 1023, 321, cuda)
    w = (ints((N, K), -2, 2, 322, cuda, torch.float32) / 4).to(H16)
    ref = w.double() @ x.double()
    out = ops.gemv(x, w)
    want = to_storage_exact(ref, H16)
    sub = (want != 0) & (want.abs() < 2.0 ** -14)
    assert int(sub.sum()) > 100 and bool((want.double() != ref).any())
    assert torch.equal(out[0], want)
    assert torch.equal(ops.gemv(x, w, out_dtype=torch.float32)[0].double(), ref)


@pytest.mark.parametrize("a_f32", [False, True])
def test_fp16_skinny_subnormal_operands(cuda, a_f32):
    """Skinny GEMM (mma.sync) with fp16 subnormal operands: W = k 2^-24 (|k| <= 63); A the same as a 16-bit operand,
    or as an fp32 operand (2k+1) 2^-25, which must stage to the even neighbour on the 2^-24 grid.  Products k k' 2^-48
    and their sums (< 1032 * 2^12 * 2^-48) are fp32-exact, so the fp32 output must equal the fp64 product; a flushed
    operand or a truncating staging would change it."""
    from videollama2_b200 import ops
    M, N, K = 9, 1000, 1032
    w = subnormals((N, K), 63, 331, cuda)
    if a_f32:
        g = torch.Generator().manual_seed(332)
        a = ((2 * torch.randint(-63, 63, (M, K), generator=g) + 1).double() * 2.0 ** -25).float().to(cuda)
        assert not torch.equal(a.to(H16).float(), a)
    else:
        a = subnormals((M, K), 63, 332, cuda)
    ref = a.to(H16).double() @ w.double().t()
    assert bool((ref != 0).any())
    out = ops.gemm_skinny(a, w, out_dtype=torch.float32)
    assert torch.equal(out.double(), ref)


@pytest.mark.parametrize("C", [256, 1152, 8192])
def test_fp16_layernorm_subnormal_input(cuda, C):
    """LayerNorm of rows of fp16 subnormals (k 2^-24, |k| <= 1023), gamma = 1, beta = 0, eps = 1e-5: the variance is far
    below eps, so y = (x - mu) * rstd ~ 316 (x - mu), a few 1e-5 at most - normal and subnormal fp16 outputs.  Flushed
    inputs would give y = 0, failing the bound (storage_bound with _ln_rows_bound) by orders of magnitude."""
    from videollama2_b200 import ops
    rows = 33
    x = subnormals((rows, C), 1023, 341 + C, cuda)
    gamma = torch.ones(C, device=cuda, dtype=H16)
    beta = torch.zeros(C, device=cuda, dtype=H16)
    out = ops.layernorm(x, gamma, beta, 1e-5)
    y, err = _ln_rows_bound(x.double(), torch.zeros_like(x, dtype=torch.float64), gamma.double(), beta.double())
    assert float(y.abs().max()) > 2.0 ** -14 and bool((out != 0).any())
    _report(f"fp16 layernorm subnormal input C {C}", check_elementwise(out, y, storage_bound(y, err, H16),
                                                                         f"fp16 layernorm subnormal input C {C}"))

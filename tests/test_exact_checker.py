"""Self-tests of the checks in test_kernels_exact_gpu.py and test_rowops_decode_exact_gpu.py, on the CPU: plant the
faults a whole-tensor relL2 < 6e-3 lets through into a correct fp64 result and show that the element-wise checker
rejects each of them, while it accepts the correctly rounded result.  Also checks on the CPU that the attention routing
problems route (fp64 softmax is one-hot on the target), that the RoPE table matcher tells rounding noise from a
wrong table, and that the all-reduce expectation of test_tp_allreduce_gpu.py pins the rank order, the fp32 accumulation
and the statistics of the rounded sum."""
import math

import pytest
import torch

from test_kernels_exact_gpu import (FP16_MAX, STORAGE_TYPES, _ln_rows_bound, _routing_problem, attention_reference,
                                    check_elementwise, exact_softmax_scale, gemm_acc_bound, relerr, storage_bound,
                                    storage_params, to_storage_exact)
from test_rowops_decode_exact_gpu import (ROPE_POSITIONS, ROPE_THETA, rope_angles_fp32, rope_table_mismatches,
                                          rope_table_parts)
from test_tp_allreduce_gpu import expected_sum, make_partials, stats_violations, to_storage

CPU = torch.device("cpu")


def _bf16_randn(shape, scale, seed):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(torch.bfloat16)


def test_checker_rejects_one_wrong_row():
    """One row of an 1100-row GEMM output off by 10 %: relL2 3e-3, far under the 6e-3 bar."""
    M, N, K = 1100, 1024, 328
    a, w = _bf16_randn((M, K), 1.0, 1), _bf16_randn((N, K), 0.06, 2)
    ref = a.double() @ w.double().t()
    bound = storage_bound(ref, gemm_acc_bound(a, w), torch.bfloat16)
    good = ref.float().to(torch.bfloat16)
    assert check_elementwise(good, ref, bound, "correct") <= 1.0
    bad = good.clone()
    bad[517] = (bad[517].float() * 1.1).to(torch.bfloat16)
    assert relerr(bad, ref) < 6e-3
    with pytest.raises(AssertionError, match=r"row 517"):
        check_elementwise(bad, ref, bound, "one row off")


def test_checker_rejects_one_missing_k_block():
    """One of 224 k-blocks (K = 14336, the decoder's down_proj depth) missing from one 128 x 64 tile of 256."""
    M, N, K = 2048, 1024, 14336
    a, w = _bf16_randn((M, K), 1.0, 3), _bf16_randn((N, K), K ** -0.5, 4)
    ref = a.double() @ w.double().t()
    bound = storage_bound(ref, gemm_acc_bound(a, w), torch.bfloat16)
    good = ref.float().to(torch.bfloat16)
    assert check_elementwise(good, ref, bound, "correct") <= 1.0
    r0, c0, k0 = 5 * 128, 7 * 64, 100 * 64
    faulty = ref.clone()
    faulty[r0:r0 + 128, c0:c0 + 64] -= a[r0:r0 + 128, k0:k0 + 64].double() @ w[c0:c0 + 64, k0:k0 + 64].double().t()
    bad = faulty.float().to(torch.bfloat16)
    assert relerr(bad, ref) < 6e-3
    with pytest.raises(AssertionError, match=r"in tile \(5, 7\)"):
        check_elementwise(bad, ref, bound, "missing k-block", tile=(128, 64))


def test_checker_rejects_one_leaked_masked_key():
    """Causal attention (S = 512, 4 heads, D = 64, N(0, 1) logits) where row 40 of head 1 also sees key 41."""
    S, H, D = 512, 4, 64
    q, k, v = (_bf16_randn((H, S, D), 1.0, s) for s in (5, 6, 7))
    scale = D ** -0.5
    ref, bound = attention_reference(q, k, v, True, scale, torch.bfloat16)
    good = ref.float().to(torch.bfloat16)
    assert check_elementwise(good, ref, bound, "correct", tile=(128, D)) <= 1.0
    s = (q[1, 40].double() @ k[1, :42].double().t()) * scale
    leaked = ref.clone()
    leaked[1, 40] = torch.softmax(s, -1) @ v[1, :42].double()
    bad = leaked.float().to(torch.bfloat16)
    assert relerr(bad, ref) < 6e-3
    with pytest.raises(AssertionError, match=r"row 40"):
        check_elementwise(bad[1], ref[1], bound[1], "leaked key", tile=(128, D))


@pytest.mark.parametrize("B,S,Hq,Hkv,D,causal", [(3, 257, 28, 4, 128, True), (3, 129, 4, 4, 40, False), (3, 45, 2, 2, 8, True),
                                                 (1, 300, 4, 2, 72, True)])
def test_routing_problem_is_one_hot(B, S, Hq, Hkv, D, causal):
    """The logits the routing problems build give an fp64 softmax that is one-hot on the intended target, with the poison
    keys (past the causal boundary, in the next batch's first rows) winning if they were visible."""
    for dt in STORAGE_TYPES:
        _check_routing_problem(B, S, Hq, Hkv, D, causal, dt)


def _check_routing_problem(B, S, Hq, Hkv, D, causal, dt):
    q, k, v, target = _routing_problem(B, S, Hq, Hkv, D, causal, dt)
    scale, sl2 = exact_softmax_scale()
    assert sl2 == 0.125
    G = Hq // Hkv
    for b in range(B):
        qf = q[b].transpose(0, 1)
        kf = k[b].transpose(0, 1).repeat_interleave(G, 0)
        s = (qf @ kf.transpose(1, 2)) * sl2                                 # log2 units
        if causal:
            s = s.masked_fill(torch.ones(S, S, dtype=torch.bool).triu(1), -math.inf)
        top2 = s.topk(min(2, S), -1).values
        assert torch.equal(s.argmax(-1), target[b].t())
        if S > 1:
            gap = top2[..., 0] - top2[..., 1]
            rows_with_two = torch.isfinite(top2[..., 1])
            assert bool((gap[rows_with_two] >= 40).all())
        if b + 1 < B and S % 128:
            # what a 2-D box past this batch's tail would read: the next batch's first rows beat every target
            n_pad = min(S, -S % 128)
            kn = k[b + 1, :n_pad].transpose(0, 1).repeat_interleave(G, 0)
            leak = (qf @ kn.transpose(1, 2)) * sl2
            assert bool((leak.amax(-1) > top2[..., 0]).all())


def test_checker_rejects_one_layernorm_row_one_percent_off():
    """LayerNorm of 1521 rows x 1024 with one row 1 % off: relL2 < 4e-3 (the bar of the relL2 LayerNorm tests) passes
    it, the _ln_rows_bound check does not."""
    R, C = 1521, 1024
    x = _bf16_randn((R, C), 1.0, 8).double()
    gamma = (_bf16_randn((C,), 0.1, 9).float() + 1).to(torch.bfloat16).double()
    beta = _bf16_randn((C,), 0.5, 10).double()
    ref, err = _ln_rows_bound(x, torch.zeros_like(x), gamma, beta)
    bound = storage_bound(ref, err, torch.bfloat16)
    good = ref.float().to(torch.bfloat16)
    assert check_elementwise(good, ref, bound, "correct") <= 1.0
    bad = good.clone()
    bad[700] = (bad[700].float() * 1.01).to(torch.bfloat16)
    assert relerr(bad, ref) < 4e-3
    with pytest.raises(AssertionError, match=r"row 700"):
        check_elementwise(bad, ref, bound, "one row 1 % off")


def _rope_fp64_table(ang32, dt):
    """cos / sin of the fp32 angles rounded from fp64 to the storage type dt: the correctly rounded table."""
    a = ang32.double()
    return a.cos().float().to(dt), a.sin().float().to(dt)


@storage_params("D", [128, 64])
def test_rope_matcher_accepts_host_table(dt, D):
    """ops.rope_table (fp32 cos / sin of torch) against the correctly rounded table over 32768 positions: the few
    differences are one-ulp roundings next to a midpoint, which the matcher accepts."""
    from videollama2_b200 import ops
    ang = rope_angles_fp32(ROPE_POSITIONS, D)
    tc, ts = rope_table_parts(ops.rope_table(ROPE_POSITIONS, D, ROPE_THETA, "cpu", dt), dt)
    fc, fs = _rope_fp64_table(ang, dt)
    n = rope_table_mismatches(tc, ts, fc, fs, ang)
    assert n <= 64, n
    assert rope_table_mismatches(tc, ts, tc, ts, ang) == 0


def test_rope_matcher_rejects_off_by_one_position():
    """The table of position p + 1 used for position p, in both storage types."""
    from videollama2_b200 import ops
    D = 128
    ang = rope_angles_fp32(ROPE_POSITIONS, D)
    for dt in STORAGE_TYPES:
        tc, ts = rope_table_parts(ops.rope_table(ROPE_POSITIONS + 1, D, ROPE_THETA, "cpu", dt), dt)
        with pytest.raises(AssertionError, match="differs at position"):
            rope_table_mismatches(tc[1:], ts[1:], tc[:-1], ts[:-1], ang)


def test_rope_matcher_rejects_fp32_range_reduction():
    """cos / sin after reducing the angle modulo 2 pi in fp32 arithmetic (the reduction loses up to |angle| 2^-24 of
    absolute accuracy, up to 2^-9 at position 32767): wrong far from any rounding midpoint, in both storage types."""
    from videollama2_b200 import ops
    D = 128
    ang = rope_angles_fp32(ROPE_POSITIONS, D)
    two_pi = torch.tensor(2 * math.pi, dtype=torch.float32)
    red = ang - torch.round(ang / two_pi) * two_pi
    for dt in STORAGE_TYPES:
        rc, rs = _rope_fp64_table(red, dt)
        tc, ts = rope_table_parts(ops.rope_table(ROPE_POSITIONS, D, ROPE_THETA, "cpu", dt), dt)
        with pytest.raises(AssertionError, match="differs at position"):
            rope_table_mismatches(rc, rs, tc, ts, ang)


# ---------------------------------------------------------------------------------------------------------------------
# fp16: the bounds of the fp16 instances still reject what they must, and the overflow reference is torch's rounding
# ---------------------------------------------------------------------------------------------------------------------
def _f16_randn(shape, scale, seed):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale).to(torch.float16)


def test_fp16_checker_rejects_one_row_0p2_percent_off():
    """One row of an fp16 GEMM output 0.2 % off: relL2 under 1.5e-3, the bar of the relL2 fp16 GEMM tests, passes it;
    the fp16 element-wise bound (2^-11 of the value) does not."""
    M, N, K = 1100, 1024, 328
    a, w = _f16_randn((M, K), 1.0, 11), _f16_randn((N, K), 0.06, 12)
    ref = a.double() @ w.double().t()
    bound = storage_bound(ref, gemm_acc_bound(a, w), torch.float16)
    good = ref.float().to(torch.float16)
    assert check_elementwise(good, ref, bound, "correct") <= 1.0
    bad = good.clone()
    bad[517] = (bad[517].float() * 1.002).to(torch.float16)
    assert relerr(bad, ref) < 1.5e-3
    with pytest.raises(AssertionError, match=r"row 517"):
        check_elementwise(bad, ref, bound, "one row 0.2 % off")


def test_fp16_attention_bound_rejects_one_leaked_masked_key():
    """The fp16 attention bound, with its subnormal term 2^-25 sum |v|, on logit std 16 (most of P subnormal): it still
    rejects row 40 of head 1 also seeing key 41."""
    S, H, D = 512, 4, 64
    q, k, v = (_f16_randn((H, S, D), 4.0, s) for s in (13, 14, 15))
    q[1, 40] = k[1, 41] * 0.25                    # make the leaked key matter: a large logit against key 41
    scale = D ** -0.5
    ref, bound = attention_reference(q, k, v, True, scale, torch.float16)
    good = ref.float().to(torch.float16)
    assert check_elementwise(good, ref, bound, "correct", tile=(128, D)) <= 1.0
    s = (q[1, 40].double() @ k[1, :42].double().t()) * scale
    leaked = ref.clone()
    leaked[1, 40] = torch.softmax(s, -1) @ v[1, :42].double()
    bad = leaked.float().to(torch.float16)
    with pytest.raises(AssertionError, match=r"row 40"):
        check_elementwise(bad[1], ref[1], bound[1], "leaked key", tile=(128, D))


def test_fp16_overflow_reference():
    """to_storage_exact rounds like the fp16 store: 65504 stays, 65519.99 becomes 65504, 65520 and beyond +-inf, the
    subnormals 2^-24 and 2.5 2^-24 (a tie: to even, 2 2^-24) are kept and rounded, 2^-25 (a tie) goes to zero."""
    x = torch.tensor([FP16_MAX, 65519.9921875, 65520.0, -65520.0, 1e6, -FP16_MAX, -65519.0,
                      2.0 ** -24, 2.5 * 2.0 ** -24, 2.0 ** -25], dtype=torch.float64)
    got = to_storage_exact(x, torch.float16).double()
    want = torch.tensor([FP16_MAX, FP16_MAX, math.inf, -math.inf, math.inf, -FP16_MAX, -FP16_MAX,
                         2.0 ** -24, 2.0 * 2.0 ** -24, 0.0], dtype=torch.float64)
    assert torch.equal(got, want)


@pytest.mark.parametrize("dt", STORAGE_TYPES, ids=["bf16", "fp16"])
def test_allreduce_expectation_rejects_other_orders_and_roundings(dt):
    """On the probe rows of make_partials (every fourth row, columns 0 and 1), the expected all-reduce changes when the
    ranks are summed in reverse order or exactly (fp64) before the one rounding; anywhere, when every step is rounded
    to the storage type.  Statistics taken from the fp32 sum before its rounding are rejected, those of the rounded
    sum accepted."""
    import numpy as np
    p = make_partials(3, 16, 64, dt, seed=7)
    want = expected_sum(p, dt)

    def differ(a, b):
        return int((a.view(np.uint32) != b.view(np.uint32)).sum())
    assert differ(expected_sum(p[::-1], dt)[0::4, :2], want[0::4, :2]) > 0
    with np.errstate(invalid="ignore", over="ignore"):
        exact = to_storage(p.astype(np.float64).sum(0).astype(np.float32), dt)
        step = np.zeros(p.shape[1:], np.float32)
        acc = np.zeros(p.shape[1:], np.float32)
        for q in p:
            step = to_storage(step + q, dt)
            acc += q
        unrounded_stats = (acc.astype(np.float64) ** 2).sum(1).astype(np.float32)
    assert differ(exact[0::4, :2], want[0::4, :2]) > 0
    assert differ(step, want) > 0
    good = (want.astype(np.float64) ** 2).sum(1).astype(np.float32)
    assert stats_violations(good, want).size == 0
    assert stats_violations(unrounded_stats, want).size > 0

"""Host side of the device sampler (vl2_sample_token): the numpy Philox4x32-10 the GPU tests predict the kernel's draws
with, the host statement of the kernel's rule against HF's warpers, the C-ABI's argument checks and the parameter block's
validation.  No GPU needed."""
import ctypes
import math

import numpy as np
import pytest
import torch

from videollama2_b200 import sampling


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(counter, key, want):
    """Random123's published known-answer vectors for Philox4x32-10."""
    assert sampling.philox4x32_10(counter, key) == want


def test_kernel_u_uses_counter_and_seed_words():
    x0 = sampling.philox4x32_10((7, 1, 0, 0), (0x89abcdef, 0x01234567))[0]
    assert sampling.kernel_u(0x0123456789abcdef, (1 << 32) + 7) == (x0 >> 8) * 2.0 ** -24
    assert 0.0 <= sampling.kernel_u(3, 4) < 1.0


def _mass_above_margin(logits, T, k, p):
    """Distance of every kept-by-top-k token's fp64 mass-above from top_p (the HF fp32 cumsum and the kernel may only
    disagree inside it)."""
    s = (logits / T).double().numpy()
    keep = np.ones_like(s, dtype=bool) if not 0 < k < s.size else s >= np.sort(s)[s.size - k]
    w = np.where(keep, np.exp(s - s.max()), 0.0)
    order = np.argsort(-s)
    above = np.concatenate([[0.0], np.cumsum(w[order])[:-1]]) / w.sum()
    return np.abs(above[keep[order]] - p).min()


@pytest.mark.parametrize("V", [7, 300, 5000])
def test_kernel_rule_matches_warp_logits_on_tie_free_rows(V):
    """On rows without ties the kernel's kept set is the set warp_logits leaves finite, and its index-order CDF ends at the
    kept tokens' softmax."""
    g = torch.Generator().manual_seed(V)
    checked = 0
    for T in (0.2, 0.7, 1.0, 1.5):
        for k in (0, 1, 50, V):
            for p in (0.01, 0.5, 0.9, 1.0):
                for _ in range(20):
                    logits = torch.randn(V, generator=g) * 3.0
                    if torch.unique(logits / T).numel() == V and (p >= 1.0 or _mass_above_margin(logits, T, k, p) > 1e-5):
                        break
                else:
                    pytest.fail("no tie-free row with a top-p margin")
                hf = sampling.warp_logits(logits[None], T, k, p)[0]
                keep, _ = sampling.kernel_kept(logits, T, k, p)
                assert np.array_equal(keep, torch.isfinite(hf).numpy()), (T, k, p)
                cdf = sampling.kernel_cdf(logits, T, k, p)
                probs = hf.double().softmax(-1).numpy()
                assert np.allclose(np.diff(np.concatenate([[0.0], cdf])), probs, atol=1e-6)
                checked += 1
    assert checked == 64


def test_kernel_token_is_the_inverse_cdf():
    logits = torch.tensor([0.0, 1.0, 2.0, -math.inf, 0.5])
    cdf = sampling.kernel_cdf(logits)
    for n in range(64):
        u = sampling.kernel_u(11, n)
        tok = sampling.kernel_token(logits, 1.0, 0, 1.0, 11, n)
        assert tok != 3 and cdf[tok] > u and (tok == 0 or cdf[tok - 1] <= u)


def test_kernel_rule_keeps_tie_groups_whole():
    logits = torch.tensor([2.0, 1.0, 1.0, 1.0, 0.0])
    p0 = math.exp(2.0) / float(torch.exp(logits.double()).sum())
    assert sampling.kernel_kept(logits, 1.0, 0, p0 + 1e-3)[0].tolist() == [True, True, True, True, False]
    assert sampling.kernel_kept(logits, 1.0, 0, p0 - 1e-3)[0].tolist() == [True, False, False, False, False]
    assert sampling.kernel_kept(torch.tensor([3.0, 3.0, 1.0]), 1.0, 1, 1.0)[0].tolist() == [True, True, False]


@pytest.fixture(scope="module")
def lib():
    from videollama2_b200 import _lib, build
    build.build()
    return _lib.load()


A16, MIS = 4096, 4100          # fake device addresses: aligned, and 4 bytes off (never dereferenced)


@pytest.mark.parametrize("args,code", [
    ((A16, 0, A16, A16, 0, A16, None), -1),
    ((A16, -5, A16, A16, 0, A16, None), -1),
    ((A16, 262145, A16, A16, 0, A16, None), -1),
    ((None, 32000, A16, A16, 0, A16, None), -3),
    ((A16, 32000, None, A16, 0, A16, None), -3),
    ((A16, 32000, A16, None, 0, A16, None), -3),
    ((A16, 32000, A16, A16, 0, None, None), -3),
    ((A16 + 2, 32000, A16, A16, 0, A16, None), -3),
    ((A16, 32000, MIS, A16, 0, A16, None), -3),
    ((A16, 32000, A16, MIS, 0, A16, None), -3),
    ((A16, 32000, A16, A16, 0, MIS, None), -3),
])
def test_sample_token_argument_validation_without_gpu(lib, args, code):
    """V and the pointers are checked before any CUDA call: VL2_E_BADSHAPE outside 1..262144, VL2_E_BADALIGN for null or
    misaligned pointers."""
    assert lib.vl2_sample_token(*args) == code, lib.vl2_last_error()


def test_sampling_params_layout_and_validation():
    from videollama2_b200 import _lib, ops
    assert ctypes.sizeof(_lib.SampleParams) == 24
    p = ops.sampling_params(0.2, 50, 0.9, 2 ** 63 - 5, "cpu")
    assert p.dtype == torch.int64 and p.shape == (3,)
    raw = _lib.SampleParams.from_buffer_copy(p.numpy().tobytes())
    assert (raw.temperature, raw.top_k, raw.seed) == (np.float32(0.2), 50, 2 ** 63 - 5)
    assert raw.top_p == np.float32(0.9)
    for t in (0.0, -1.0, math.nan, math.inf):
        with pytest.raises(ValueError):
            ops.sampling_params(t, 50, 0.9, 1, "cpu")
    for tp in (0.0, -0.1, 1.5, math.nan):
        with pytest.raises(ValueError):
            ops.sampling_params(1.0, 50, tp, 1, "cpu")
    with pytest.raises(ValueError):
        ops.sampling_params(1.0, -1, 0.9, 1, "cpu")
    ops.sampling_params(1.0, 0, 1.0, 0, "cpu")            # top-k and top-p off

"""The device sampler (vl2_sample_token) token by token against the host statement of its rule (sampling.kernel_kept: HF's
warpers with the documented tie rule, fp64 softmax, index-order inverse CDF, Philox4x32-10 in Python), and
generate(do_sample=True) through every decode path on the tiny configurations."""

import numpy as np
import pytest
import torch

from helpers import build_engine

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16]
# The kernel's weights are exact to 2^-41 of the maximum's (fixed point) and expf to 2 ulp, so its CDF boundaries and
# masses lie within ~3e-7 of the fp64 ones.  Top-p inputs keep every token's fp64 mass-above MARGIN away from top_p (a
# full-vocabulary row has its masses ~1e-5 apart, so a 1e-5 margin would leave no such row); draws within U_MARGIN of a
# boundary of the host CDF may land on either side of it.
MARGIN = 1e-6
U_MARGIN = 1e-6


def philox_u(seed: int, n: np.ndarray) -> np.ndarray:
    """sampling.kernel_u vectorised over counters (uint64 numpy arithmetic)."""
    m = np.uint64(0xFFFFFFFF)
    c0, c1 = n.astype(np.uint64) & m, n.astype(np.uint64) >> np.uint64(32)
    c2, c3 = np.zeros_like(c0), np.zeros_like(c0)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m, (k1 + np.uint64(0xBB67AE85)) & m
    return (c0 >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def draw(logits, T, k, p, seed, n_draws, dtype=torch.bfloat16, counter0=0, add0=0):
    """n_draws tokens with counters counter0 + add0 + j, each its own launch writing out[j]."""
    from videollama2_b200 import _lib, ops
    dev = logits.device
    params = ops.sampling_params(T, k, p, seed, dev)
    counter = torch.full((1,), counter0, dtype=torch.int64, device=dev)
    out = torch.full((n_draws,), -1, dtype=torch.int64, device=dev)
    lib, st = _lib.load(dtype), torch.cuda.current_stream().cuda_stream
    row = logits.contiguous()
    for j in range(n_draws):
        _lib.check(lib.vl2_sample_token(row.data_ptr(), row.numel(), params.data_ptr(), counter.data_ptr(), add0 + j,
                                        out.data_ptr() + 8 * j, st), "vl2_sample_token", lib)
    return out.cpu().numpy()


def predicted(logits, T, k, p, seed, n):
    """(predicted tokens, which draws lie within U_MARGIN of a boundary, the kept tokens next to each prediction, the
    fraction of draws expected that close: 2 * U_MARGIN per kept token)."""
    from videollama2_b200 import sampling
    cdf = sampling.kernel_cdf(logits.cpu(), T, k, p)
    u = philox_u(seed, np.arange(n))
    tok = np.minimum(np.searchsorted(cdf, u, side="right"), cdf.size - 1)
    kept = np.nonzero(np.diff(np.concatenate([[0.0], cdf])) > 0)[0]
    pos = np.searchsorted(kept, tok)
    lo = np.where(pos > 0, cdf[kept[np.maximum(pos - 1, 0)]], 0.0)    # cdf[previous kept] <= u < cdf[tok]
    near = np.minimum(np.abs(u - lo), np.abs(cdf[tok] - u)) <= U_MARGIN
    neighbours = np.stack([kept[np.maximum(pos - 1, 0)], tok, kept[np.minimum(pos + 1, kept.size - 1)]], 1)
    return tok, near, neighbours, 2 * U_MARGIN * kept.size


def mass_margin(logits, T, k, p):
    s = (logits.cpu() / T).double().numpy()
    keep = np.ones_like(s, dtype=bool) if not 0 < k < s.size else s >= np.sort(s)[s.size - k]
    w = np.where(keep, np.exp(s - s.max()), 0.0)
    vals, inv = np.unique(s, return_inverse=True)
    group = np.bincount(inv, weights=w, minlength=vals.size)
    above = np.concatenate([np.cumsum(group[::-1])[::-1][1:], [0.0]])[inv] / w.sum()
    return np.abs(above[keep] - p).min()


def _cases():
    Ts, ks, ps, sigmas = [0.2, 0.7, 1.0, 1.5], [0, 1, 50, 1000, "V"], [0.01, 0.5, 0.9, 0.95, 1.0], [1.0, 3.0, 8.0]
    i = 0
    for V in (7, 1000, 32000, 152064):
        for k in ks:
            for p in ps:
                yield V, Ts[i % 4], (V if k == "V" else k), p, sigmas[(i // 4) % 3]
                i += 1


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
def test_tokens_match_host_prediction(cuda, dt):
    """4096 counters per case over V x top_k x top_p, temperature and sigma cycling through their values: every draw
    farther than U_MARGIN from a boundary of the host CDF returns the predicted token, and one closer returns a kept
    neighbour of it.  Close draws are counted: under 1 %, or where the kept set is so dense that the boundaries alone
    cover more, under 3 x the fraction its density predicts.  A wrongly kept or dropped token would shift every later
    boundary by its mass and show up as wrong tokens."""
    n = 4096
    rng = np.random.default_rng(0)
    for case, (V, T, k, p, sigma) in enumerate(_cases()):
        for _ in range(50):
            logits = torch.from_numpy(rng.normal(0.0, sigma, V).astype(np.float32))
            if p >= 1.0 or mass_margin(logits, T, k, p) > MARGIN:
                break
        else:
            pytest.fail(f"no row with a top-p margin for {(V, T, k, p, sigma)}")
        assert p >= 1.0 or mass_margin(logits, T, k, p) > MARGIN
        seed = 1000 + case
        got = draw(logits.to(cuda), T, k, p, seed, n, dt)
        want, near, neighbours, dense = predicted(logits, T, k, p, seed, n)
        assert near.mean() < max(0.01, 3 * dense), (V, T, k, p, sigma, near.mean(), dense)
        bad = (got != want) & ~near
        assert not bad.any(), (V, T, k, p, sigma, int(bad.sum()), got[bad][:5], want[bad][:5])
        assert (neighbours == got[:, None]).any(1).all(), (V, T, k, p, sigma)


def test_distribution_chi_square(cuda):
    """20 000 draws from one row with 50 kept tokens follow warp_logits' softmax (chi-square p > 1e-4)."""
    from scipy.stats import chisquare
    from videollama2_b200 import sampling
    logits = torch.randn(32000, generator=torch.Generator().manual_seed(3)) * 2.0
    probs = sampling.warp_logits(logits[None], 1.0, 50, 1.0)[0].double().softmax(-1).numpy()
    got = draw(logits.to(cuda), 1.0, 50, 1.0, 77, 20000)
    kept = np.nonzero(probs > 0)[0]
    assert kept.size == 50 and np.isin(got, kept).all()
    obs = np.array([(got == t).sum() for t in kept], dtype=np.float64)
    assert chisquare(obs, probs[kept] * obs.sum()).pvalue > 1e-4


def test_edges(cuda):
    dev = cuda
    t = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)
    # ties at the top-k boundary are all reachable, and with k = 1 the ties at the maximum
    assert set(draw(t([2.0, 2.0, 1.9, 1.9, 1.9, 0.0, 0.0, 0.0]), 1.0, 3, 1.0, 1, 2048)) == {0, 1, 2, 3, 4}
    assert set(draw(t([3.0, 0.0, 3.0, 1.0, 3.0]), 1.0, 1, 1.0, 2, 1024)) == {0, 2, 4}
    # a tie group at the top-p boundary is kept or dropped whole
    row = [2.0, 1.0, 1.0, 1.0, 0.0, 0.0]
    p0 = float(np.exp(2.0) / np.exp(np.array(row)).sum())
    assert set(draw(t(row), 1.0, 0, p0 + 1e-3, 3, 2048)) == {0, 1, 2, 3}
    assert set(draw(t(row), 1.0, 0, p0 - 1e-3, 4, 256)) == {0}
    # -inf logits are never drawn, also when t_k itself is -inf
    inf = float("-inf")
    assert set(draw(t([inf, 0.5, inf, 0.0, inf, 0.2, inf]), 1.0, 5, 1.0, 5, 2048)) == {1, 3, 5}
    big = torch.full((32000,), inf, device=dev)
    big[[7, 19000, 31999]] = torch.tensor([0.0, 0.1, -0.1], device=dev)
    assert set(draw(big, 0.7, 50, 0.9, 6, 1024)) <= {7, 19000, 31999}
    # a single finite logit always returns its index
    one = torch.full((152064,), inf, device=dev)
    one[123456] = -3.0
    assert set(draw(one, 1.5, 0, 0.5, 7, 64)) == {123456}
    # top_k = 1 is the arg-max on rows without ties
    for s in range(8):
        row = torch.randn(32000, generator=torch.Generator().manual_seed(s)).to(dev)
        assert set(draw(row, 0.7, 1, 0.9, s, 16)) == {int(torch.argmax(row))}
    # weights that underflow to zero at a small temperature leave the arg-max
    assert set(draw(t([0.0, 1.0, 2.0, 3.0, 2.5]), 1e-3, 0, 1.0, 8, 256)) == {3}


def test_determinism_and_counter(cuda):
    """Same inputs -> same tokens; the bf16 and fp16 builds agree; the kernel reads *counter_dev + counter_add."""
    row = (torch.randn(152064, generator=torch.Generator().manual_seed(9)) * 3.0).to(cuda)
    a = draw(row, 1.0, 0, 0.95, 42, 512)
    assert np.array_equal(a, draw(row, 1.0, 0, 0.95, 42, 512))
    assert np.array_equal(a, draw(row, 1.0, 0, 0.95, 42, 512, torch.float16))
    assert np.array_equal(draw(row, 0.7, 50, 0.9, 5, 64, counter0=5, add0=0), draw(row, 0.7, 50, 0.9, 5, 64, add0=5))


# ---- generate(do_sample=True) ---------------------------------------------------------------------------------------
GEN_CFGS = [("tiny", torch.bfloat16), ("tiny_qwen2", torch.bfloat16), ("tiny", torch.float16)]


@pytest.fixture(scope="module", params=GEN_CFGS, ids=["tiny", "tiny_qwen2", "tiny-fp16"])
def gen(request, cuda):
    from oracle import synth
    from helpers import engine_config
    from videollama2_b200.model import VLLMs
    name, dt = request.param
    cfg = synth.CONFIGS[name]
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    if dt == torch.bfloat16:
        model = build_engine(cfg, sd, cuda)
    else:
        ec = engine_config(cfg)
        model = VLLMs[ec.model_type].from_state_dict(ec, sd, device=cuda, dtype=dt)
    return model, ids, [(px.to(cuda).to(dt), "video")]


KW = dict(do_sample=True, temperature=1.5, top_p=0.95, top_k=50, eos_token_id=None)


def _g(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def host_prediction(model, ids, imgs, n_new, seed_gen, T, k, p):
    """Sample the eager loop's own logits with the host rule and Philox, token by token."""
    from videollama2_b200 import sampling
    from videollama2_b200.sampling import draw_seed
    seed = draw_seed(seed_gen)
    dec = model.get_model().decoder
    _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, None, None, None, imgs)
    x = emb[0].to(dec.dtype).contiguous()
    logits, _ = dec.prefill(x, all_logits=False, keep_cache=True, max_len=x.shape[0] + n_new)
    toks = []
    for n in range(n_new):
        toks.append(sampling.kernel_token(logits[0].cpu(), T, k, p, seed, n))
        if n + 1 < n_new:
            logits = dec.decode_step(model.get_model().embed_tokens(torch.tensor([toks[-1]])).to(dec.dtype))
    return toks


def test_generate_sampled_graphed_equals_eager_and_host(gen, cuda):
    model, ids, imgs = gen
    dec = model.get_model().decoder
    eager = model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda), **KW)
    assert eager.shape == (1, 7)
    assert eager[0].tolist() == host_prediction(model, ids, imgs, 7, _g(3, cuda), 1.5, 50, 0.95)
    nocache = model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda), use_cache=False, **KW)
    assert torch.equal(nocache, eager)
    model.enable_cuda_graphs(True)
    try:
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda), **KW), eager)
        graph = dec._decode_graph_sampled
        assert graph is not None
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda), **KW), eager)
        assert dec._decode_graph_sampled is graph                       # the captured sampled graph is reused
        other = model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda),
                               **{**KW, "temperature": 0.2, "top_p": 0.9})
        assert dec._decode_graph_sampled is graph                       # new parameters, same graph
        model.enable_cuda_graphs(False)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=7, generator=_g(3, cuda),
                                          **{**KW, "temperature": 0.2, "top_p": 0.9}), other)
    finally:
        model.enable_cuda_graphs(False)


def test_generate_sampled_stopping_and_mixing(gen, cuda):
    model, ids, imgs = gen
    dec = model.get_model().decoder
    eager = model.generate(ids, images=imgs, max_new_tokens=9, generator=_g(5, cuda), **KW)
    greedy = model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None)
    stop = [lambda out_ids, _s: out_ids.shape[1] >= 4]
    eager_stop = model.generate(ids, images=imgs, max_new_tokens=9, generator=_g(5, cuda), stopping_criteria=stop, **KW)
    assert torch.equal(eager_stop, eager[:, :4])
    model.enable_cuda_graphs(True)
    try:
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, generator=_g(5, cuda),
                                          stopping_criteria=stop, **KW), eager_stop)
        # greedy after sampled and sampled after greedy: neither graph disturbs the other
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None), greedy)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, generator=_g(5, cuda), **KW), eager)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None), greedy)
        # a longer generation reallocates the KV cache: the sampled graph is captured again on the new cache
        old = dec._decode_graph_sampled
        cap = dec.kv[0].shape[0]
        longer = model.generate(ids, images=imgs, max_new_tokens=cap + 1, generator=_g(5, cuda), **KW)
        assert dec.kv[0].shape[0] > cap and dec._decode_graph_sampled is not old
        assert torch.equal(longer[:, :9], eager)
    finally:
        model.enable_cuda_graphs(False)


def test_generate_sampled_reproducible_and_batched(gen, cuda):
    model, ids, imgs = gen
    torch.manual_seed(11)
    a = model.generate(ids, images=imgs, max_new_tokens=5, **KW)
    torch.manual_seed(11)
    assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=5, **KW), a)
    # a batch of two rows draws one seed per row, in row order, from the one generator
    both = torch.cat([ids, ids], 0)
    b1 = model.generate(both, images=imgs + imgs, max_new_tokens=5, generator=_g(8, cuda), **KW)
    b2 = model.generate(both, images=imgs + imgs, max_new_tokens=5, generator=_g(8, cuda), **KW)
    assert b1.shape == (2, 5) and torch.equal(b1, b2)
    g = _g(8, cuda)
    r0 = model.generate(ids, images=imgs, max_new_tokens=5, generator=g, **KW)
    r1 = model.generate(ids, images=imgs, max_new_tokens=5, generator=g, **KW)
    assert torch.equal(b1, torch.cat([r0, r1], 0))

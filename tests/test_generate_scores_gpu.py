"""generate(output_scores / output_logits) on the device: the row recorder (vl2_record_row), the scored sampler
(vl2_sample_token_scored) against the host statement sampling.expected_scores, and generate() on every decode path of
the tiny configurations, on both library builds."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import build_engine

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16]
NEG_INF = float("-inf")


def bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


# ---- recorder ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("V", [7, 1000, 32000, 152064])
def test_record_rows_land_in_their_slot(cuda, dt, V):
    """Row r lands bit for bit in slot *step + add of the chosen buffer only; slots outside [0, capacity) write nothing;
    guard rows around each buffer stay untouched."""
    from videollama2_b200 import _lib, ops
    cap, g = 5, torch.Generator().manual_seed(V)
    arena = {w: torch.full((cap + 2, V), 7.0, device=cuda) for w in ("scores", "logits")}      # guard row each side
    bufs = {w: a[1:cap + 1] for w, a in arena.items()}
    blk = ops.score_record_params(V, cap, bufs["scores"], bufs["logits"])
    step = torch.tensor([2], dtype=torch.int64, device=cuda)
    want = {w: torch.full((cap + 2, V), 7.0) for w in arena}
    for add, which in [(-2, _lib.RECORD_LOGITS), (0, _lib.RECORD_SCORES), (2, _lib.RECORD_LOGITS), (-3, _lib.RECORD_SCORES),
                       (3, _lib.RECORD_SCORES), (9, _lib.RECORD_LOGITS), (-1, _lib.RECORD_SCORES)]:
        row = torch.randn(V, generator=g)
        row[::17] = -0.0
        ops.record_rows(row.to(cuda), blk, which, step, add, dt)
        slot = 2 + add
        if 0 <= slot < cap:
            want["scores" if which == _lib.RECORD_SCORES else "logits"][1 + slot] = row
    torch.cuda.synchronize()
    for w in arena:
        assert torch.equal(bits(arena[w]), bits(want[w])), w
    # a block without a buffer, or of another V, writes nothing
    empty = ops.score_record_params(V, cap, None, bufs["logits"], cuda)
    ops.record_rows(torch.zeros(V, device=cuda), empty, _lib.RECORD_SCORES, step, 0, dt)
    if V > 1:
        other = ops.score_record_params(V - 1, cap, torch.zeros((cap, V - 1), device=cuda), None)
        ops.record_rows(torch.zeros(V, device=cuda), other, _lib.RECORD_SCORES, step, 0, dt)
    assert torch.equal(bits(arena["scores"]), bits(want["scores"]))


def test_one_graph_records_into_two_buffers(cuda):
    """A captured graph reads its destination from the block: copying in a second block redirects it."""
    from videollama2_b200 import _lib, ops
    V, cap = 32000, 3
    row = torch.randn(V, device=cuda)
    step = torch.zeros((1,), dtype=torch.int64, device=cuda)
    fixed = torch.zeros((ops.SCORE_RECORD_WORDS,), dtype=torch.int64, device=cuda)
    a, b = torch.zeros((cap, V), device=cuda), torch.zeros((cap, V), device=cuda)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.record_rows(row, fixed, _lib.RECORD_LOGITS, step, 1, torch.bfloat16)       # warm-up: null block, no write
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.record_rows(row, fixed, _lib.RECORD_LOGITS, step, 1, torch.bfloat16)
        step.add_(1)
    fixed.copy_(ops.score_record_params(V, cap, None, a))
    graph.replay()
    graph.replay()
    fixed.copy_(ops.score_record_params(V, cap, None, b))
    step.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(a[1], row) and torch.equal(a[2], row) and not a[0].any()
    assert torch.equal(b[1], row) and not b[0].any() and not b[2].any()


# ---- scored sampler ---------------------------------------------------------------------------------------------------
MARGIN = 1e-6      # top-p rows keep every token's fp64 mass-above this far from top_p (test_sampling_gpu.py's reasoning)


def mass_margin(logits, T, k, p):
    s = (logits.cpu() / T).double().numpy()
    keep = np.ones_like(s, dtype=bool) if not 0 < k < s.size else s >= np.sort(s)[s.size - k]
    w = np.where(keep, np.exp(s - s.max()), 0.0)
    vals, inv = np.unique(s, return_inverse=True)
    group = np.bincount(inv, weights=w, minlength=vals.size)
    above = np.concatenate([np.cumsum(group[::-1])[::-1][1:], [0.0]])[inv] / w.sum()
    return np.abs(above[keep] - p).min()


SETTINGS = [(1.0, 0, 1.0), (0.7, 50, 0.9), (1.5, 0, 0.95), (0.3, 1000, 0.5), (1.0, 1, 0.9)]


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("V", [7, 1000, 32000, 152064])
def test_scored_sampler_row_and_tokens(cuda, dt, V):
    """The warped row equals expected_scores bit for bit (both the shared-memory and the L2 instantiation), in the slot
    of every counter; over 4096 counters the token equals vl2_sample_token's."""
    from videollama2_b200 import ops, sampling
    n = 4096
    rng = np.random.default_rng(V)
    for T, k, p in SETTINGS:
        for _ in range(50):
            # a wide spread at large V, where a narrow one leaves no top-p boundary 1e-6 away from every token's mass
            row = torch.from_numpy(rng.normal(0.0, 3.0 if V < 32000 else 8.0, V).astype(np.float32))
            row[rng.integers(0, V, max(1, V // 50))] = -0.0
            if p >= 1.0 or mass_margin(row, T, k, p) > MARGIN:
                break
        else:
            pytest.fail(f"no row with a top-p margin for {(V, T, k, p)}")
        want = sampling.expected_scores(row, [], do_sample=True, temperature=T, top_k=k, top_p=p)
        cap = n if V <= 32000 else 4                       # 4 rows of 608 KB suffice to check the slot rule at Qwen2's V
        buf = torch.full((cap, V), 5.0, device=cuda)
        blk = ops.score_record_params(V, cap, buf, None)
        params = ops.sampling_params(T, k, p, 1000 + V, cuda)
        counter = torch.zeros((1,), dtype=torch.int64, device=cuda)
        plain = torch.empty((n,), dtype=torch.int64, device=cuda)
        scored = torch.empty((n,), dtype=torch.int64, device=cuda)
        lg = row.to(cuda)
        for j in range(n):
            ops.sample_token(lg, params, counter, j, plain[j:j + 1], dt)
            ops.sample_token(lg, params, counter, j, scored[j:j + 1], dt, record=blk)
        assert torch.equal(plain, scored), (V, T, k, p)
        got = bits(buf)
        assert torch.equal(got[0], bits(want)), (V, T, k, p)
        assert (got == got[0]).all(), (V, T, k, p)
        assert torch.isfinite(want[plain.cpu()]).all()       # every drawn token is kept in the row


# ---- generate() -------------------------------------------------------------------------------------------------------
GEN_CFGS = [("tiny", torch.bfloat16), ("tiny_qwen2", torch.bfloat16), ("tiny", torch.float16)]


@pytest.fixture(scope="module", params=GEN_CFGS, ids=["tiny", "tiny_qwen2", "tiny-fp16"])
def gen(request, cuda):
    from helpers import engine_config
    from oracle import synth
    from videollama2_b200.model import VLLMs
    name, dt = request.param
    cfg = synth.CONFIGS[name]
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    if dt == torch.bfloat16:
        model = build_engine(cfg, sd, cuda)
    else:
        model = VLLMs[engine_config(cfg).model_type].from_state_dict(engine_config(cfg), sd, device=cuda, dtype=dt)
    return model, ids, [(px.to(cuda).to(dt), "video")]


SAMPLED = dict(do_sample=True, temperature=1.5, top_p=0.95, top_k=50)
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, suppress_tokens=[3, 5])
MODES = {"greedy": {}, "greedy+proc": PROC, "sampled": SAMPLED, "sampled+proc": {**SAMPLED, **PROC}}
REC = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)


def _run(model, ids, imgs, mode, path, max_new=9, **extra):
    kw = {**MODES[mode], "max_new_tokens": max_new, "eos_token_id": None, **extra}
    if "do_sample" in kw:
        kw["generator"] = torch.Generator(device=model.device).manual_seed(4)
    model.enable_cuda_graphs(path == "graphed")
    try:
        return model.generate(ids, images=imgs, use_cache=path != "nocache", **kw)
    finally:
        model.enable_cuda_graphs(False)


def check_rows(out, mode):
    """Each scores[n] is the host statement of logits[n] after the ids before n (sampled: where the top-p boundary has
    no near tie)."""
    from videollama2_b200 import sampling
    seq = out.sequences[0].tolist()
    kw = MODES[mode]
    proc = {k: kw[k] for k in PROC if k in kw}
    checked = 0
    for n in range(len(seq)):
        raw = out.logits[n][0].cpu()
        if kw.get("do_sample"):
            pr = sampling.process_logits(raw, seq[:n], **proc)
            if mass_margin(pr, kw["temperature"], kw["top_k"], kw["top_p"]) <= MARGIN:
                continue
        want = sampling.expected_scores(raw, seq[:n], do_sample=bool(kw.get("do_sample")),
                                        temperature=kw.get("temperature", 1.0), top_k=kw.get("top_k", 0),
                                        top_p=kw.get("top_p", 1.0), **proc)
        assert torch.equal(bits(out.scores[n][0]), bits(want)), (mode, n)
        assert torch.isfinite(want[seq[n]])
        checked += 1
    assert checked >= len(seq) - 1


@pytest.mark.parametrize("mode", list(MODES))
def test_generate_records_on_every_path(gen, mode):
    model, ids, imgs = gen
    V = model.vocab_size
    plain = {p: _run(model, ids, imgs, mode, p) for p in ("eager", "nocache", "graphed")}
    assert torch.equal(plain["eager"], plain["graphed"]) and torch.equal(plain["eager"], plain["nocache"])
    outs = {}
    for p in ("eager", "nocache", "graphed"):
        out = outs[p] = _run(model, ids, imgs, mode, p, **REC)
        assert torch.equal(out.sequences, plain[p]), (mode, p)            # recording changes no token
        assert out["sequences"] is out.sequences and out.attentions is None and out.past_key_values is None
        assert len(out.scores) == len(out.logits) == out.sequences.shape[1]
        assert all(t.shape == (1, V) and t.dtype == torch.float32 and t.is_cuda for t in out.scores + out.logits)
        check_rows(out, mode)
    for a, b in zip(outs["graphed"].scores + outs["graphed"].logits, outs["eager"].scores + outs["eager"].logits):
        assert torch.equal(bits(a), bits(b)), mode
    # again through the already captured recording graph, with new buffers; and one output only
    again = _run(model, ids, imgs, mode, "graphed", **REC)
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(again.scores, outs["eager"].scores))
    only = _run(model, ids, imgs, mode, "graphed", return_dict_in_generate=True, output_logits=True)
    assert only.scores is None and all(torch.equal(bits(a), bits(b)) for a, b in zip(only.logits, outs["eager"].logits))


def test_generate_return_value_shapes(gen):
    model, ids, imgs = gen
    V = model.vocab_size
    for p in ("eager", "graphed"):
        one = _run(model, ids, imgs, "greedy+proc", p, max_new=1, **REC)
        assert one.sequences.shape == (1, 1) and len(one.scores) == 1 and len(one.logits) == 1
        assert int(torch.argmax(one.scores[0])) == int(one.sequences[0, 0])
        # without return_dict_in_generate the flags are ignored: the bare id tensor, as before
        ids_only = _run(model, ids, imgs, "sampled", p, output_scores=True, output_logits=True)
        assert isinstance(ids_only, torch.Tensor) and torch.equal(ids_only, _run(model, ids, imgs, "sampled", p))
        none = _run(model, ids, imgs, "greedy", p, return_dict_in_generate=True)
        assert none.scores is None and none.logits is None and torch.equal(none.sequences, _run(model, ids, imgs, "greedy", p))
    # EOS stops early: only the rows of the returned ids are exposed
    full = _run(model, ids, imgs, "greedy", "graphed", max_new=12, **REC)
    eos = int(full.sequences[0, 3])
    stop = _run(model, ids, imgs, "greedy", "graphed", max_new=12, **{**REC, "eos_token_id": eos})
    n = stop.sequences.shape[1]
    assert n <= 4 and len(stop.scores) == n and all(torch.equal(a, b) for a, b in zip(stop.scores, full.scores))


def test_generate_batch_pads_scores(gen):
    """Rows are padded to the longest row; at the steps after a row stopped both outputs are -inf except 0.0 at
    pad_token_id, so compute_transition_scores gives 0 there."""
    model, ids, imgs = gen
    V, pad, max_new = model.vocab_size, 1, 8
    other = ids[:, :9].clone()                                # a second prompt, shorter, with its own text after <video>
    other[0, 5:] = (other[0, 5:] * 7 + 11) % (V - 3) + 3
    seqs = [_run(model, r, imgs, "greedy", "eager", max_new=max_new)[0].tolist() for r in (ids, other)]
    # an EOS that ends one row early and never appears in the other: the rows get different lengths
    eos = next((t for a, b in (seqs, seqs[::-1]) for i, t in enumerate(a[:-1]) if t not in a[:i] and t not in b), None)
    assert eos is not None, seqs
    both = torch.zeros((2, ids.shape[1]), dtype=ids.dtype)
    both[0], both[1, :other.shape[1]] = ids[0], other[0]
    mask = torch.zeros_like(both, dtype=torch.bool)
    mask[0], mask[1, :other.shape[1]] = True, True
    kw = dict(REC, eos_token_id=eos, pad_token_id=pad)
    out = _run(model, both, imgs + imgs, "greedy", "eager", max_new=max_new, attention_mask=mask, **kw)
    rows = [_run(model, r, imgs, "greedy", "eager", max_new=max_new, **kw) for r in (ids, other)]
    lens = [r.sequences.shape[1] for r in rows]
    n = out.sequences.shape[1]
    assert lens[0] != lens[1] and n == max(lens) and len(out.scores) == len(out.logits) == n
    filler = torch.full((V,), NEG_INF)
    filler[pad] = 0.0
    for b, r in enumerate(rows):
        assert torch.equal(out.sequences[b, :lens[b]], r.sequences[0]) and (out.sequences[b, lens[b]:] == pad).all()
        for t in range(n):
            for got, mine in ((out.scores, r.scores), (out.logits, r.logits)):
                assert got[t].shape == (2, V)
                want = mine[t][0] if t < lens[b] else filler
                assert torch.equal(bits(got[t][b]), bits(want)), (b, t)
    ts = model.compute_transition_scores(out.sequences, out.scores)
    for b, r in enumerate(rows):
        m = lens[b]
        assert (ts[b, m:] == 0).all()
        assert torch.equal(ts[b, :m].cpu(), torch.stack([r.scores[t][0, r.sequences[0, t]] for t in range(m)]).cpu())


def test_no_score_buffer_without_request(gen):
    """A call that asks for no scores allocates no [max_new, V] buffer."""
    model, ids, imgs = gen
    V, max_new = model.vocab_size, 1024

    def peak(**kw):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _run(model, ids, imgs, "greedy", "eager", max_new=max_new, stopping_criteria=[lambda o, _s: o.shape[1] >= 3], **kw)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    peak()                                      # first call: the KV cache and workspaces the engine keeps
    plain = peak()
    assert peak(output_scores=True, output_logits=True) == plain
    assert peak(return_dict_in_generate=True) == plain
    assert peak(return_dict_in_generate=True, output_scores=True) >= max_new * V * 4


# ---- tensor parallel --------------------------------------------------------------------------------------------------
def test_tp_ranks_return_identical_scores():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_tp_scores_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert all(f"RANK{i} OK" in r.stdout for i in range(world)), r.stdout[-2000:]

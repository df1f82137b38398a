"""The device logits processors (vl2_process_logits) against their host statement (sampling.process_logits) on both
builds, inside a captured graph, and generate() with processors through every decode path on the tiny configurations."""

import pytest
import torch

from helpers import build_engine

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16]


def same(a, b):
    """== with identical +-inf / NaN positions."""
    a, b = a.cpu(), b.cpu()
    return bool(torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.isposinf(a), torch.isposinf(b)) and
                torch.equal(torch.isneginf(a), torch.isneginf(b)) and (a[torch.isfinite(a)] == b[torch.isfinite(b)]).all())


def run_kernel(row, hist, dtype=torch.bfloat16, **proc):
    """vl2_process_logits on a copy of `row` with n split between *n_dev and n_add."""
    from videollama2_b200 import ops
    dev = row.device
    n = len(hist)
    h = torch.tensor(list(hist) + [0], dtype=torch.int64, device=dev)       # one spare id: never read
    params = ops.logits_process_params(row.numel(), dev, **proc)
    out = row.clone()
    ops.process_logits(out, params, h, torch.tensor([n // 2], dtype=torch.int64, device=dev), n - n // 2, dtype)
    return out


def _cases():
    for V in (7, 1000, 32000, 152064):
        for n in (0, 1, 5, 64, 2048):
            for i, pen in enumerate((0.8, 1.05, 1.3)):
                yield V, n, pen, 1 + (i + n) % 3


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
def test_kernel_equals_host_statement(cuda, dt):
    """Every listed V, history length (0 = the first step), penalty and n-gram size, with multi-token bad words whose
    prefixes match the history's tail, a minimum length on both sides of n, and suppressed tokens.  Histories repeat
    ids (a small id range, and a periodic stretch) so that repeats and n-gram matches occur."""
    from videollama2_b200 import sampling
    g = torch.Generator().manual_seed(0)
    for V, n, pen, N in _cases():
        row = torch.randn(V, generator=g) * 4.0
        row[torch.randint(0, V, (max(1, V // 50),), generator=g)] = -0.0
        hist = torch.randint(0, min(V, 40), (n,), generator=g).tolist()
        if n > 16:
            hist[n // 2:n // 2 + 12] = hist[:4] * 3
        tail = hist[-2:] if n >= 2 else [0, 1]
        proc = dict(repetition_penalty=pen, no_repeat_ngram_size=N, min_new_tokens=(n + 1) if N != 2 else n,
                    eos_token_ids=(V - 1, 0), suppress_tokens=[V // 2, 3 % V],
                    bad_words_ids=[[V - 2], tail + [V // 3], tail[-1:] + [V // 4], [1 % V, 2 % V, V - 3]])
        want = sampling.process_logits(row, hist, **proc)
        got = run_kernel(row.to(cuda), hist, dt, **proc)
        assert same(got, want), (V, n, pen, N)
        for single in (dict(repetition_penalty=pen), dict(no_repeat_ngram_size=N)):
            assert same(run_kernel(row.to(cuda), hist, dt, **single), sampling.process_logits(row, hist, **single))


def test_captured_graph_serves_every_setting(cuda):
    """One captured launch reads the block, the tables, the history and n from device memory: changing them between
    replays changes the result exactly as the host statement predicts."""
    from videollama2_b200 import ops, sampling
    V = 32000
    g = torch.Generator().manual_seed(1)
    row = torch.zeros(V, device=cuda)
    out = torch.zeros(V, device=cuda)
    hist = torch.zeros(4096, dtype=torch.int64, device=cuda)
    n_dev = torch.zeros(1, dtype=torch.int64, device=cuda)
    block = torch.zeros(ops.PROCESS_HEADER_WORDS, dtype=torch.int64, device=cuda)
    keep = ops.logits_process_params(V, cuda)
    block.copy_(keep[:ops.PROCESS_HEADER_WORDS])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out.copy_(row)
        ops.process_logits(out, block, hist, n_dev, 1)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out.copy_(row)
        ops.process_logits(out, block, hist, n_dev, 1)
    settings = [dict(repetition_penalty=1.3, no_repeat_ngram_size=2), dict(suppress_tokens=[5, 6, 7]),
                dict(repetition_penalty=0.8, bad_words_ids=[[9], [4, 4, 11]], min_new_tokens=2000, eos_token_ids=(2,)),
                dict(no_repeat_ngram_size=3, repetition_penalty=1.05), dict()]
    for i, proc in enumerate(settings):
        n = [0, 17, 700, 2048, 5][i]
        r = torch.randn(V, generator=g) * 3.0
        h = torch.randint(0, 30, (n + 1,), generator=g)
        row.copy_(r)
        hist[:n + 1].copy_(h)
        n_dev.fill_(n)                                  # the history is hist[0 .. n + 1)
        keep = ops.logits_process_params(V, cuda, **proc)
        block.copy_(keep[:ops.PROCESS_HEADER_WORDS])
        graph.replay()
        assert same(out, sampling.process_logits(r, h.tolist(), **proc)), proc


def test_every_token_banned(cuda):
    """A row whose every token is banned is all -inf: the arg-max and the sampling kernel both return token 0, the first
    index of the maximum."""
    from videollama2_b200 import ops
    for V in (7, 32000):
        row = torch.randn(V, device=cuda)
        got = run_kernel(row, [1, 2, 3], suppress_tokens=list(range(V)))
        assert torch.isneginf(got).all()
        assert int(torch.argmax(got)) == 0
        tok = torch.zeros(1, dtype=torch.int64, device=cuda)
        ops.sample_token(got, ops.sampling_params(1.0, 50, 0.9, 3, cuda), torch.zeros(1, dtype=torch.int64, device=cuda),
                         0, tok)
        assert int(tok) == 0


# ---- generate() with processors -------------------------------------------------------------------------------------
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


def _g(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def processors_for(model, ids, imgs, n):
    """Processors that bite on this model: bans built from its own greedy ids, EOS = its first greedy id."""
    plain = model.generate(ids, images=imgs, max_new_tokens=n, do_sample=False, eos_token_id=None)[0].tolist()
    return plain, dict(repetition_penalty=1.3, no_repeat_ngram_size=2, bad_words_ids=[[plain[2]], [plain[0], plain[1]]],
                       suppress_tokens=[plain[3]], min_new_tokens=5, eos_token_id=plain[0])


def host_greedy(model, ids, imgs, n_new, proc):
    """decode_step logits -> process_logits with the new ids so far -> arg-max, token by token."""
    from videollama2_b200 import sampling
    dec = model.get_model().decoder
    _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, None, None, None, imgs)
    x = emb[0].to(dec.dtype).contiguous()
    kw = {k: v for k, v in proc.items() if k != "eos_token_id"}
    logits, _ = dec.prefill(x, all_logits=False, keep_cache=True, max_len=x.shape[0] + n_new)
    toks = []
    for _ in range(n_new):
        row = sampling.process_logits(logits[0], toks, eos_token_ids=(proc["eos_token_id"],), **kw)
        toks.append(int(torch.argmax(row)))
        if toks[-1] == proc["eos_token_id"]:
            break
        logits = dec.decode_step(model.get_model().embed_tokens(torch.tensor([toks[-1]])).to(dec.dtype))
    return toks


def test_generate_processed_paths_agree(gen, cuda):
    """Greedy and sampled (fixed generator): the eager KV-cache loop, use_cache=False and the graphed loop return the
    same ids; greedy ids equal the host loop; the processed graphs are captured once and reused."""
    model, ids, imgs = gen
    dec = model.get_model().decoder
    plain, proc = processors_for(model, ids, imgs, 12)
    greedy = model.generate(ids, images=imgs, max_new_tokens=12, do_sample=False, **proc)
    assert greedy[0].tolist() == host_greedy(model, ids, imgs, 12, proc)
    banned = {plain[3]} | ({plain[2]} if plain[2] != plain[0] else set())    # a single-EOS bad word is dropped
    assert plain[0] not in greedy[0, :5].tolist() and not banned & set(greedy[0].tolist())
    skw = dict(do_sample=True, temperature=1.5, top_p=0.95, top_k=50, **proc)
    sampled = model.generate(ids, images=imgs, max_new_tokens=12, generator=_g(3, cuda), **skw)
    assert plain[0] not in sampled[0, :5].tolist() and not banned & set(sampled[0].tolist())
    assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=12, do_sample=False, use_cache=False, **proc), greedy)
    # use_cache=False recomputes every row with the prefill GEMM rather than the decode GEMV, so its logits are not the
    # same bits: compare its draws where the distribution is peaked (mm_infer's defaults), away from CDF boundaries
    peaked = dict(skw, temperature=0.2, top_p=0.9)
    assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=12, generator=_g(4, cuda), use_cache=False,
                                      **peaked),
                       model.generate(ids, images=imgs, max_new_tokens=12, generator=_g(4, cuda), **peaked))
    model.enable_cuda_graphs(True)
    try:
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=12, do_sample=False, **proc), greedy)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=12, generator=_g(3, cuda), **skw), sampled)
        gp, sp = dec._decode_graph_processed, dec._decode_graph_sampled_processed
        assert gp is not None and sp is not None
        assert dec._decode_graph is None and dec._decode_graph_sampled is None      # the plain graphs were not needed
        other = dict(proc, repetition_penalty=0.8, no_repeat_ngram_size=3, min_new_tokens=2)
        got = model.generate(ids, images=imgs, max_new_tokens=12, do_sample=False, **other)
        assert dec._decode_graph_processed is gp                                      # new settings, same graph
        model.enable_cuda_graphs(False)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=12, do_sample=False, **other), got)
    finally:
        model.enable_cuda_graphs(False)


def test_generate_without_processors_is_unchanged(gen, cuda):
    """Processor settings that are off leave the ids and the captured graph as they are; the processed graph differs from
    the plain one by exactly the vl2_process_logits launch."""
    from videollama2_b200 import ops
    model, ids, imgs = gen
    dec = model.get_model().decoder
    base = model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None)
    off = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=3)       # no EOS: the minimum is moot
    assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None, **off), base)
    model.enable_cuda_graphs(True)
    try:
        model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None)   # vision graphs
        dec._drop_decode_graphs()
        c0 = ops.launch_count()
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None, **off),
                           base)
        plain = ops.launch_count() - c0
        assert dec._decode_graph is not None and dec._decode_graph_processed is None
        c0 = ops.launch_count()
        model.generate(ids, images=imgs, max_new_tokens=9, do_sample=False, eos_token_id=None, repetition_penalty=1.2)
        processed = ops.launch_count() - c0
        # prefill + first-token processing + (2 warm-ups + 1 capture) x the step: 1 + 3 launches more than the plain run
        assert processed == plain + 4, (plain, processed)
    finally:
        model.enable_cuda_graphs(False)


def test_generate_every_token_banned_and_realloc(gen, cuda):
    model, ids, imgs = gen
    dec = model.get_model().decoder
    V = model.vocab_size
    everything = dict(suppress_tokens=list(range(V)), eos_token_id=None)
    eager = model.generate(ids, images=imgs, max_new_tokens=5, do_sample=False, **everything)
    assert eager[0].tolist() == [0] * 5
    model.enable_cuda_graphs(True)
    try:
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=5, generator=_g(1, cuda), do_sample=True,
                                          **everything), eager)
        # a longer generation reallocates the KV cache: the processed graph is captured again on the new cache
        model.generate(ids, images=imgs, max_new_tokens=5, do_sample=False, repetition_penalty=1.2)
        old = dec._decode_graph_processed
        cap = dec.kv[0].shape[0]
        longer = model.generate(ids, images=imgs, max_new_tokens=cap + 1, do_sample=False, repetition_penalty=1.2,
                                eos_token_id=None)
        assert dec.kv[0].shape[0] > cap and dec._decode_graph_processed is not old
        model.enable_cuda_graphs(False)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=cap + 1, do_sample=False,
                                          repetition_penalty=1.2, eos_token_id=None), longer)
    finally:
        model.enable_cuda_graphs(False)


def test_generate_batch_applies_processors_per_row(gen, cuda):
    model, ids, imgs = gen
    plain, proc = processors_for(model, ids, imgs, 8)
    one = model.generate(ids, images=imgs, max_new_tokens=8, do_sample=False, **proc)
    both = model.generate(torch.cat([ids, ids], 0), images=imgs + imgs, max_new_tokens=8, do_sample=False, **proc)
    assert torch.equal(both[0, :one.shape[1]], one[0]) and torch.equal(both[1, :one.shape[1]], one[0])

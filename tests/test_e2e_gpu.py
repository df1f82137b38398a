"""End-to-end parity of the engine against the CPU oracle (oracle/torch_ref.py, fp32 math on the same bf16-rounded
synthetic weights = "G32"), stage by stage and through the reference-shaped public API.

Tolerances (SURVEY.md §8c): relL2 <= 1e-2 against the fp32 golden for a stage fed the golden's stage input
(bf16-rounded); where a long chain of bf16 ops is compared at once (whole connector, end to end) the bar is
max(1e-2, 1.25 x the error the reference-style bf16 run itself has against the same golden at that point) — the
reference's own bf16 forward sits at 1.2e-2 (ViT) / 1.7e-2 (STC) at real size (BASELINE.md §4).
Integer work (splice rows, masks, labels, token ids) is exact."""
import pytest
import torch

from helpers import build_engine, rel

pytestmark = pytest.mark.gpu

CFGS = ["tiny", "tiny_qwen2", "tiny_v35", "tiny_siglip", "mid"]


@pytest.fixture(scope="module", params=CFGS)
def setup(request, cuda):
    from oracle import synth, torch_ref
    cfg = synth.CONFIGS[request.param]
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    gold = torch_ref.full_forward(sd, cfg, px, ids, torch.float32)
    hb = torch_ref.full_forward(sd, cfg, px, ids, torch.bfloat16)           # what the reference literally computes
    gold["noise_mm"] = rel(hb["mm"], gold["mm"])
    gold["noise_logits"] = rel(hb["logits"], gold["logits"])
    model = build_engine(cfg, sd, cuda)
    return cfg, sd, px, ids, gold, model


def test_vit_stage(setup, cuda):
    cfg, sd, px, ids, gold, model = setup
    feats = model.get_vision_tower()(px.to(cuda))
    assert feats.shape == gold["vit"].shape and feats.dtype == torch.bfloat16
    assert rel(feats, gold["vit"]) < 1e-2


def _tol(noise_bf16):
    """Parity bar: 1e-2, or the reference's own bf16-vs-fp32 error at that point when a chain of ops exceeds it."""
    return max(1e-2, 1.25 * noise_bf16)


def test_stc_substages_fed_oracle_input(setup, cuda):
    """Each connector stage is fed the fp32 golden of the previous stage (bf16-rounded) and compared with the golden."""
    from oracle import torch_ref
    cfg, sd, px, ids, gold, model = setup
    stc = model.get_model().mm_projector
    g = cfg.vision.grid
    vit_in = gold["vit"].to(torch.bfloat16)
    nb = torch_ref.stc_stages(sd, vit_in[None], cfg.stc_pad, cfg.stc_depth, torch.bfloat16)   # reference-style bf16 run
    gg = torch_ref.stc_stages(sd, vit_in[None].float(), cfg.stc_pad, cfg.stc_depth, torch.float32)
    s1 = stc.run_s1(vit_in.to(cuda).view(cfg.frames, g, g, -1))
    assert rel(s1, gg["s1"]) < _tol(rel(nb["s1"], gg["s1"]))
    smp = stc.run_sampler(gg["s1"].to(torch.bfloat16).to(cuda))
    ref_smp = torch_ref.F.silu(torch_ref.F.conv3d(gg["s1"].to(torch.bfloat16).float().permute(3, 0, 1, 2)[None],
                                                  sd["model.mm_projector.sampler.0.weight"].float(),
                                                  sd["model.mm_projector.sampler.0.bias"].float(), stride=2,
                                                  padding=cfg.stc_pad))[0].permute(1, 2, 3, 0)
    assert smp.shape == ref_smp.shape and rel(smp, ref_smp) < 1e-2
    out = stc(vit_in.to(cuda)[None])
    assert out.shape == (1,) + gold["mm"].shape
    assert rel(out[0], gg["out"][0]) < _tol(rel(nb["out"], gg["out"]))
    # 5-D input form (projector.py:199-200)
    out5 = stc(vit_in.to(cuda).view(1, cfg.frames, g, g, -1))
    assert torch.equal(out5, out)


def test_encode_and_aliases(setup, cuda):
    cfg, sd, px, ids, gold, model = setup
    mm = model.encode_images_or_videos([(px.to(cuda), "video")])
    assert mm.shape == (1, cfg.vis_tokens, cfg.llm.hidden)
    assert rel(mm[0], gold["mm"]) < _tol(gold["noise_mm"])
    assert model.encode_videos.__func__ is model.encode_images_or_videos.__func__
    # an image is encoded as num_frames identical frames (videollama2_arch.py:119-120)
    im = model.encode_images_or_videos([(px[:1].to(cuda), "image")])
    ref = model.encode_images_or_videos([(px[:1].expand(cfg.frames, -1, -1, -1).contiguous().to(cuda), "video")])
    assert torch.equal(im, ref)


def test_splice_is_exact(setup, cuda):
    cfg, sd, px, ids, gold, model = setup
    mask = torch.ones_like(ids, dtype=torch.bool)
    labels = ids.clone()
    r_ids, r_mask, _, embeds, r_labels = model.prepare_inputs_labels_for_multimodal(ids, mask, None, labels, [(px.to(cuda), "video")])
    assert r_ids is None and embeds.shape == (1, cfg.seq, cfg.llm.hidden)
    table = sd["model.embed_tokens.weight"].to(cuda)
    L = cfg.vis_tokens
    assert torch.equal(embeds[0, :4], table[ids[0, :4]])                       # text rows are bit-exact gathers
    assert torch.equal(embeds[0, 4 + L:], table[ids[0, 5:]])
    assert r_mask.shape == (1, cfg.seq) and bool(r_mask.all())
    assert torch.equal(r_labels[0, :4], ids[0, :4]) and (r_labels[0, 4:4 + L] == -100).all()
    assert torch.equal(r_labels[0, 4 + L:], ids[0, 5:])
    # early-outs (videollama2_arch.py:166-169)
    one = ids[:, :1].clamp(min=0)
    out = model.prepare_inputs_labels_for_multimodal(one, None, None, None, [(px.to(cuda), "video")])
    assert out[0] is one and out[3] is None


def test_decoder_stage_fed_oracle_input(setup, cuda):
    from oracle import torch_ref
    cfg, sd, px, ids, gold, model = setup
    emb = gold["inputs_embeds"].to(torch.bfloat16)
    ref = torch_ref.decoder_forward(sd, cfg.llm, emb, torch.float32)
    out = model(inputs_embeds=emb.to(cuda)[None])
    assert out.logits.shape == (1, cfg.seq, cfg.llm.vocab) and out.logits.dtype == torch.float32
    assert rel(out.logits[0], ref) < 1e-2
    last, _ = model.get_model().decoder.prefill(emb.to(cuda), all_logits=False)
    assert rel(last[0], ref[-1]) < 1e-2


def test_full_forward_and_generate(setup, cuda):
    cfg, sd, px, ids, gold, model = setup
    out = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(px.to(cuda), "video")])
    assert out.logits.shape == (1, cfg.seq, cfg.llm.vocab)
    assert rel(out.logits[0], gold["logits"]) < _tol(gold["noise_logits"])
    g_last = gold["logits"][-1]
    top2 = torch.topk(g_last, 2).values
    if (top2[0] - top2[1]) > 0.05 * g_last.abs().max():                       # unambiguous argmax only
        assert int(out.logits[0, -1].argmax()) == int(g_last.argmax())
    new = model.generate(ids, images=[(px.to(cuda), "video")], max_new_tokens=3, do_sample=False)
    assert new.shape[0] == 1 and 1 <= new.shape[1] <= 3 and new.dtype == torch.long
    assert int(new[0, 0]) == int(out.logits[0, -1].argmax())                  # first new token = prefill argmax


def test_kv_cache_decode_matches_recompute(setup, cuda):
    """KV-cache decode (GEMV + single-token attention kernels) against re-running the prefill kernels on the grown
    sequence, and against the oracle's greedy continuation computed in fp32 on the same weights."""
    from oracle import torch_ref
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    a = model.generate(ids, images=imgs, max_new_tokens=5, do_sample=False, use_cache=True)
    b = model.generate(ids, images=imgs, max_new_tokens=5, do_sample=False, use_cache=False)
    assert a.shape == (1, 5) and torch.equal(a, b)
    # logits of the decode step agree with a full recompute of the same sequence
    dec = model.get_model().decoder
    emb = gold["inputs_embeds"].to(torch.bfloat16).to(cuda)
    logits0, _ = dec.prefill(emb, all_logits=False, keep_cache=True, max_len=emb.shape[0] + 2)
    tok = int(logits0[0].argmax())
    e = model.get_model().embed_tokens(torch.tensor([tok]))
    step = dec.decode_step(e)
    full, _ = dec.prefill(torch.cat([emb, e], 0), all_logits=False)
    assert rel(step, full) < 1e-2
    ref = torch_ref.decoder_forward(sd, cfg.llm, torch.cat([emb.cpu(), e.cpu()], 0), torch.float32, all_logits=False)
    assert rel(step, ref) < 1.5e-2


def test_graph_replayed_decode_is_bit_exact(setup, cuda):
    """The single-token step captured as ONE CUDA graph (token and position in device memory, K/V appended by the
    RoPE kernel) must produce the same tokens and logits as the eager decode loop, across two generate() calls that
    reuse the captured graph, and with a stopping criterion that ends the loop early."""
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    dec = model.get_model().decoder
    eager = model.generate(ids, images=imgs, max_new_tokens=7, do_sample=False, use_cache=True)
    emb = gold["inputs_embeds"].to(torch.bfloat16).to(cuda)
    l0, _ = dec.prefill(emb, all_logits=False, keep_cache=True, max_len=emb.shape[0] + 4)
    t0 = int(l0[0].argmax())
    eager_logits = dec.decode_step(model.get_model().embed_tokens(torch.tensor([t0]))).clone()
    model.enable_cuda_graphs(True)
    try:
        for _ in range(2):
            assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=7, do_sample=False, use_cache=True), eager)
        assert dec._decode_graph is not None
        short = model.generate(ids, images=imgs, max_new_tokens=7, do_sample=False, use_cache=True,
                               stopping_criteria=[lambda out_ids, _s: out_ids.shape[1] >= 3])
        assert torch.equal(short, eager[:, :3])
        dec.prefill(emb, all_logits=False, keep_cache=True, max_len=emb.shape[0] + 4)
        dec.decode_graph_begin(t0)
        dec.decode_graph_step()
        assert torch.equal(dec.decode_graph_logits, eager_logits)
    finally:
        model.enable_cuda_graphs(False)


def test_graph_decode_with_l2_prefetch_fork(setup, cuda):
    """The decode graph with the forked weight-prefetch branch (vl2_l2_prefetch next to the attention phase) produces
    the same tokens: the fork only moves bytes into L2."""
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    dec = model.get_model().decoder
    eager = model.generate(ids, images=imgs, max_new_tokens=6, do_sample=False, use_cache=True)
    old = dec.decode_prefetch_mb
    dec.decode_prefetch_mb = 0.05
    model.enable_cuda_graphs(True)
    try:
        for _ in range(2):
            assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=6, do_sample=False, use_cache=True), eager)
    finally:
        model.enable_cuda_graphs(False)
        dec.decode_prefetch_mb = old


def test_cuda_graph_replay_is_bit_exact(setup, cuda):
    """Graph-replayed stages (tower, connector, last-position prefill) must reproduce the eager launches bit for bit,
    also on the second replay and after a different input went through the same graph."""
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    eager_mm = model.encode_images_or_videos(imgs).clone()
    eager_tok = model.generate(ids, images=imgs, max_new_tokens=1, do_sample=False)
    model.enable_cuda_graphs(True)
    try:
        for _ in range(2):
            assert torch.equal(model.encode_images_or_videos(imgs), eager_mm)
            assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=1, do_sample=False), eager_tok)
        other = [((px * 0.5).to(cuda), "video")]
        model.enable_cuda_graphs(False)
        ref_other = model.encode_images_or_videos(other).clone()
        model.enable_cuda_graphs(True)
        model.encode_images_or_videos(imgs)
        assert torch.equal(model.encode_images_or_videos(other), ref_other)
        assert torch.equal(model.encode_images_or_videos(imgs), eager_mm)
    finally:
        model.enable_cuda_graphs(False)


def test_vision_feature_cache(setup, cuda):
    """Second encode of the same frames (the eval runners' pattern) is served from the cache, bit-identical; changed
    pixels miss."""
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    ref = model.encode_images_or_videos(imgs).clone()
    model.enable_vision_cache(2)
    try:
        a = model.encode_images_or_videos(imgs)
        b = model.encode_images_or_videos([(px.to(cuda).clone(), "video")])       # a different tensor, same content
        assert model.vision_cache_hits == 1 and torch.equal(a, ref) and torch.equal(b, ref)
        other = model.encode_images_or_videos([((px * 0.5).to(cuda), "video")])
        assert model.vision_cache_hits == 1 and not torch.equal(other, ref)
        t0 = model.generate(ids, images=imgs, max_new_tokens=2, do_sample=False)
        assert model.vision_cache_hits == 2
        model.enable_vision_cache(0)
        assert torch.equal(model.generate(ids, images=imgs, max_new_tokens=2, do_sample=False), t0)
    finally:
        model.enable_vision_cache(0)


def test_raw_frames_to_tokens(setup, cuda):
    """The whole mm_infer-shaped path from decoded uint8 frames: device preprocessing (pad, Pillow-exact resize,
    normalise) -> tower -> connector -> splice -> prefill -> greedy tokens, against the oracle fed the oracle's own
    preprocessing of the same frames."""
    import numpy as np
    from oracle import preprocess_ref, torch_ref
    from videollama2_b200 import mm_utils
    cfg, sd, px, ids, gold, model = setup
    proc = model.get_vision_tower().image_processor
    size = cfg.vision.image
    kind = "siglip" if cfg.vision.kind == "siglip" else "clip"
    rng = np.random.default_rng(11)
    small = rng.integers(0, 256, (cfg.frames, 12, 20, 3), dtype=np.uint8)
    frames = np.repeat(np.repeat(small, 9, axis=1), 9, axis=2)                      # 108 x 180 blocky frames
    pix = mm_utils.process_video(frames, proc, num_frames=cfg.frames, device=cuda)
    _, ref_px = preprocess_ref.preprocess_frames(list(frames), size, kind, "pad", mean=tuple(proc.image_mean),
                                                 std=tuple(proc.image_std))
    assert pix.shape == (cfg.frames, 3, size, size)
    assert torch.equal(pix.cpu(), torch.from_numpy(ref_px).to(torch.bfloat16))    # pixel_values: bit-exact
    ref = torch_ref.full_forward(sd, cfg, pix.cpu(), ids, torch.float32)
    out = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(pix, "video")])
    noise = torch_ref.full_forward(sd, cfg, pix.cpu(), ids, torch.bfloat16)
    assert rel(out.logits[0], ref["logits"]) < _tol(rel(noise["logits"], ref["logits"]))
    new = model.generate(ids, images=[(pix, "video")], max_new_tokens=2, do_sample=False)
    assert int(new[0, 0]) == int(out.logits[0, -1].argmax())


def test_sampling_generate(setup, cuda):
    """do_sample=True: top_k = 1 reduces to greedy; a fixed generator gives the same tokens from the eager decode loop
    and from the graph-replayed one (the sampled token is written back into the graph's token buffer)."""
    cfg, sd, px, ids, gold, model = setup
    imgs = [(px.to(cuda), "video")]
    # eos_token_id=None: a sampled EOS must not cut the sequences short (this is a determinism test, not a stopping test)
    greedy = model.generate(ids, images=imgs, max_new_tokens=5, do_sample=False, eos_token_id=None)
    k1 = model.generate(ids, images=imgs, max_new_tokens=5, do_sample=True, temperature=0.7, top_p=0.9, top_k=1,
                        eos_token_id=None)
    assert torch.equal(k1, greedy)
    kw = dict(max_new_tokens=6, do_sample=True, temperature=1.5, top_p=0.95, eos_token_id=None)
    a = model.generate(ids, images=imgs, generator=torch.Generator(device=cuda).manual_seed(9), **kw)
    b = model.generate(ids, images=imgs, generator=torch.Generator(device=cuda).manual_seed(9), **kw)
    assert a.shape == (1, 6) and torch.equal(a, b)
    model.enable_cuda_graphs(True)
    try:
        c = model.generate(ids, images=imgs, generator=torch.Generator(device=cuda).manual_seed(9), **kw)
    finally:
        model.enable_cuda_graphs(False)
    assert torch.equal(c, a)


def test_no_cpu_fallback(setup):
    from videollama2_b200._lib import Vl2Error
    cfg, sd, px, ids, gold, model = setup
    with pytest.raises(Vl2Error):
        model.get_vision_tower()(px)                                           # CPU tensor must be refused loudly


@pytest.mark.parametrize("frames", [1, 7, 32])
def test_frame_count_edges(cuda, frames):
    """T = 1 (a single frame: every Conv3d window touches the zero padding), odd T, and the reference's MAX_FRAMES = 32
    (videollama2/constants.py:21) at tiny width, against the fp32 oracle; token count follows (T//2+1) * 3 * 3 here."""
    import dataclasses
    from oracle import synth, torch_ref
    cfg = dataclasses.replace(synth.CONFIGS["tiny"], frames=frames, name=f"tiny_f{frames}")
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    gold = torch_ref.full_forward(sd, cfg, px, ids, torch.float32)
    noise = torch_ref.full_forward(sd, cfg, px, ids, torch.bfloat16)
    model = build_engine(cfg, sd, cuda)
    mm = model.encode_images_or_videos([(px.to(cuda), "video")])
    assert mm.shape == (1, cfg.vis_tokens, cfg.llm.hidden) and cfg.vis_tokens == (frames // 2 + 1) * 9
    assert rel(mm[0], gold["mm"]) < _tol(rel(noise["mm"], gold["mm"]))
    out = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(px.to(cuda), "video")])
    assert rel(out.logits[0], gold["logits"]) < _tol(rel(noise["logits"], gold["logits"]))


def test_batch_of_two_videos_and_ragged_prompts(setup, cuda):
    """encode_images_or_videos with b = 2 (videollama2_arch.py:117-132) and a ragged batch through forward():
    per-sample results equal the single-sample runs bit for bit, padded logits rows are zero."""
    cfg, sd, px, ids, gold, model = setup
    px2 = (px * 0.7).to(cuda)
    both = model.encode_images_or_videos([(px.to(cuda), "video"), (px2, "video")])
    assert both.shape[0] == 2
    assert torch.equal(both[0], model.encode_images_or_videos([(px.to(cuda), "video")])[0])
    assert torch.equal(both[1], model.encode_images_or_videos([(px2, "video")])[0])
    ids_b = torch.stack([ids[0], ids[0].clone()])
    ids_b[1, 4] = 9            # second sample: text only (consumes a feature slot, inserts nothing: arch.py:181-191)
    mask_b = torch.ones_like(ids_b, dtype=torch.bool)
    out = model(input_ids=ids_b, attention_mask=mask_b, images=[(px.to(cuda), "video"), (px2, "video")])
    S_long, S_short = cfg.seq, cfg.prompt
    assert out.logits.shape == (2, S_long, cfg.llm.vocab)
    single = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(px.to(cuda), "video")])
    assert torch.equal(out.logits[0], single.logits[0])
    assert float(out.logits[1, S_short:].abs().max()) == 0.0
    text_only = model(inputs_embeds=model.get_model().embed_tokens(ids_b[1:2]))
    assert torch.equal(out.logits[1, :S_short], text_only.logits[0])


def test_generate_batch_of_two(setup, cuda):
    """generate() on a right-padded batch of two prompts (one with a video, one text-only that still consumes its image
    slot): every row equals its own batch-1 generate, shorter outputs are padded with pad_token_id."""
    cfg, sd, px, ids, gold, model = setup
    px2 = (px * 0.7).to(cuda)
    short = ids[0, :8].clone()
    short[4] = 9                                                    # no placeholder in the short prompt
    P = ids.shape[1]
    ids_b = torch.zeros((2, P), dtype=torch.long)
    ids_b[0] = ids[0]
    ids_b[1, :8] = short
    mask_b = torch.zeros((2, P), dtype=torch.bool)
    mask_b[0] = True
    mask_b[1, :8] = True
    images = [(px.to(cuda), "video"), (px2, "video")]
    out = model.generate(ids_b, images=images, attention_mask=mask_b, max_new_tokens=4, do_sample=False, pad_token_id=0)
    a = model.generate(ids, images=images[:1], max_new_tokens=4, do_sample=False)
    b = model.generate(short[None], images=images[1:], max_new_tokens=4, do_sample=False)
    assert out.shape[0] == 2 and torch.equal(out[0, : a.shape[1]], a[0]) and torch.equal(out[1, : b.shape[1]], b[0])
    assert int(out[0, a.shape[1]:].abs().sum()) == 0 and int(out[1, b.shape[1]:].abs().sum()) == 0


def test_forward_with_past_key_values(setup, cuda):
    """HF generation-loop call pattern through forward(): prefill with use_cache=True, then one token at a time with the
    returned past_key_values handle; the greedy tokens equal generate()'s, stale handles are refused."""
    cfg, sd, px, ids, gold, model = setup
    images = [(px.to(cuda), "video")]
    want = model.generate(ids, images=images, max_new_tokens=4, do_sample=False)
    out = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=images, use_cache=True)
    assert out.past_key_values is not None and out.past_key_values.get_seq_length() == cfg.seq
    toks = [int(out.logits[0, -1].argmax())]
    pkv = out.past_key_values
    for _ in range(3):
        step = model(input_ids=torch.tensor([[toks[-1]]]), past_key_values=pkv)
        assert step.logits.shape == (1, 1, cfg.llm.vocab)
        toks.append(int(step.logits[0, -1].argmax()))
        pkv = step.past_key_values
    assert toks == want[0].tolist()
    model.generate(ids, images=images, max_new_tokens=2, do_sample=False)        # a new prefill invalidates the handle
    with pytest.raises(ValueError):
        model(input_ids=torch.tensor([[toks[-1]]]), past_key_values=pkv)

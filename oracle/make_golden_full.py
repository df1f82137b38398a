"""Full-depth goldens for the BASELINE configs (cfg1, cfg2 = Mistral-7B; cfg3 = Qwen2-7B at its real geometry), produced
by the REAL reference classes (oracle/ref_loader.py imports them from /root/reference) on CPU with the deterministic
synthetic weights / inputs of oracle/synth.py (SURVEY.md §8d).  TEST INFRASTRUCTURE; build container only:

    python -m oracle.make_golden_full [mistral] [qwen2]

For each config two runs of the unmodified reference forward (videollama2_mistral.py:63-108 / videollama2_qwen2.py:61-102):
  G32   fp32 arithmetic on the bf16-rounded weights  (the golden)
  Hbf16 the reference as it literally computes in bf16 (the noise floor a bf16 engine is judged against)
Both runs are tapped with forward hooks at: ViT tower output (hidden_states[-2][:,1:]), mm_projector output, decoder
layers {0, mid, last} outputs, and the last-position logits.  The 7B tensors do not fit a repo, so the fixture keeps
  * G32 row slices at fixed pseudo-random rows (16 rows per tap, every column), G32 + Hbf16 last-position logits,
  * per-tap relL2(Hbf16, G32) on the slice and on the full tensor, per-frame / per-tap norms of the full G32 tensors.
The GPU box regenerates the same weights from the seed (same image => same torch CPU RNG stream), runs the engine at
full depth and compares at the same rows (tests/test_fulldepth_gpu.py, bench.py --check)."""
from __future__ import annotations

import concurrent.futures as cf
import gc
import os
import sys
import time

import torch

from . import ref_loader, synth

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
ROWS = 16


def tap_rows(cfg) -> dict:
    """Fixed rows per tap (a function of the config only: the GPU side recomputes them)."""
    g = torch.Generator(device="cpu").manual_seed(4242)
    F, NP = cfg.frames, cfg.vision.num_patches
    vit = torch.stack([torch.randint(0, F, (ROWS,), generator=g), torch.randint(0, NP, (ROWS,), generator=g)], 1)
    vit[0] = torch.tensor([0, 0])
    vit[1] = torch.tensor([F - 1, NP - 1])
    mm = torch.randint(0, cfg.vis_tokens, (ROWS,), generator=g)
    mm[0], mm[1] = 0, cfg.vis_tokens - 1
    S = cfg.seq
    dec = torch.randint(0, S, (ROWS,), generator=g)
    dec[0], dec[1], dec[2], dec[3] = 0, 3, 4, S - 1     # text row, row before <video>, first visual row, last row
    return {"vit": vit, "mm": mm.sort().values, "dec": dec.sort().values}


def dec_tap_layers(n_layers: int):
    return (0, n_layers // 2 - 1, n_layers - 1)


def build_streaming(cfg, dtype):
    """The reference *ForCausalLM for `cfg`, weights filled tensor by tensor from oracle.synth (never two copies of the
    7B state in memory).  Same config construction as ref_loader.build_reference_model."""
    model_mod = ref_loader.load()
    try:
        from transformers.initialization import no_init_weights
    except Exception:                                                       # older transformers
        from transformers.modeling_utils import no_init_weights
    l = cfg.llm
    common = dict(hidden_size=l.hidden, intermediate_size=l.inter, num_hidden_layers=l.layers,
                  num_attention_heads=l.heads, num_key_value_heads=l.kv_heads, vocab_size=l.vocab,
                  rms_norm_eps=l.eps, rope_theta=l.theta, max_position_embeddings=32768, tie_word_embeddings=False,
                  attn_implementation=os.environ.get("VL2_ORACLE_ATTN", "sdpa"))
    if l.kind == "qwen2":
        hf_cfg = model_mod.Videollama2Qwen2Config(**common, use_sliding_window=False)
        cls = model_mod.Videollama2Qwen2ForCausalLM
    else:
        hf_cfg = model_mod.Videollama2MistralConfig(**common, sliding_window=None)
        cls = model_mod.Videollama2MistralForCausalLM
    hf_cfg.mm_vision_tower = ref_loader.clip_dir(cfg.vision)
    hf_cfg.mm_projector_type = cfg.projector
    hf_cfg.mm_hidden_size = cfg.vision.hidden
    hf_cfg.mm_vision_select_layer = cfg.select_layer
    hf_cfg.mm_vision_select_feature = "patch"
    hf_cfg.num_frames = cfg.frames
    t0 = time.time()
    old = torch.get_default_dtype()
    torch.set_default_dtype(dtype)          # parameters are created directly in the target dtype (no fp32 detour)
    try:
        with no_init_weights():
            model = cls(hf_cfg)
    finally:
        torch.set_default_dtype(old)
    params = dict(model.named_parameters())
    specs = synth.model_specs(cfg)
    names = {s[0] for s in specs}
    missing = [k for k in params if k not in names]
    extra = [k for k in names if k not in params]
    if missing or extra:
        raise RuntimeError(f"state-dict mismatch: model-only={missing[:6]} synth-only={extra[:6]}")

    def fill(spec):
        name, shape, kind = spec
        p = params[name]
        assert tuple(p.shape) == tuple(shape), (name, p.shape, shape)
        with torch.no_grad():
            p.copy_(synth.make_tensor(name, shape, kind))          # bf16-rounded values into fp32 / bf16 storage
        return p.numel()

    with cf.ThreadPoolExecutor(8) as ex:
        n = sum(ex.map(fill, specs))
    # no_init_weights leaves buffers alone: inv_freq (fp32, from the config) and CLIP position_ids are computed in the
    # constructors; make sure they survived and are not bf16-rounded
    for bname, buf in model.named_buffers():
        if "inv_freq" in bname:
            assert buf.dtype == torch.float32, (bname, buf.dtype)
    model.eval()
    print(f"  built {cls.__name__} {dtype}: {n / 1e9:.2f} B params in {time.time() - t0:.0f}s", flush=True)
    return model


def run_tapped(model, cfg, dtype):
    px, ids = synth.inputs(cfg)
    taps = {}
    hooks = []
    inner = model.get_model()
    hooks.append(inner.get_vision_tower().register_forward_hook(lambda m, i, o: taps.__setitem__("vit", o.detach().float())))
    hooks.append(inner.mm_projector.register_forward_hook(lambda m, i, o: taps.__setitem__("mm", o.detach().float())))
    for li in dec_tap_layers(cfg.llm.layers):
        def hook(m, i, o, li=li):
            taps[f"dec{li}"] = (o[0] if isinstance(o, (tuple, list)) else o).detach().float()[0]
        hooks.append(inner.layers[li].register_forward_hook(hook))
    t0 = time.time()
    with torch.no_grad():
        model.config.num_frames = cfg.frames
        res = model(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(px.to(dtype), "video")])
    taps["logits_last"] = res.logits[0, -1].detach().float().clone()
    for h in hooks:
        h.remove()
    taps["vit"] = taps["vit"].reshape(cfg.frames, cfg.vision.num_patches, cfg.vision.hidden)
    taps["mm"] = taps["mm"].reshape(cfg.vis_tokens, cfg.llm.hidden)
    print(f"    {cfg.name} {dtype} forward {time.time() - t0:.0f}s  S={taps[f'dec0'].shape[0]}", flush=True)
    return taps


def slice_taps(taps, rows, cfg):
    out = {"vit": taps["vit"][rows["vit"][:, 0], rows["vit"][:, 1]].clone(), "mm": taps["mm"][rows["mm"]].clone()}
    for li in dec_tap_layers(cfg.llm.layers):
        out[f"dec{li}"] = taps[f"dec{li}"][rows["dec"]].clone()
    return out


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def main():
    os.makedirs(OUT, exist_ok=True)
    want = sys.argv[1:] or ["mistral", "qwen2"]
    groups = {"mistral": ["cfg1", "cfg2"], "qwen2": ["cfg3"]}
    torch.set_num_threads(os.cpu_count() or 1)
    for grp in want:
        names = groups[grp]
        gold, noise = {}, {}
        for tag, dt in (("g32", torch.float32), ("hbf16", torch.bfloat16)):
            model = build_streaming(synth.CONFIGS[names[0]], dt)
            for name in names:
                cfg = synth.CONFIGS[name]
                taps = run_tapped(model, cfg, dt)
                (gold if tag == "g32" else noise)[name] = taps
            del model
            gc.collect()
        for name in names:
            cfg = synth.CONFIGS[name]
            rows = tap_rows(cfg)
            g, h = gold[name], noise[name]
            gs, hs = slice_taps(g, rows, cfg), slice_taps(h, rows, cfg)
            keys = list(gs.keys())
            top = torch.topk(g["logits_last"], 5)
            fx = {
                "config": name, "rows": rows, "dec_tap_layers": [int(i) for i in dec_tap_layers(cfg.llm.layers)],
                # fp16 storage (relative rounding <= 2^-11, far below the >= 1e-2 parity bars) keeps a fixture under 1 MB
                "g32": {k: v.half() for k, v in {**gs, "logits_last": g["logits_last"]}.items()},
                "noise_slice": {k: rel(hs[k], gs[k]) for k in keys},
                "noise_full": {**{k: rel(h[k], g[k]) for k in keys}, "logits_last": rel(h["logits_last"], g["logits_last"])},
                "norms": {"vit_per_frame": g["vit"].flatten(1).norm(dim=1), "mm": g["mm"].norm().item(),
                          **{k: g[k].norm().item() for k in keys if k.startswith("dec")}},
                "argmax_g32": int(top.indices[0]), "argmax_hbf16": int(h["logits_last"].argmax()),
                "top5_g32": top.indices.tolist(), "top2_margin_g32": float(top.values[0] - top.values[1]),
                "logit_noise_absmax": float((h["logits_last"] - g["logits_last"]).abs().max()),
                "torch": str(torch.__version__),
            }
            torch.save(fx, os.path.join(OUT, f"full_{name}.pt"))
            print(name, "noise_full", {k: round(v, 4) for k, v in fx["noise_full"].items()}, "argmax g32/hbf16",
                  fx["argmax_g32"], fx["argmax_hbf16"], "margin", round(fx["top2_margin_g32"], 4), "logit noise max",
                  round(fx["logit_noise_absmax"], 4), flush=True)
        del gold, noise
        gc.collect()


if __name__ == "__main__":
    main()

"""Full-depth parity check of a loaded engine against a committed golden fixture (tests/golden/full_<cfg>.pt).

The fixtures hold what the REAL reference classes computed on CPU for the synthetic checkpoint of presets.synth_tensor
(fp32 arithmetic "g32" = golden; the reference's own bf16 run gives the noise floor) at fixed rows of five taps: ViT
tower output, connector output, decoder layers {first, middle, last}, plus the last-position logits.  This module only
reads that data file: it runs the engine's own kernels end to end (pixels + ids -> logits) and compares at the same rows.
Used by tests/test_fulldepth_gpu.py and by `bench.py --check` so the benchmarked weights/output are themselves verified.
Bars (SURVEY.md §8c): relL2 <= max(1e-2, 1.25 x the reference's bf16-vs-fp32 error at that tap); same arg-max token unless
the golden's own top-2 gap is inside the bf16 noise."""
from __future__ import annotations

import os
from typing import Optional

import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def fixture_path(name: str) -> str:
    return os.path.join(GOLDEN_DIR, f"full_{name}.pt")


def _rel(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


@torch.no_grad()
def fulldepth_check(model, fixture: str, pixels: torch.Tensor, input_ids: torch.Tensor, slack: float = 1.25) -> dict:
    """Runs pixels [T,3,H,W] + input_ids [1,P] through the engine eagerly with taps; returns per-tap errors, bars and
    `ok`.  `fixture` is a config name ("cfg2") or a path."""
    path = fixture if os.path.exists(fixture) else fixture_path(fixture)
    fx = torch.load(path, map_location="cpu")
    rows, gold = fx["rows"], {k: v.float() for k, v in fx["g32"].items()}   # stored as fp16
    dev = model.device
    inner = model.get_model()
    tower = inner.get_vision_tower()
    px = pixels.to(dev)
    feats = tower(px)                                                    # [T, np, C]
    T = px.shape[0]
    mm = inner.mm_projector(feats.view(1, T, feats.shape[1], feats.shape[2]))[0]      # [L, H]
    mask = torch.ones_like(input_ids, dtype=torch.bool)
    _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(input_ids, mask, None, None, [(px, "video")])
    dec_rows = rows["dec"].to(dev)
    taps = {}
    want = set(int(i) for i in fx["dec_tap_layers"])
    logits, _ = inner.decoder.prefill(emb[0], all_logits=False,
                                      tap=lambda i, x: taps.__setitem__(f"dec{i}", x[dec_rows].float().cpu()) if i in want else None)
    torch.cuda.synchronize(dev)
    got = {"vit": feats[rows["vit"][:, 0].to(dev), rows["vit"][:, 1].to(dev)], "mm": mm[rows["mm"].to(dev)], **taps}
    out = {"fixture": os.path.basename(path), "taps": {}, "ok": True}
    for k, g in gold.items():
        if k == "logits_last":
            continue
        err = _rel(got[k], g)
        bar = max(1e-2, slack * float(fx["noise_slice"][k]))
        out["taps"][k] = {"rel_l2": err, "bar": bar, "reference_bf16_rel_l2": float(fx["noise_slice"][k])}
        out["ok"] = out["ok"] and err <= bar
    lg = logits[0].float().cpu()
    err = _rel(lg, gold["logits_last"])
    bar = max(1e-2, slack * float(fx["noise_full"]["logits_last"]))
    am = int(lg.argmax())
    gap = float(gold["logits_last"][fx["argmax_g32"]] - gold["logits_last"][am])     # 0 when the tokens agree
    am_ok = am == int(fx["argmax_g32"]) or gap <= 2.0 * float(fx["logit_noise_absmax"])
    out["taps"]["logits_last"] = {"rel_l2": err, "bar": bar, "reference_bf16_rel_l2": float(fx["noise_full"]["logits_last"])}
    out["argmax"] = {"engine": am, "golden_fp32": int(fx["argmax_g32"]), "reference_bf16": int(fx["argmax_hbf16"]),
                     "golden_gap_to_engine_token": gap, "ok": bool(am_ok)}
    out["ok"] = bool(out["ok"] and err <= bar and am_ok)
    # size-independent property on the FULL ViT output: per-frame norms against the golden's
    nf = feats.float().flatten(1).norm(dim=1).cpu()
    out["vit_frame_norm_max_rel_dev"] = float(((nf - fx["norms"]["vit_per_frame"]).abs() / fx["norms"]["vit_per_frame"]).max())
    out["ok"] = bool(out["ok"] and out["vit_frame_norm_max_rel_dev"] < 2e-2)
    return out

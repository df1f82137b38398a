"""vl2_gemm_bf16 against cuBLAS at every GEMM of one config-2 step (Mistral-7B, 16 frames at 336 px), with the kernel's
own cycle trace.

The shapes are recorded, not listed: one eager step of the model (random weights) runs with `ops.gemm` wrapped the way
bench.py wraps it, and every distinct (M, N, K, epilogue) is kept together with the operands of its first call.  Each one
is then timed with CUDA events, alternating our kernel (with its epilogue) and cuBLAS (`torch.nn.functional.linear`,
bf16, no epilogue) on the same operands.  The kernel's trace (`trace=True`: first consumer thread of CTA 0, up to 7
tiles) gives per tile the k-loop cycles (start -> accumulator complete), the same per k-block, and the epilogue cycles
(accumulator complete -> stored).  The tensor pipe's bound for one k-block of a 128 x BN tile is 128 * BN * 64 MACs at
2048 MACs per clock per SM, i.e. 4 * BN cycles.

Inside the first 32-column slot of a tile the trace also records (generic epilogue only) the accumulators selected and
the residuals loaded, and (every epilogue) the slot stored: `slot0_cyc` = [select, residual round trip, whole slot].

Usage: python scripts/microbench_gemm.py [--reps R] [--iters N] [--json FILE] [--generic]
       --generic forces the library's generic epilogue instead of each launch's specialised variant.
       VL2_LIBVL2=/path/to/libvl2.so selects another build of the library (to compare two builds; --generic and the
       slot trace need a build that has them).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from videollama2_b200 import _lib, ops, presets
from videollama2_b200.model import VLLMs

FRAMES, PROMPT = 16, 256   # bench.py's config-2 step
BK = 64


def record_step_gemms(dev):
    cfg = presets.make_config(presets.MISTRAL_7B, FRAMES)
    sd = presets.random_state_dict(cfg, dev)
    model = VLLMs[cfg.model_type].from_state_dict(cfg, sd, device=dev)
    del sd
    model.enable_cuda_graphs(False)
    px, ids = presets.synthetic_inputs(cfg, FRAMES, PROMPT)
    px = px.to(cfg.storage_dtype).to(dev)
    mask = torch.ones_like(ids, dtype=torch.bool)
    seen = {}
    orig = ops.gemm

    def key_of(a, w, kw):
        out = kw.get("out")
        return (a.shape[0], w.shape[0], a.shape[1], int(kw.get("act", 0)),
                "bias" if kw.get("bias") is not None else "", "res" if kw.get("residual") is not None else "",
                "rms" if kw.get("rms_in") is not None else "", "ln" if kw.get("ln_in") is not None else "",
                "stats" if kw.get("sumsq_out") is not None else "", "rope" if kw.get("rope") is not None else "",
                "f32" if (out is not None and out.dtype == torch.float32) or kw.get("out_dtype") == torch.float32 else "")

    def gemm_rec(a, w, **kw):
        out = orig(a, w, **kw)
        k = key_of(a, w, kw)
        if k in seen:
            seen[k]["calls"] += 1
        else:
            kw = dict(kw)
            kw.setdefault("out", out)
            seen[k] = {"a": a, "w": w, "kw": kw, "calls": 1}
        return out

    mods = [sys.modules["videollama2_b200.model." + m] for m in ("encoder", "projector", "decoder")]
    for m in mods:
        m.ops = type("OpsProxy", (), {"__getattr__": lambda self, n, _o=ops: gemm_rec if n == "gemm" else getattr(_o, n)})()
    try:
        with torch.no_grad():
            _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, mask, None, None, [(px, "video")])
            model.get_model().decoder.prefill(emb[0], all_logits=False)
        torch.cuda.synchronize()
    finally:
        for m in mods:
            m.ops = ops
    return seen


def events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--generic", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.load()
    props = torch.cuda.get_device_properties(dev)
    info = {"lib": _lib.LIB_PATH, "device": props.name, "sms": props.multi_processor_count, "generic": args.generic}
    if hasattr(lib, "vl2_gemm_coresident"):   # absent from builds older than the query
        lib.vl2_gemm_coresident.argtypes = [C.c_int, C.c_int, C.c_void_p]
        res = C.c_int32()
        info["coresident_pairs"] = {}
        for bn in (128, 160, 192, 224, 256):
            ops.check(lib.vl2_gemm_coresident(bn, 1, C.byref(res)), "vl2_gemm_coresident")
            info["coresident_pairs"][bn] = res.value
    print(json.dumps(info), flush=True)

    seen = record_step_gemms(dev)
    plan = (C.c_int32 * 6)()
    rows = []
    for k, rec in seen.items():
        a, w, kw = rec["a"], rec["w"], rec["kw"]
        if args.generic:
            kw = dict(kw, generic_epilogue=True)
        M, N, K = k[0], k[1], k[2]
        ops.check(lib.vl2_gemm_plan(M, N, K, 0, plan), "vl2_gemm_plan")
        bn, pair = plan[0], plan[1]

        def ours():
            ops.gemm(a, w, **kw)

        def cublas():
            F.linear(a, w)

        for _ in range(3):
            ours()
            cublas()
        torch.cuda.synchronize()
        t_ours, t_cub = [], []
        for _ in range(args.reps):   # alternated: both see the same clocks and neighbours
            t_ours.append(events_ms(ours, args.iters))
            t_cub.append(events_ms(cublas, args.iters))
        us, us_cub = statistics.median(t_ours) * 1e3, statistics.median(t_cub) * 1e3
        flop = 2.0 * M * N * K

        ops.gemm(a, w, **kw, trace=True)
        t = ops.gemm_trace()
        nkb = (K + BK - 1) // BK
        tiles = [(t[8 * i + 4], t[8 * i + 5], t[8 * i + 6]) for i in range(int(t[0]))]
        kloop = [acc - st for st, acc, _ in tiles]
        epi = [done - acc for _, acc, done in tiles]
        # first slot of each tile: [accumulators selected, residuals loaded, slot stored] after the accumulator is complete
        slot0 = [[t[8 * i + j] - t[8 * i + 5] if t[8 * i + j] >= t[8 * i + 5] else None for j in (1, 2, 3)]
                 for i in range(int(t[0]))]
        row = {"M": M, "N": N, "K": K, "epilogue": "+".join([f"act{k[3]}"] * (k[3] != 0) + [x for x in k[4:] if x]) or "-",
               "act": k[3], "calls_per_step": rec["calls"], "bn": bn, "pair": pair,
               "us": round(us, 1), "TFs": round(flop / us / 1e6, 1), "cublas_us": round(us_cub, 1),
               "cublas_TFs": round(flop / us_cub / 1e6, 1), "frac_of_cublas": round(us_cub / us, 3),
               "kb_per_tile": nkb, "mma_bound_cyc_per_kb": 4 * bn,
               "kloop_cyc_per_kb": [round(c / nkb) for c in kloop], "epi_cyc": epi, "slot0_cyc": slot0}
        rows.append(row)
        print(json.dumps(row), flush=True)

    tot = sum(r["us"] * r["calls_per_step"] for r in rows) / 1e3
    tot_cub = sum(r["cublas_us"] * r["calls_per_step"] for r in rows) / 1e3
    summary = {"distinct": len(rows), "launches_per_step": sum(r["calls_per_step"] for r in rows),
               "gemm_ms_per_step": round(tot, 2), "cublas_ms_per_step": round(tot_cub, 2)}
    print(json.dumps(summary), flush=True)
    print(f"\n{'M':>6} {'N':>6} {'K':>6} {'epilogue':<14} {'x':>3} {'tile':>6} {'us':>8} {'TF/s':>6} {'cuBLAS':>7} "
          f"{'frac':>5} {'cyc/kb':>7} {'bound':>6} {'epi cyc':>8}")
    for r in rows:
        kb = statistics.median(r["kloop_cyc_per_kb"][1:] or r["kloop_cyc_per_kb"]) if r["kloop_cyc_per_kb"] else 0
        ep = statistics.median(r["epi_cyc"]) if r["epi_cyc"] else 0
        tile = f"{'2x' if r['pair'] else ''}{r['bn']}"
        print(f"{r['M']:>6} {r['N']:>6} {r['K']:>6} {r['epilogue']:<14} {r['calls_per_step']:>3} {tile:>6} {r['us']:>8.1f} "
              f"{r['TFs']:>6.1f} {r['cublas_TFs']:>7.1f} {r['frac_of_cublas']:>5.2f} {kb:>7.0f} {r['mma_bound_cyc_per_kb']:>6} "
              f"{ep:>8.0f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"info": info, "rows": rows, "summary": summary}, fh, indent=1)


if __name__ == "__main__":
    main()

"""Cost of recording generate()'s per-step scores on the GPU.  Prints one JSON line with the card's name, power limit
and SM clock, read in the same run.

1. Kernels at V = 32000 (Mistral) and 152064 (Qwen2), CUDA graphs of 500 launches timed by CUDA events: vl2_record_row
   alone, and vl2_sample_token_scored against vl2_sample_token on the same row, alternated.
2. Decode graphs on the synthetic checkpoints of config 2 (Mistral-7B) and of Qwen2-7B's geometry, after a prefill of
   S = 1776 random embeddings (the vision tower does not enter a decode step): device ms per token of the recording
   decode graph (scores and logits both recorded) against the plain one, greedy and sampled, alternated in one run.
Usage: python scripts/microbench_scores.py [--no-model]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from videollama2_b200 import _lib, ops

dev = torch.device("cuda:0")
SAMPLING = dict(temperature=0.7, top_k=50, top_p=0.9)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True).stdout.strip()
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def events_us(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


def graph_of(fn, n):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    return g


def kernel_times():
    res = {}
    n = 500
    for V in (32000, 152064):
        row = (torch.randn(V, generator=torch.Generator().manual_seed(V)) * 3.0).to(dev)
        step = torch.zeros((1,), dtype=torch.int64, device=dev)
        tok = torch.zeros((1,), dtype=torch.int64, device=dev)
        buf = torch.empty((2, V), dtype=torch.float32, device=dev)
        rec = ops.score_record_params(V, 2, buf, buf.clone())
        params = ops.sampling_params(SAMPLING["temperature"], SAMPLING["top_k"], SAMPLING["top_p"], 1, dev)
        graphs = {
            "record_row": graph_of(lambda: ops.record_rows(row, rec, _lib.RECORD_LOGITS, step, 1), n),
            "sample_token": graph_of(lambda: ops.sample_token(row, params, step, 1, tok), n),
            "sample_token_scored": graph_of(lambda: ops.sample_token(row, params, step, 1, tok, record=rec), n),
        }
        t = {k: [] for k in graphs}
        for _ in range(5):
            for k, g in graphs.items():
                t[k].append(events_us(g.replay, n))
        res[f"V{V}"] = {f"{k}_us": round(min(v), 2) for k, v in t.items()}
        res[f"V{V}"]["scored_added_us"] = round(min(t["sample_token_scored"]) - min(t["sample_token"]), 2)
    return res


def model_times(llm: dict, label: str):
    from videollama2_b200 import presets
    from videollama2_b200.model import VLLMs
    cfg = presets.make_config(llm, 16)
    sd = presets.synthetic_state_dict(cfg, dev, threads=max(1, min(16, os.cpu_count() or 8)))
    model = VLLMs[cfg.model_type].from_state_dict(cfg, sd, device=dev)
    del sd
    torch.cuda.empty_cache()
    model.enable_cuda_graphs(True)
    dec = model.get_model().decoder
    V, S, K = cfg.vocab_size, 1776, 64
    x = (torch.randn((S, cfg.hidden_size), generator=torch.Generator().manual_seed(0)) * 0.02).to(dev, dec.dtype)
    dec.prefill(x, all_logits=False, keep_cache=True, max_len=S + K + 1)
    rec = ops.score_record_params(V, K + 1, torch.empty((K + 1, V), device=dev), torch.empty((K + 1, V), device=dev))
    sampling = ops.sampling_params(SAMPLING["temperature"], SAMPLING["top_k"], SAMPLING["top_p"], 5, dev)
    res = {"S": S, "V": V, "tokens_per_run": K}
    for mode, sp in (("greedy", None), ("sampled", sampling)):
        ms = {"plain": [], "recorded": []}
        for _ in range(4):
            for name, r in (("plain", None), ("recorded", rec)):
                dec.kv_len = S                           # every run decodes positions S .. S + K - 1 again
                dec.decode_graph_begin(3, sp, None, r)
                ms[name].append(events_us(lambda: dec.decode_graph_run(K), K) / 1e3)
        res[f"{mode}_graph_ms_per_token_device"] = {k: [round(v, 4) for v in vs] for k, vs in ms.items()}
        res[f"{mode}_added_us_per_token"] = round((min(ms["recorded"]) - min(ms["plain"])) * 1e3, 1)
    del model, dec
    torch.cuda.empty_cache()
    return {label: res}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("microbench_scores needs a CUDA device")
    from videollama2_b200 import presets
    out = {"card": card(), "kernel": kernel_times()}
    if "--no-model" not in sys.argv:
        out.update(model_times(presets.MISTRAL_7B, "config2_mistral7b"))
        out.update(model_times(presets.QWEN2_7B, "qwen2_7b_geometry"))
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

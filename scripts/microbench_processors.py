"""Cost of the logits processors on the GPU.  Prints one JSON line with the card's name, power limit and SM clock.

1. The tail of a decode step at V = 32000 (Mistral) and 152064 (Qwen2), with history lengths 1 to 2048: a CUDA graph of
   500 x { vl2_process_logits -> arg-max } against 500 x { arg-max }, alternated, CUDA events.  Every processor is on:
   repetition_penalty 1.1, no_repeat_ngram_size 3, min_new_tokens above n with two EOS ids, four bad-word sequences and
   eight suppressed tokens.  The history repeats a few ids, so the penalty, n-gram and bad-word paths all do work.
2. Config 2 (Mistral-7B, 16 frames@336, S = 1776) on the synthetic checkpoint bench.py builds: ms per token of the
   processed greedy decode graph against the plain greedy graph, replayed back to back and alternated in one run, with
   64 and 2048 new tokens of history.
Usage: python scripts/microbench_processors.py [--no-model]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from videollama2_b200 import ops

dev = torch.device("cuda:0")
HISTORIES = (1, 64, 512, 2048)


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


def processors(V, n):
    return dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=n + 1, eos_token_ids=(2, V - 1),
                bad_words_ids=[[5], [7, 9], [3, 4, 11], [1, 2, 3, 4, 6]], suppress_tokens=list(range(100, 108)))


def history(n):
    g = torch.Generator().manual_seed(n)
    return torch.randint(0, 50, (n,), generator=g).to(dev)


def graph_of(fn, n):
    fn()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    return g


def kernel_times():
    res = {}
    n_launch = 500
    for V in (32000, 152064):
        row = (torch.randn(V, generator=torch.Generator().manual_seed(V)) * 3.0).to(dev)
        tok = torch.zeros((1,), dtype=torch.int64, device=dev)
        zero = torch.zeros((1,), dtype=torch.int64, device=dev)
        plain = graph_of(lambda: tok.copy_(torch.argmax(row[None], dim=1)), n_launch)
        for n in HISTORIES:
            params, hist = ops.logits_process_params(V, dev, **processors(V, n)), history(n)
            work = row.clone()

            def step():
                ops.process_logits(work, params, hist, zero, n)
                tok.copy_(torch.argmax(work[None], dim=1))
            processed = graph_of(step, n_launch)
            t = {"plain": [], "processed": []}
            for _ in range(3):
                t["plain"].append(events_us(plain.replay, n_launch))
                t["processed"].append(events_us(processed.replay, n_launch))
            res[f"V{V}_n{n}"] = {"plain_us": round(min(t["plain"]), 2), "processed_us": round(min(t["processed"]), 2),
                                 "added_us": round(min(t["processed"]) - min(t["plain"]), 2)}
    return res


def model_times():
    import bench
    from videollama2_b200 import presets
    from videollama2_b200.model import VLLMs
    cfg = presets.make_config(presets.MISTRAL_7B, bench.FRAMES)
    sd = presets.synthetic_state_dict(cfg, dev, threads=max(1, min(16, os.cpu_count() or 8)))
    model = VLLMs[cfg.model_type].from_state_dict(cfg, sd, device=dev)
    del sd
    torch.cuda.empty_cache()
    model.enable_cuda_graphs(True)
    px, ids = presets.synthetic_inputs(cfg, bench.FRAMES, bench.PROMPT)
    imgs = [(px.to(cfg.storage_dtype).to(dev), "video")]
    mask = torch.ones_like(ids, dtype=torch.bool)
    dec = model.get_model().decoder
    _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, mask, None, None, imgs)
    x = emb[0].to(dec.dtype).contiguous()
    S = x.shape[0]
    K = 64
    dec.prefill(x, all_logits=False, keep_cache=True, max_len=S + max(HISTORIES) + K)
    res = {"S": S}
    for n in (64, 2048):
        params = ops.logits_process_params(cfg.vocab_size, dev, **processors(cfg.vocab_size, n))
        ms = {"plain": [], "processed": []}
        for _ in range(3):
            for name, p in (("plain", None), ("processed", params)):
                dec.kv_len = S + n                       # K/V rows past the prefill are not meaningful: timing only
                dec.decode_graph_begin(3, None, p)
                dec._decode_hist[:n].copy_(history(n))
                dec._decode_log[1].fill_(n - 1)          # the history holds n ids when the first replay runs
                ms[name].append(events_us(lambda: dec.decode_graph_run(K), K) / 1e3)
        res[f"n{n}_graph_ms_per_token_device"] = {k: [round(v, 4) for v in vs] for k, vs in ms.items()}
        res[f"n{n}_added_us_per_token"] = round((min(ms["processed"]) - min(ms["plain"])) * 1e3, 1)
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("microbench_processors needs a CUDA device")
    out = {"card": card(), "kernel": kernel_times()}
    if "--no-model" not in sys.argv:
        out["config2"] = model_times()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

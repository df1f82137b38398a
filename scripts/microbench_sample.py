"""Cost of token sampling on the GPU.  Prints one JSON line with the card's name, power limit and SM clock.

1. vl2_sample_token at V = 32000 (Mistral) and 152064 (Qwen2) with CUDA events over 500 launches captured in one CUDA
   graph, for (top_k 50, top_p 0.9), (top_k 0, top_p 0.9), (top_k 1) and mm_infer's defaults (T 0.2, top_p 0.9, top_k 50);
   against torch's warp_logits + softmax + multinomial on the same row (eager, no host synchronisation inside the loop).
2. Config 2 (Mistral-7B, 16 frames@336, S = 1776) on the synthetic checkpoint bench.py builds:
   - ms per token of the sampled decode graph replayed back to back, against the greedy graph, alternated in one run;
   - generate() wall time per token, do_sample=True at mm_infer's defaults against greedy, from two runs that differ only
     in max_new_tokens (the prefill cancels);
   - the same for the host-sampled loop generate(do_sample=True) ran before the device sampler: one greedy-graph replay,
     then sampling.sample_token on its logits (.item()), then the token written back into the graph's token buffer.
Usage: python scripts/microbench_sample.py [--no-model]"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from videollama2_b200 import ops, sampling

dev = torch.device("cuda:0")
DEFAULTS = dict(temperature=0.2, top_k=50, top_p=0.9)
CASES = {"k50_p0.9": dict(temperature=1.0, top_k=50, top_p=0.9), "k0_p0.9": dict(temperature=1.0, top_k=0, top_p=0.9),
         "k1": dict(temperature=1.0, top_k=1, top_p=1.0), "mm_infer_defaults": DEFAULTS}


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


def kernel_times():
    res = {}
    n = 500
    for V in (32000, 152064):
        row = (torch.randn(V, generator=torch.Generator().manual_seed(V)) * 3.0).to(dev)
        counter = torch.zeros((1,), dtype=torch.int64, device=dev)
        out = torch.zeros((n,), dtype=torch.int64, device=dev)
        for name, c in CASES.items():
            params = ops.sampling_params(c["temperature"], c["top_k"], c["top_p"], 1234, dev)
            for i in range(3):
                ops.sample_token(row, params, counter, i, out[i:i + 1])
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for i in range(n):
                    ops.sample_token(row, params, counter, i, out[i:i + 1])
            g.replay()
            us = min(events_us(g.replay, n) for _ in range(3))
            gen = torch.Generator(device=dev).manual_seed(0)

            def torch_path():
                for _ in range(n):
                    p = sampling.warp_logits(row[None], c["temperature"], c["top_k"], c["top_p"]).softmax(-1)
                    torch.multinomial(p, 1, generator=gen)
            torch_path()
            us_torch = min(events_us(torch_path, n) for _ in range(3))
            res[f"V{V}_{name}"] = {"kernel_us": round(us, 2), "torch_us": round(us_torch, 2)}
    return res


def model_times():
    import bench
    from videollama2_b200 import presets
    from videollama2_b200.model import VLLMs
    cfg = presets.make_config(presets.MISTRAL_7B, bench.FRAMES)
    S = presets.flops(cfg, bench.FRAMES, bench.PROMPT)["S"]
    sd = presets.synthetic_state_dict(cfg, dev, threads=max(1, min(16, os.cpu_count() or 8)))
    model = VLLMs[cfg.model_type].from_state_dict(cfg, sd, device=dev)
    del sd
    torch.cuda.empty_cache()
    model.enable_cuda_graphs(True)
    px, ids = presets.synthetic_inputs(cfg, bench.FRAMES, bench.PROMPT)
    imgs = [(px.to(cfg.storage_dtype).to(dev), "video")]
    mask = torch.ones_like(ids, dtype=torch.bool)
    dec = model.get_model().decoder
    res = {"S": S}

    def gen(n, sample):
        kw = dict(do_sample=True, generator=torch.Generator().manual_seed(n), **DEFAULTS) if sample else dict(do_sample=False)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=n, use_cache=True, eos_token_id=None, **kw)
        torch.cuda.synchronize()
        assert out.shape[1] == n
        return (time.perf_counter() - t) * 1e3

    _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, mask, None, None, imgs)
    x = emb[0].to(dec.dtype).contiguous()

    def host_loop(n):
        """generate(do_sample=True)'s former graphed loop, token for token."""
        g = torch.Generator(device=dev).manual_seed(n)
        torch.cuda.synchronize()
        t = time.perf_counter()
        model.encode_images_or_videos(imgs)            # the same front end generate() runs
        logits, _ = dec.prefill(x, all_logits=False, keep_cache=True, max_len=S + n)
        tok = sampling.sample_token(logits[0], DEFAULTS["temperature"], DEFAULTS["top_p"], DEFAULTS["top_k"], g)
        dec.decode_graph_begin(tok)
        for _ in range(n - 1):
            tok_dev = dec.decode_graph_step()
            tok = sampling.sample_token(dec.decode_graph_logits[0], DEFAULTS["temperature"], DEFAULTS["top_p"],
                                        DEFAULTS["top_k"], g)
            tok_dev.fill_(tok)
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3

    short, long_ = 8, 72
    for f in (lambda n: gen(n, False), lambda n: gen(n, True), host_loop):
        f(long_)                                        # sizes the KV cache, captures the graphs
    per = {"greedy": [], "sampled": [], "host_sampled": []}
    for _ in range(3):
        for name, f in (("greedy", lambda n: gen(n, False)), ("sampled", lambda n: gen(n, True)), ("host_sampled", host_loop)):
            a, b = f(short), f(long_)
            per[name].append((b - a) / (long_ - short))
    res["generate_ms_per_token"] = {k: [round(v, 3) for v in vs] for k, vs in per.items()}

    # the two graphs replayed back to back on the device, alternated
    K = 64
    params = ops.sampling_params(DEFAULTS["temperature"], DEFAULTS["top_k"], DEFAULTS["top_p"], 99, dev)
    dev_ms = {"greedy": [], "sampled": []}
    for _ in range(3):
        for name, sp in (("greedy", None), ("sampled", params)):
            dec.kv_len = S
            dec.decode_graph_begin(3, sp)
            dev_ms[name].append(events_us(lambda: dec.decode_graph_run(K), K) / 1e3)
    res["graph_ms_per_token_device"] = {k: [round(v, 4) for v in vs] for k, vs in dev_ms.items()}
    g, s = min(dev_ms["greedy"]), min(dev_ms["sampled"])
    res["sampled_over_greedy_graph"] = round(s / g, 4)
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("microbench_sample needs a CUDA device")
    out = {"card": card(), "kernel": kernel_times()}
    if "--no-model" not in sys.argv:
        out["config2"] = model_times()
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""One rank of the tensor-parallel logits-processor check (launched by torchrun, NCCL): generate() with processors on the
tensor-parallel decoder, greedy and sampled, must return the same ids on every rank (every rank processes the identical
gathered logits with identical tables)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    from helpers import engine_config
    from oracle import synth
    from videollama2_b200.model import VLLMs
    ok, msgs = True, []
    for name in ("tiny", "tiny_qwen2"):
        cfg = synth.CONFIGS[name]
        if cfg.llm.kv_heads % world or cfg.llm.heads % world:
            continue
        sd = synth.state_dict(cfg)
        ec = engine_config(cfg)
        tp = VLLMs[ec.model_type].from_state_dict(ec, sd, device=dev, tp_group=True)
        px, ids = synth.inputs(cfg)
        images = [(px.to(dev), "video")]
        plain = tp.generate(ids, images=images, max_new_tokens=8, do_sample=False, eos_token_id=None)[0].tolist()
        proc = dict(max_new_tokens=12, repetition_penalty=1.3, no_repeat_ngram_size=2, bad_words_ids=[[plain[2]]],
                    suppress_tokens=[plain[3]], min_new_tokens=4, eos_token_id=plain[0])
        for sample in (False, True):
            torch.manual_seed(100 + rank)                     # every rank's default generator differs
            kw = dict(proc, do_sample=True, temperature=1.5, top_p=0.95) if sample else dict(proc, do_sample=False)
            got = tp.generate(ids, images=images, **kw)
            out = torch.full((1, kw["max_new_tokens"]), -1, dtype=torch.long, device=dev)   # ranks may stop apart
            out[:, :got.shape[1]] = got
            allo = [torch.empty_like(out) for _ in range(world)]
            dist.all_gather(allo, out)
            if not all(torch.equal(t, out) for t in allo):
                ok = False
                msgs.append(f"ranks disagree on the processed ids ({name}, sampled={sample})")
    if msgs:
        print(f"RANK{rank} " + "; ".join(msgs), flush=True)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    print(f"RANK{rank} {'OK' if int(flag.item()) == 1 else 'FAIL'}", flush=True)
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()

"""One rank of the tensor-parallel scores check (launched by torchrun, NCCL): generate(return_dict_in_generate=True,
output_scores=True, output_logits=True) on the tensor-parallel decoder must return identical sequences, scores and logits
on every rank, greedy with processors and sampled."""
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
        base = dict(max_new_tokens=6, eos_token_id=None, return_dict_in_generate=True, output_scores=True,
                    output_logits=True)
        for kw in (dict(repetition_penalty=1.3), dict(do_sample=True, temperature=1.5, top_p=0.95)):
            torch.manual_seed(100 + rank)                     # every rank's default generator differs
            out = tp.generate(ids, images=images, **base, **kw)
            tensors = [out.sequences.to(torch.float32)] + [torch.cat(out.scores, 0), torch.cat(out.logits, 0)]
            for what, t in zip(("sequences", "scores", "logits"), tensors):
                allo = [torch.empty_like(t) for _ in range(world)]
                dist.all_gather(allo, t.contiguous())
                if not all(torch.equal(a.view(torch.int32), t.view(torch.int32)) for a in allo):
                    ok = False
                    msgs.append(f"ranks disagree on {what} ({name}, {kw})")
    if msgs:
        print(f"RANK{rank} " + "; ".join(msgs), flush=True)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    print(f"RANK{rank} {'OK' if int(flag.item()) == 1 else 'FAIL'}", flush=True)
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()

"""One rank of the tensor-parallel sampling check (launched by torchrun, NCCL): generate(do_sample=True) on the
tensor-parallel decoder must return the same ids on every rank even when each rank's torch generators were seeded
differently before the call (the decoder broadcasts the first rank's sampling seed)."""
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
        kw = dict(max_new_tokens=8, do_sample=True, temperature=1.5, top_p=0.95, eos_token_id=None)
        for use_gen in (False, True):
            torch.manual_seed(100 + rank)                     # every rank's default generator differs
            gen = torch.Generator(device=dev).manual_seed(200 + rank) if use_gen else None
            out = tp.generate(ids, images=images, generator=gen, **kw)
            allo = [torch.empty_like(out) for _ in range(world)]
            dist.all_gather(allo, out)
            if not all(torch.equal(t, out) for t in allo):
                ok = False
                msgs.append(f"ranks disagree on the sampled ids ({name}, generator={use_gen})")
    if msgs:
        print(f"RANK{rank} " + "; ".join(msgs), flush=True)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    print(f"RANK{rank} {'OK' if int(flag.item()) == 1 else 'FAIL'}", flush=True)
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()

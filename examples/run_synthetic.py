"""End-to-end walk through the engine with random weights (no checkpoints or tokenizers are available offline):
decoded uint8 frames -> device preprocessing -> tower -> connector -> splice -> prefill -> graph-replayed decode.

    python examples/run_synthetic.py [--model mistral7b|qwen2_7b|qwen2_7b_v21] [--frames 16] [--new-tokens 32]

Needs one H100 and ~20 GB of HBM (the 7B decoder in bf16).  The token ids are meaningless (random weights); the point is
the call sequence a user of the reference's `mm_infer` would make, and the timings."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from videollama2_b200 import mm_utils, presets
from videollama2_b200.model import VLLMs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="mistral7b", choices=["mistral7b", "qwen2_7b", "qwen2_7b_v21"])
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--new-tokens", type=int, default=32)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    llm = presets.MISTRAL_7B if args.model == "mistral7b" else presets.QWEN2_7B
    if args.model == "qwen2_7b_v21":
        cfg = presets.make_config(llm, args.frames, "stc_connector_v35", presets.SIGLIP_SO400M_384)
    else:
        cfg = presets.make_config(llm, args.frames)
    model = VLLMs[cfg.model_type].from_state_dict(cfg, presets.random_state_dict(cfg, dev), device=dev)
    model.enable_cuda_graphs(True)          # tower / connector / prefill stages and the per-token decode step as graphs
    model.enable_vision_cache(2)            # a second question about the same video skips the vision stages

    # "decoded video": what decord / PIL hand out, uint8 [T, H, W, 3]
    raw = torch.randint(0, 256, (args.frames, 720, 1280, 3), dtype=torch.uint8)
    processor = model.get_vision_tower().image_processor
    ids = torch.randint(3, cfg.vocab_size, (1, 64))
    ids[0, 4] = -201                         # the <video> placeholder tokenizer_multimodal_token would insert

    for question in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pixels = mm_utils.process_video(raw, processor, aspect_ratio="pad", num_frames=args.frames, device=dev)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        out = model.generate(ids, images=[(pixels, "video")], max_new_tokens=args.new_tokens, do_sample=False,
                             eos_token_id=None)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        print(f"question {question}: preprocess {1e3 * (t1 - t0):.1f} ms, prefill + {out.shape[1]} tokens "
              f"{1e3 * (t2 - t1):.1f} ms (vision cache hits so far: {model.vision_cache_hits}); first ids {out[0, :8].tolist()}")


if __name__ == "__main__":
    main()

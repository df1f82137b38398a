"""Regenerate tests/golden/live_reference.pt: what the tests that used to call the REAL reference live compare against
(tokenizer_multimodal_token, mm_infer, KeywordsStoppingCriteria and the tiny-config forward / STC connector), computed by
the reference classes on CPU (oracle/ref_loader.py).  Needs the reference checkout; the tests only read the file."""
import importlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "live_reference.pt")

TOKENIZER_PROMPTS_EXTRA = [("a <video> b <video> c", "<video>"), ("", "<video>")]
STC_SEED = 1234


def main():
    from oracle import mm_infer_ref, ref_loader, synth
    from oracle.make_golden import PROMPTS, ToyTokenizer
    ref_loader.load()
    ref_mm = importlib.import_module("videollama2.mm_utils")
    out = {}
    tok = ToyTokenizer()
    out["tokenizer"] = [(p, t, ref_mm.tokenizer_multimodal_token(p, tok, t)) for p, t in PROMPTS + TOKENIZER_PROMPTS_EXTRA]
    instruct, modal, mtype, kw = mm_infer_ref.CASES[0]
    text, call = mm_infer_ref.run_reference(instruct, modal, mtype, torch.zeros((2, 3, 4, 4)), **kw)
    out["mm_infer"] = {"text": text, "input_ids": mm_infer_ref.summarise(call)["input_ids"]}
    from test_host_logic import _DecodingToyTokenizer, keyword_cases
    dtok = _DecodingToyTokenizer()
    prompt = torch.zeros(1, 2, dtype=torch.long)
    ref = ref_mm.KeywordsStoppingCriteria(["hello"], dtok, prompt)
    out["keywords_decoded"] = [bool(ref(c, None)) for c in keyword_cases(dtok)]
    cfg = synth.CONFIGS["tiny"]
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    m = ref_loader.build_reference_model(cfg, torch.float32, sd)
    with torch.no_grad():
        res = m(input_ids=ids, attention_mask=torch.ones_like(ids), images=[(px.float(), "video")])
        stc_in = torch.randn(2, 4, 16, cfg.vision.hidden, generator=torch.Generator().manual_seed(STC_SEED))
        stc_ref = m.get_model().mm_projector(stc_in)
    out["tiny"] = {"logits": res.logits[0].clone(), "stc_in": stc_in, "stc": stc_ref.clone(),
                   "state_dict_shapes": {k: tuple(v.shape) for k, v in m.state_dict().items()}}
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")


if __name__ == "__main__":
    main()

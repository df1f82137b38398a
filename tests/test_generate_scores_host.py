"""Host side of generate(output_scores / output_logits): the statement sampling.expected_scores against a tiny randomly
initialised HF MistralForCausalLM's generate(return_dict_in_generate=True) (transformers 5.5), compute_transition_scores
against HF's, the output object, the record block and the C-ABI's argument checks.  No GPU needed."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from videollama2_b200 import sampling

transformers = pytest.importorskip("transformers")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, MAX_NEW, EMB = 9, 24, 32
PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=2)


@pytest.fixture(scope="module")
def hf():
    from transformers import MistralConfig, MistralForCausalLM
    torch.manual_seed(0)
    cfg = MistralConfig(vocab_size=48, hidden_size=EMB, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, max_position_embeddings=256, sliding_window=None)
    return MistralForCausalLM(cfg).eval(), torch.randn(1, S, EMB)


def bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def hf_generate(model, emb, **kw):
    with torch.no_grad():
        return model.generate(inputs_embeds=emb, max_new_tokens=MAX_NEW, return_dict_in_generate=True,
                              output_scores=True, output_logits=True, eos_token_id=None, pad_token_id=0, **kw)


def test_greedy_scores_are_the_processed_logits(hf):
    """Every step's scores row is process_logits(logits row, ids before it) bit for bit, with the history of new ids
    only and min_length turned into min_length - S new tokens."""
    model, emb = hf
    plain = hf_generate(model, emb, do_sample=False)
    eos = int(plain.sequences[0, 1])
    proc = dict(PROC, bad_words_ids=[[int(plain.sequences[0, 2])]], suppress_tokens=[int(plain.sequences[0, 4])])
    with torch.no_grad():
        out = model.generate(inputs_embeds=emb, max_new_tokens=MAX_NEW, return_dict_in_generate=True,
                             output_scores=True, output_logits=True, do_sample=False, min_length=S + 6,
                             eos_token_id=eos, pad_token_id=eos, **proc)
    seq = out.sequences[0].tolist()
    assert len(out.scores) == len(out.logits) == len(seq) > 6
    changed = 0
    for n in range(len(seq)):
        want = sampling.expected_scores(out.logits[n][0], seq[:n], min_new_tokens=6, eos_token_ids=(eos,), **proc)
        assert torch.equal(bits(want), bits(out.scores[n][0])), n
        assert int(torch.argmax(want)) == seq[n]
        changed += int(not torch.equal(want, out.logits[n][0]))
    assert changed == len(seq)                       # every step had something processed


def top_p_margin(row, T, k, p):
    """Distance of the closest kept token's mass-above from top_p (fp64), as in the sampler tests."""
    s = (row / T).double().numpy()
    keep = np.ones_like(s, dtype=bool) if not 0 < k < s.size else s >= np.sort(s)[s.size - k]
    w = np.where(keep & np.isfinite(s), np.exp(s - s.max()), 0.0)
    vals, inv = np.unique(s, return_inverse=True)
    above = np.concatenate([np.cumsum(np.bincount(inv, weights=w)[::-1])[::-1][1:], [0.0]])[inv] / w.sum()
    return np.abs(above[keep] - p).min()


@pytest.mark.parametrize("T,k,p", [(0.7, 10, 0.9), (1.5, 0, 0.8), (1.0, 5, 1.0), (0.3, 20, 0.5)])
def test_sampled_scores_are_the_warped_rows(hf, T, k, p):
    """do_sample with processors and temperature / top-k / top-p: scores[n] is the processed row's fp32(l / T) where
    the kernel's rule keeps the token and -inf elsewhere, on every step whose top-p boundary has no near tie."""
    model, emb = hf
    torch.manual_seed(5)
    out = hf_generate(model, emb, do_sample=True, temperature=T, top_k=k, top_p=p, **PROC)
    seq = out.sequences[0].tolist()
    checked = 0
    for n in range(len(seq)):
        proc_row = sampling.process_logits(out.logits[n][0], seq[:n], **PROC)
        if p < 1.0 and top_p_margin(proc_row, T, k, p) < 1e-5:
            continue
        want = sampling.expected_scores(out.logits[n][0], seq[:n], do_sample=True, temperature=T, top_k=k, top_p=p,
                                        **PROC)
        assert torch.equal(bits(want), bits(out.scores[n][0])), n
        assert torch.isfinite(want[seq[n]])
        checked += 1
    assert checked >= len(seq) // 2


@pytest.mark.parametrize("normalize", [False, True])
def test_compute_transition_scores_equals_hf(hf, normalize):
    from videollama2_b200.model.videollama2_mistral import Videollama2MistralForCausalLM
    model, emb = hf
    torch.manual_seed(7)
    out = hf_generate(model, emb, do_sample=True, temperature=0.8, top_k=12, top_p=0.9, num_return_sequences=2)
    engine = object.__new__(Videollama2MistralForCausalLM)
    for scores in (out.scores, out.logits):
        want = model.compute_transition_scores(out.sequences, scores, normalize_logits=normalize)
        got = engine.compute_transition_scores(out.sequences, scores, normalize_logits=normalize)
        assert got.shape == (2, len(scores)) and torch.equal(got, want)
        # a prompt in front of the new ids: only the last len(scores) columns are read
        front = torch.cat([torch.full((2, 5), 3), out.sequences], 1)
        assert torch.equal(engine.compute_transition_scores(front, scores, normalize_logits=normalize), want)
    with pytest.raises(NotImplementedError):
        engine.compute_transition_scores(out.sequences, out.scores, beam_indices=torch.zeros((2, 3), dtype=torch.long))


def test_generate_output_access():
    from videollama2_b200.model.videollama2_mistral import GenerateOutput
    seq, sc = torch.tensor([[4, 5]]), (torch.zeros(1, 8), torch.ones(1, 8))
    out = GenerateOutput(seq, scores=sc)
    assert out["sequences"] is seq and out.scores is sc and out["logits"] is None and out.logits is None
    assert out.attentions is None and out.hidden_states is None and out.past_key_values is None
    assert out.keys() == ["sequences", "scores"] and out[0] is seq and out[1] is sc and out.to_tuple() == (seq, sc)


def test_record_block_layout_and_validation():
    from videollama2_b200 import _lib, ops
    assert ctypes.sizeof(_lib.ScoreRecordParams) == 32 and ops.SCORE_RECORD_WORDS == 4
    s, lg = torch.empty((5, 100)), torch.empty((5, 100))
    blk = _lib.ScoreRecordParams.from_buffer_copy(ops.score_record_params(100, 5, s, lg).numpy().tobytes())
    assert (blk.scores, blk.logits, blk.capacity, blk.V) == (s.data_ptr(), lg.data_ptr(), 5, 100)
    blk = _lib.ScoreRecordParams.from_buffer_copy(ops.score_record_params(100, 5, logits=lg).numpy().tobytes())
    assert blk.scores is None and blk.logits == lg.data_ptr()
    assert ops.score_record_params(100, 0, device="cpu").numel() == 4
    for args in [(100, -1), (0, 5), (262145, 5), (100, 5, torch.empty((4, 100))), (100, 5, None, torch.empty((5, 99))),
                 (100, 5, torch.empty((5, 100), dtype=torch.float64)), (100, 5, torch.empty((100, 5)).t())]:
        with pytest.raises(ValueError):
            ops.score_record_params(*args)


def test_struct_size_matches_the_header(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    from videollama2_b200 import _lib
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vl2.h"\nint main(void) { printf("%zu %zu %zu %zu", '
                   'sizeof(vl2_score_record_params), offsetof(vl2_score_record_params, capacity), '
                   'offsetof(vl2_score_record_params, V), (size_t)VL2_RECORD_SCORES); return 0; }\n')
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(tmp_path / "sz")],
                   check=True)
    got = subprocess.run([str(tmp_path / "sz")], capture_output=True, text=True, check=True).stdout.split()
    R = _lib.ScoreRecordParams
    assert [int(x) for x in got] == [ctypes.sizeof(R), R.capacity.offset, R.V.offset, _lib.RECORD_SCORES]


@pytest.fixture(scope="module")
def lib():
    from videollama2_b200 import _lib, build
    build.build()
    return _lib.load()


A16, MIS = 4096, 4100          # fake device addresses: aligned, and 4 bytes off (never dereferenced)


@pytest.mark.parametrize("args,code", [
    ((A16, 0, A16, 0, A16, 0, None), -1),
    ((A16, -3, A16, 1, A16, 0, None), -1),
    ((A16, 262145, A16, 0, A16, 0, None), -1),
    ((A16, 32000, A16, 2, A16, 0, None), -1),
    ((A16, 32000, A16, -1, A16, 0, None), -1),
    ((None, 32000, A16, 0, A16, 0, None), -3),
    ((A16, 32000, None, 0, A16, 0, None), -3),
    ((A16, 32000, A16, 1, None, 0, None), -3),
    ((A16 + 2, 32000, A16, 0, A16, 0, None), -3),
    ((A16, 32000, MIS, 0, A16, 0, None), -3),
    ((A16, 32000, A16, 1, MIS, 0, None), -3),
])
def test_record_row_argument_validation_without_gpu(lib, args, code):
    """V and `which` are checked before any CUDA call (VL2_E_BADSHAPE), then null and misaligned pointers
    (VL2_E_BADALIGN)."""
    assert lib.vl2_record_row(*args) == code, lib.vl2_last_error()


@pytest.mark.parametrize("args,code", [
    ((A16, 0, A16, A16, 0, A16, A16, None), -1),
    ((A16, 262145, A16, A16, 0, A16, A16, None), -1),
    ((None, 32000, A16, A16, 0, A16, A16, None), -3),
    ((A16, 32000, None, A16, 0, A16, A16, None), -3),
    ((A16, 32000, A16, None, 0, A16, A16, None), -3),
    ((A16, 32000, A16, A16, 0, None, A16, None), -3),
    ((A16, 32000, A16, A16, 0, A16, None, None), -3),
    ((A16 + 2, 32000, A16, A16, 0, A16, A16, None), -3),
    ((A16, 32000, MIS, A16, 0, A16, A16, None), -3),
    ((A16, 32000, A16, MIS, 0, A16, A16, None), -3),
    ((A16, 32000, A16, A16, 0, MIS, A16, None), -3),
    ((A16, 32000, A16, A16, 0, A16, MIS, None), -3),
])
def test_scored_sampler_argument_validation_without_gpu(lib, args, code):
    assert lib.vl2_sample_token_scored(*args) == code, lib.vl2_last_error()


def test_expected_scores_keeps_negative_zero_and_drops_to_minus_inf():
    row = torch.tensor([-0.0, 2.0, 1.0, -math.inf, 0.5])
    assert torch.equal(bits(sampling.expected_scores(row, [])), bits(row))
    got = sampling.expected_scores(row, [], do_sample=True, temperature=2.0, top_k=4, top_p=1.0)
    assert torch.equal(bits(got), bits(torch.tensor([-0.0, 1.0, 0.5, -math.inf, 0.25])))
    got = sampling.expected_scores(row, [], do_sample=True, temperature=2.0, top_k=3, top_p=1.0)
    assert torch.equal(bits(got), bits(torch.tensor([-math.inf, 1.0, 0.5, -math.inf, 0.25])))

"""Host side of the device logits processors (vl2_process_logits): the torch statement sampling.process_logits against
HF's processor classes, a tiny HF MistralForCausalLM's generate(inputs_embeds=...) against a loop through that statement,
the parameter validation and the C-ABI's argument checks.  No GPU needed."""
import ctypes
import math

import pytest
import torch

from videollama2_b200 import sampling

transformers = pytest.importorskip("transformers")
from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,  # noqa: E402
                                                    NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                    RepetitionPenaltyLogitsProcessor, SuppressTokensLogitsProcessor)


def hf_process(row, history, repetition_penalty=None, no_repeat_ngram_size=None, min_new_tokens=0, eos_token_ids=(),
               bad_words_ids=None, suppress_tokens=None):
    """HF's processors in the order GenerationMixin._get_logits_processor adds them, on a [1, V] row."""
    procs = LogitsProcessorList()
    if repetition_penalty is not None:
        procs.append(RepetitionPenaltyLogitsProcessor(float(repetition_penalty)))
    if no_repeat_ngram_size is not None:
        procs.append(NoRepeatNGramLogitsProcessor(no_repeat_ngram_size))
    if bad_words_ids is not None:
        procs.append(NoBadWordsLogitsProcessor(bad_words_ids, list(eos_token_ids)))
    if min_new_tokens > 0 and eos_token_ids:
        procs.append(MinNewTokensLengthLogitsProcessor(0, min_new_tokens, list(eos_token_ids)))
    if suppress_tokens is not None:
        procs.append(SuppressTokensLogitsProcessor(suppress_tokens))
    ids = torch.tensor([list(history)], dtype=torch.long).reshape(1, -1)
    return procs(ids, row.reshape(1, -1).clone())[0]


def same(a, b):
    """== with identical +-inf / NaN positions (HF's bad-word bias turns -0.0 into +0.0: zeros compare by value)."""
    return bool(torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.isposinf(a), torch.isposinf(b)) and
                torch.equal(torch.isneginf(a), torch.isneginf(b)) and (a[torch.isfinite(a)] == b[torch.isfinite(b)]).all())


def random_case(g, V, n, ids_range):
    row = torch.randn(V, generator=g) * 3.0
    row[torch.randint(0, V, (V // 10,), generator=g)] = 0.0
    row[torch.randint(0, V, (V // 10,), generator=g)] = -0.0
    history = torch.randint(0, ids_range, (n,), generator=g).tolist()      # a small id range: repeats and n-gram hits
    return row, history


SETTINGS = [
    dict(repetition_penalty=0.8), dict(repetition_penalty=1.05), dict(repetition_penalty=1.3),
    dict(no_repeat_ngram_size=1), dict(no_repeat_ngram_size=2), dict(no_repeat_ngram_size=3), dict(no_repeat_ngram_size=7),
    dict(bad_words_ids=[[3], [5, 6], [1, 2, 4], [0, 0, 0, 1], [9]], eos_token_ids=(9,)),
    dict(min_new_tokens=6, eos_token_ids=(2, 7)),
    dict(suppress_tokens=[0, 4, 13]),
    dict(repetition_penalty=1.3, no_repeat_ngram_size=2, bad_words_ids=[[3], [1, 2], [2, 2, 5]], min_new_tokens=4,
         eos_token_ids=(5,), suppress_tokens=[6]),
]


@pytest.mark.parametrize("setting", SETTINGS, ids=lambda s: "+".join(s))
def test_host_statement_equals_hf_processors(setting):
    """Random rows (with +-0.0) and histories of 0 to 40 ids drawn from a few ids, so that repeats, n-gram and bad-word
    matches occur; n-gram sizes up to longer than the history."""
    g = torch.Generator().manual_seed(len(str(setting)))
    hits = 0
    for V in (16, 1000):
        for n in list(range(0, 8)) + [15, 40]:
            for rep in range(4):
                row, hist = random_case(g, V, n, 6)
                if rep == 3:                   # a periodic history: every n-gram size finds a repeat once n allows
                    hist = (hist[:5] * n)[:n]
                want = hf_process(row, hist, **setting)
                got = sampling.process_logits(row, hist, **setting)
                assert same(got, want), (V, hist, setting)
                hits += int(not torch.equal(torch.isneginf(got), torch.isneginf(row)) or not torch.equal(got, row))
    assert hits > 0                        # the setting changed some rows


def test_host_statement_penalty_is_fp32_and_once_per_token():
    row = torch.tensor([3.0, -3.0, 1e-30, -0.0, 7.0])
    got = sampling.process_logits(row, [0, 1, 0, 0, 2, 3], repetition_penalty=1.1)
    p = torch.tensor(1.1, dtype=torch.float32)
    assert got.tolist() == [(row[0] / p).item(), (row[1] * p).item(), (row[2] / p).item(), -0.0, 7.0]
    # a +inf score that is banned ends as -inf (HF's additive bias would leave NaN there)
    assert sampling.process_logits(torch.tensor([math.inf, 0.0]), [], suppress_tokens=[0]).tolist() == [-math.inf, 0.0]


def test_bad_words_need_the_whole_sequence_length_of_history():
    """HF applies a sequence of L ids only once the history holds at least L ids, even if the prefix already matched."""
    row = torch.zeros(10)
    assert not torch.isinf(sampling.process_logits(row, [1], bad_words_ids=[[1, 4]])).any()
    assert torch.isneginf(sampling.process_logits(row, [1, 1], bad_words_ids=[[1, 4]]))[4]
    assert not torch.isinf(hf_process(row, [1], bad_words_ids=[[1, 4]])).any()


def test_parameter_validation():
    from videollama2_b200 import ops
    bad = [dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=math.nan),
           dict(no_repeat_ngram_size=0), dict(no_repeat_ngram_size=-2), dict(no_repeat_ngram_size=1.5),
           dict(min_new_tokens=-1), dict(bad_words_ids=[]), dict(bad_words_ids=[3]), dict(bad_words_ids=[[]]),
           dict(bad_words_ids=[[1, -2]]), dict(bad_words_ids=[[1, 100]]), dict(bad_words_ids=[[1.0]]),
           dict(suppress_tokens=[100]), dict(suppress_tokens=[-1]), dict(min_new_tokens=2, eos_token_ids=(100,))]
    for kw in bad:
        with pytest.raises(ValueError):
            ops.logits_process_params(100, "cpu", **kw)
        with pytest.raises(ValueError):
            sampling.process_logits(torch.zeros(100), [], **kw)
    ops.logits_process_params(100, "cpu", eos_token_ids=(100,))       # EOS ids only matter with a minimum length


def test_parameter_block_layout():
    from videollama2_b200 import _lib, ops
    assert ctypes.sizeof(_lib.LogitsProcessParams) == 64 and ops.PROCESS_HEADER_WORDS == 8
    buf = ops.logits_process_params(100, "cpu", repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5,
                                    eos_token_ids=(2, 9), bad_words_ids=[[5], [2], [7, 8, 9]], suppress_tokens=[11])
    hdr = _lib.LogitsProcessParams.from_buffer_copy(buf[:8].numpy().tobytes())
    assert hdr.repetition_penalty == torch.tensor(1.3).item() and hdr.no_repeat_ngram_size == 3
    assert (hdr.min_new_tokens, hdr.n_eos, hdr.n_suppress, hdr.n_bad) == (5, 2, 1, 2)    # [2] is an EOS id: dropped
    base = buf.data_ptr()
    word = lambda p: buf[(p - base) // 8].item()
    assert (word(hdr.eos_ids), word(hdr.eos_ids + 8), word(hdr.suppress_ids)) == (2, 9, 11)
    assert [word(hdr.bad_offsets + 8 * i) for i in range(3)] == [0, 1, 4]
    assert [word(hdr.bad_ids + 8 * i) for i in range(4)] == [5, 7, 8, 9]
    off = _lib.LogitsProcessParams.from_buffer_copy(ops.logits_process_params(100, "cpu")[:8].numpy().tobytes())
    assert (off.repetition_penalty, off.no_repeat_ngram_size, off.min_new_tokens, off.n_eos, off.n_bad) == (1.0, 0, 0, 0, 0)


def test_generate_processors_follows_hf_conditions():
    gp = sampling.generate_processors
    assert gp({}, {2}, 50, 100) is None
    assert gp(dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0), {2}, 50, 100) is None
    assert gp(dict(min_new_tokens=5), set(), 50, 100) is None                        # no EOS: nothing to hold back
    assert gp(dict(min_length=40), {2}, 50, 100) is None                             # 40 - 50 < 0 new tokens
    assert gp(dict(min_length=57), {2}, 50, 100)["min_new_tokens"] == 7              # min_length counts the prompt
    assert gp(dict(min_length=57, min_new_tokens=3), {2}, 50, 100)["min_new_tokens"] == 3
    assert gp(dict(no_repeat_ngram_size=-1, repetition_penalty=1.2), {2}, 50, 100)["no_repeat_ngram_size"] is None
    cfg = gp(dict(bad_words_ids=[[2], [4, 5]], suppress_tokens=[1]), {2}, 50, 100)
    assert cfg["bad_words_ids"] == ((4, 5),) and cfg["suppress_tokens"] == (1,)
    cfg = gp(dict(bad_words_ids=[[2]], repetition_penalty=1.2), {2}, 50, 100)     # only an EOS: bad words off
    assert cfg["bad_words_ids"] is None
    from videollama2_b200 import ops
    ops.logits_process_params(100, "cpu", **cfg)                  # the normalised settings are valid input again
    with pytest.raises(ValueError):
        gp(dict(repetition_penalty=0.0), {2}, 50, 100)


def test_tiny_hf_mistral_generate_equals_host_loop():
    """generate(inputs_embeds=...) of a randomly initialised HF MistralForCausalLM with processors, greedy and without a
    KV cache, gives the ids of a loop over the same model's logits through process_logits with the history of new ids
    only and min_length turned into min_length - S new tokens."""
    from transformers import MistralConfig, MistralForCausalLM
    torch.manual_seed(0)
    cfg = MistralConfig(vocab_size=48, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, max_position_embeddings=256, sliding_window=None)
    model = MistralForCausalLM(cfg).eval()
    S, max_new = 9, 24
    emb = torch.randn(1, S, 32)

    def host_loop(eos, min_new, **proc):
        out = []
        with torch.no_grad():
            x = emb
            for n in range(max_new):
                logits = model(inputs_embeds=x).logits[0, -1]
                row = sampling.process_logits(logits, out, min_new_tokens=min_new, eos_token_ids=(eos,), **proc)
                tok = int(torch.argmax(row))
                out.append(tok)
                if tok == eos:
                    break
                x = torch.cat([x, model.get_input_embeddings()(torch.tensor([[tok]]))], 1)
        return out

    plain = host_loop(-1, 0)
    eos = plain[1]                       # an EOS that greedy decoding would emit at once: the minimum must hold it back
    proc = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, bad_words_ids=[[plain[2]], [plain[0], plain[3]]],
                suppress_tokens=[plain[4]])
    want = host_loop(eos, 6, **proc)
    assert len(want) > 2 and plain[2] not in want and plain[4] not in want
    with torch.no_grad():
        got = model.generate(inputs_embeds=emb, do_sample=False, max_new_tokens=max_new, min_length=S + 6,
                             eos_token_id=eos, pad_token_id=eos, use_cache=False, **proc)
    assert got[0].tolist()[:len(want)] == want
    assert eos not in want[:6]


@pytest.fixture(scope="module")
def lib():
    from videollama2_b200 import _lib, build
    build.build()
    return _lib.load()


A16, MIS = 4096, 4100          # fake device addresses: aligned, and 4 bytes off (never dereferenced)


@pytest.mark.parametrize("args,code", [
    ((A16, 0, A16, A16, A16, 0, None), -1),
    ((A16, -3, A16, A16, A16, 0, None), -1),
    ((A16, 262145, A16, A16, A16, 0, None), -1),
    ((None, 32000, A16, A16, A16, 0, None), -3),
    ((A16, 32000, None, A16, A16, 0, None), -3),
    ((A16, 32000, A16, None, A16, 0, None), -3),
    ((A16, 32000, A16, A16, None, 0, None), -3),
    ((A16 + 2, 32000, A16, A16, A16, 0, None), -3),
    ((A16, 32000, MIS, A16, A16, 0, None), -3),
    ((A16, 32000, A16, MIS, A16, 0, None), -3),
    ((A16, 32000, A16, A16, MIS, 0, None), -3),
])
def test_process_logits_argument_validation_without_gpu(lib, args, code):
    """V and the pointers are checked before any CUDA call: VL2_E_BADSHAPE outside 1..262144, VL2_E_BADALIGN for null or
    misaligned pointers."""
    assert lib.vl2_process_logits(*args) == code, lib.vl2_last_error()

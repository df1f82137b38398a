"""Token selection for `generate(do_sample=True, ...)`: the logits warpers HF's GenerationMixin applies for the arguments
the reference's mm_infer passes (videollama2/__init__.py:93-110: temperature, top_p; top_k stays at GenerationConfig's
default 50) — temperature -> top-k -> top-p -> softmax -> multinomial.

generate() draws with the vl2_sample_token kernel (ops.sample_token).  This module is the host statement of what it
computes: `warp_logits` / `sample_token` in plain torch (HF's semantics, any device), and `kernel_kept` /
`kernel_token` / `philox4x32_10`, the kernel's own rule in numpy (fp64), which the tests predict its tokens with.

HF's logits processors (repetition penalty, n-gram and bad-word bans, minimum new tokens, suppressed tokens) run before
the warpers, on the device in vl2_process_logits (ops.process_logits); `process_logits` here is their host statement.
`expected_scores` states the row generate(output_scores=True) records for each step."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch


def warp_logits(logits: torch.Tensor, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0,
                min_tokens_to_keep: int = 1) -> torch.Tensor:
    """[..., V] fp32 scores after TemperatureLogitsWarper, TopKLogitsWarper and TopPLogitsWarper (HF semantics: top-p
    removes the low-probability tail whose cumulative probability is <= 1 - top_p, always keeping the best token)."""
    scores = logits.float()
    if temperature is not None and temperature != 1.0:
        if temperature <= 0:
            raise ValueError("temperature must be positive when sampling")
        scores = scores / temperature
    if top_k is not None and top_k > 0:
        k = min(max(int(top_k), min_tokens_to_keep), scores.shape[-1])
        kth = torch.topk(scores, k, dim=-1).values[..., -1, None]
        scores = scores.masked_fill(scores < kth, float("-inf"))
    if top_p is not None and top_p < 1.0:
        sorted_scores, sorted_idx = torch.sort(scores, descending=False, dim=-1)
        cum = sorted_scores.softmax(dim=-1).cumsum(dim=-1)
        remove = cum <= (1.0 - top_p)
        remove[..., -min_tokens_to_keep:] = False
        scores = scores.masked_fill(remove.scatter(-1, sorted_idx, remove), float("-inf"))
    return scores


def sample_token(logits: torch.Tensor, temperature: float, top_p: float, top_k: int = 50,
                 generator: Optional[torch.Generator] = None) -> int:
    probs = warp_logits(logits.reshape(1, -1), temperature, top_k, top_p).softmax(dim=-1)
    return int(torch.multinomial(probs, 1, generator=generator).item())


# ---- logits processors: applied before the warpers (and before the arg-max when greedy) ----------------------------
def _ids(name: str, xs, V: int) -> tuple:
    out = []
    for t in xs:
        if isinstance(t, bool) or not isinstance(t, (int, np.integer)) or not 0 <= int(t) < V:
            raise ValueError(f"{name}: {t!r} is not a token id in [0, {V})")
        out.append(int(t))
    return tuple(out)


def check_processors(V: int, repetition_penalty=None, no_repeat_ngram_size=None, min_new_tokens: int = 0,
                     eos_token_ids=(), bad_words_ids=None, suppress_tokens=None) -> dict:
    """Processor settings in the form process_logits and ops.logits_process_params take them.  None (or 0 / () where
    that is the default) turns a processor off.  Raises ValueError for what HF's processor classes reject: a penalty
    <= 0, an n-gram size <= 0, a negative minimum, bad_words_ids that is not a non-empty list of non-empty id lists, and
    any id outside [0, V).  Bad-word sequences that are a single EOS id are dropped, as NoBadWordsLogitsProcessor drops
    them."""
    V = int(V)
    if V < 1:
        raise ValueError(f"vocabulary size {V} < 1")
    pen = None
    if repetition_penalty is not None:
        pen = float(repetition_penalty)
        if not pen > 0:
            raise ValueError(f"repetition_penalty has to be strictly positive, got {repetition_penalty}")
    N = None
    if no_repeat_ngram_size is not None:
        if isinstance(no_repeat_ngram_size, bool) or not isinstance(no_repeat_ngram_size, (int, np.integer)) \
                or no_repeat_ngram_size <= 0:
            raise ValueError(f"no_repeat_ngram_size has to be a strictly positive integer, got {no_repeat_ngram_size}")
        N = int(no_repeat_ngram_size)
    if isinstance(min_new_tokens, bool) or not isinstance(min_new_tokens, (int, np.integer)) or min_new_tokens < 0:
        raise ValueError(f"min_new_tokens has to be a non-negative integer, got {min_new_tokens}")
    eos_token_ids = tuple(eos_token_ids or ())
    eos = _ids("eos_token_id", eos_token_ids, V) if min_new_tokens > 0 else tuple(int(t) for t in eos_token_ids)
    bad = None                     # off, also when every sequence was a single EOS id
    if bad_words_ids is not None:
        if not isinstance(bad_words_ids, (list, tuple)) or len(bad_words_ids) == 0 or \
                any(not isinstance(s, (list, tuple)) or len(s) == 0 for s in bad_words_ids):
            raise ValueError(f"bad_words_ids has to be a non-empty list of non-empty lists of token ids, got {bad_words_ids!r}")
        bad = tuple(_ids("bad_words_ids", s, V) for s in bad_words_ids)
        bad = tuple(s for s in bad if not (len(s) == 1 and s[0] in eos)) or None
    return dict(repetition_penalty=pen, no_repeat_ngram_size=N, min_new_tokens=int(min_new_tokens),
                eos_token_ids=eos, bad_words_ids=bad, suppress_tokens=_ids("suppress_tokens", suppress_tokens or (), V))


def generate_processors(kwargs: dict, eos_ids, prompt_len: int, V: int) -> Optional[dict]:
    """The processors HF's GenerationMixin.generate(inputs_embeds=...) adds for these generate() kwargs, as
    check_processors settings, or None when it adds none that changes a score.  Follows transformers 5.5
    (generation/utils.py: _get_logits_processor, _prepare_generated_length); that the reference's pinned 4.40 does the
    same bad-word and minimum-length arithmetic is unverified.
     - repetition_penalty: on unless None or 1.0; no_repeat_ngram_size: on when > 0.
     - min_new_tokens wins over min_length; min_length alone becomes max(min_length - prompt_len, 0) new tokens, where
       prompt_len is the spliced inputs_embeds length, visual tokens included.  Both need an EOS id.
     - bad_words_ids and suppress_tokens: on when given."""
    pen = kwargs.get("repetition_penalty")
    pen = None if pen is None or pen == 1.0 else pen
    N = kwargs.get("no_repeat_ngram_size")
    N = N if N is not None and not isinstance(N, bool) and N > 0 else None
    mnt, ml = kwargs.get("min_new_tokens"), kwargs.get("min_length")
    min_new = int(mnt) if mnt is not None else (int(ml) - int(prompt_len) if ml is not None else 0)
    eos = tuple(sorted(int(e) for e in eos_ids))
    min_new = max(min_new, 0) if eos else 0
    bad, sup = kwargs.get("bad_words_ids"), kwargs.get("suppress_tokens")
    if pen is None and N is None and min_new == 0 and bad is None and not sup:
        return None
    return check_processors(V, pen, N, min_new, eos, bad, sup)


def process_logits(logits: torch.Tensor, history, repetition_penalty=None, no_repeat_ngram_size=None,
                   min_new_tokens: int = 0, eos_token_ids=(), bad_words_ids=None, suppress_tokens=None) -> torch.Tensor:
    """The scores HF's processors leave for one logits row [V] (returned as a new fp32 CPU row) after the generated ids
    `history` - RepetitionPenalty -> NoRepeatNGram -> NoBadWords -> MinNewTokensLength -> SuppressTokens, in HF's
    order, with check_processors' settings.  The statement vl2_process_logits is tested against:
     - the penalty: each distinct history token's s becomes s < 0 ? s * p : s / p in fp32 (p rounded to fp32; IEEE
       division, as torch computes `scores / penalty` on the CPU);
     - every ban is -inf, applied after the penalty.  HF adds -inf as a bias for bad words, which turns -0.0 scores into
       +0.0 and a banned +inf into NaN; this statement (and the kernel) keep -0.0 and ban +inf to -inf.
    A row whose every token is banned is all -inf: the arg-max and the sampling kernel then both pick token 0 (the first
    index of the maximum)."""
    s = logits.detach().float().reshape(-1).cpu().clone()
    cfg = check_processors(s.numel(), repetition_penalty, no_repeat_ngram_size, min_new_tokens, eos_token_ids,
                           bad_words_ids, suppress_tokens)
    h = [int(t) for t in (history.tolist() if isinstance(history, torch.Tensor) else history)]
    n = len(h)
    p = cfg["repetition_penalty"]
    if p is not None and n:
        idx = torch.tensor(sorted(set(h)), dtype=torch.long)
        v, pf = s[idx], torch.tensor(p, dtype=torch.float32)
        s[idx] = torch.where(v < 0, v * pf, v / pf)
    ban = set()
    N = cfg["no_repeat_ngram_size"]
    if N is not None and n >= N:
        tail = h[n - N + 1:]
        ban.update(h[i + N - 1] for i in range(n - N + 1) if h[i:i + N - 1] == tail)
    for seq in cfg["bad_words_ids"] or ():
        L = len(seq)
        if L == 1 or (n >= L and tuple(h[n - L + 1:]) == seq[:-1]):
            ban.add(seq[-1])
    if n < cfg["min_new_tokens"]:
        ban.update(cfg["eos_token_ids"])
    ban.update(cfg["suppress_tokens"])
    if ban:
        s[torch.tensor(sorted(ban), dtype=torch.long)] = float("-inf")
    return s


_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)
_MASK32 = 0xFFFFFFFF


def philox4x32_10(counter, key) -> tuple:
    """Random123's Philox4x32-10: four 32-bit counter words and two 32-bit key words -> four 32-bit words."""
    c0, c1, c2, c3 = (int(x) & _MASK32 for x in counter)
    k0, k1 = (int(x) & _MASK32 for x in key)
    for _ in range(10):
        p0, p1 = _PHILOX_M[0] * c0, _PHILOX_M[1] * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & _MASK32, p1 & _MASK32, ((p0 >> 32) ^ c3 ^ k1) & _MASK32, p0 & _MASK32
        k0, k1 = (k0 + _PHILOX_W[0]) & _MASK32, (k1 + _PHILOX_W[1]) & _MASK32
    return c0, c1, c2, c3


def kernel_u(seed: int, n: int) -> float:
    """The kernel's uniform draw for counter n: (x0 >> 8) * 2^-24 of Philox(counter (n_lo, n_hi, 0, 0), key = seed)."""
    seed, n = int(seed) & (2 ** 64 - 1), int(n) & (2 ** 64 - 1)
    x0 = philox4x32_10((n, n >> 32, 0, 0), (seed, seed >> 32))[0]
    return (x0 >> 8) * 2.0 ** -24


def kernel_kept(logits, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0):
    """The kernel's kept set and the fp64 weights exp(s - max) of a logits row [V]: (kept bool [V], weights [V]).
    s = fp32(l / T); top-k keeps s >= the k-th largest s (counting duplicates); top-p then drops a token when the
    probability mass of the kept tokens strictly above it is >= top_p, so a tie group is kept or dropped whole."""
    s = (torch.as_tensor(logits, dtype=torch.float32).reshape(-1).cpu() / float(temperature)).numpy().astype(np.float64)
    s = np.where(np.isnan(s), -np.inf, s)
    V = s.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        keep = s >= np.sort(s)[V - int(top_k)]
    mx = s.max()
    with np.errstate(invalid="ignore", over="ignore"):
        w = np.where(s == -np.inf, 0.0, np.where(s == mx, 1.0, np.exp(s - mx)))
    if top_p < 1.0:
        wk = np.where(keep, w, 0.0)
        vals, inv = np.unique(s, return_inverse=True)            # ascending unique scores
        group = np.bincount(inv.reshape(-1), weights=wk, minlength=vals.shape[0])
        above = np.concatenate([np.cumsum(group[::-1])[::-1][1:], [0.0]])   # mass of the strictly larger groups
        keep &= above[inv.reshape(-1)] / wk.sum() < top_p
    return keep, w


def kernel_cdf(logits, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0) -> np.ndarray:
    """fp64 index-order CDF of the kept tokens (the kernel's inverse CDF runs over it)."""
    keep, w = kernel_kept(logits, temperature, top_k, top_p)
    wk = np.where(keep, w, 0.0)
    return np.cumsum(wk) / wk.sum()


def kernel_token(logits, temperature: float, top_k: int, top_p: float, seed: int, n: int) -> int:
    """The token vl2_sample_token draws with counter n: the first index whose CDF exceeds u."""
    return int(np.searchsorted(kernel_cdf(logits, temperature, top_k, top_p), kernel_u(seed, n), side="right"))


def expected_scores(logits: torch.Tensor, history, do_sample: bool = False, temperature: float = 1.0, top_k: int = 0,
                    top_p: float = 1.0, **processors) -> torch.Tensor:
    """The `scores` row generate(output_scores=True) records for one raw logits row [V] (a new fp32 CPU row), after the
    generated ids `history`: process_logits(logits, history, **processors); when sampling, that row's fp32(l / T) where
    kernel_kept keeps the token and -inf elsewhere - HF's warped row, with the kernel's whole-tie-group top-p rule."""
    s = process_logits(logits, history, **processors)
    if not do_sample:
        return s
    keep, _ = kernel_kept(s, temperature, top_k, top_p)
    return torch.where(torch.from_numpy(keep), s / float(temperature), torch.tensor(float("-inf")))


def draw_seed(generator: Optional[torch.Generator] = None) -> int:
    """The per-generate() seed of the sampling kernel: one 63-bit draw from `generator`, or from torch's default CPU
    generator (so torch.manual_seed makes runs reproducible)."""
    if generator is None:
        return int(torch.randint(0, 2 ** 63 - 1, (1,)).item())
    return int(torch.randint(0, 2 ** 63 - 1, (1,), generator=generator, device=generator.device).item())

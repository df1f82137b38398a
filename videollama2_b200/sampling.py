"""Token selection for `generate(do_sample=True, ...)`: the logits warpers HF's GenerationMixin applies for the arguments
the reference's mm_infer passes (videollama2/__init__.py:93-110: temperature, top_p; top_k stays at GenerationConfig's
default 50) — temperature -> top-k -> top-p -> softmax -> multinomial.

generate() draws with the vl2_sample_token kernel (ops.sample_token).  This module is the host statement of what it
computes: `warp_logits` / `sample_token` in plain torch (HF's semantics, any device), and `kernel_kept` /
`kernel_token` / `philox4x32_10`, the kernel's own rule in numpy (fp64), which the tests predict its tokens with."""
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


def draw_seed(generator: Optional[torch.Generator] = None) -> int:
    """The per-generate() seed of the sampling kernel: one 63-bit draw from `generator`, or from torch's default CPU
    generator (so torch.manual_seed makes runs reproducible)."""
    if generator is None:
        return int(torch.randint(0, 2 ** 63 - 1, (1,)).item())
    return int(torch.randint(0, 2 ** 63 - 1, (1,), generator=generator, device=generator.device).item())

"""Float64 reference of the sampling kernels (eagle_b200/csrc/sampling.cu) and of how far their fp32 arithmetic may move
a decision.

What the kernels compute, for one logits row l of the model dtype (T = round to the model dtype, to nearest even):

    lt  = T(fp32(l) / fp32(temperature))    TemperatureLogitsWarper, in the model dtype (skipped at temperature 1)
    max = max lt,  z = sum exp(lt - max)
    top-p: keep the value classes v with mass(lt <= v) > (1 - top_p) z; ties at the threshold are all kept, and so is the
           row maximum (min_tokens_to_keep = 1)
    top-k: keep lt >= the k-th largest kept value, counted with multiplicity
    thr = max(thr_p, thr_k),  sum = sum_{lt >= thr} exp(lt - max),  p(v) = lt_v >= thr ? exp(lt_v - max) / sum : 0

and a token is drawn by inverse CDF over the eligible tokens (kept, and not rejected by the posterior) in index order.

This module evaluates the same in float64.  Where fp32 rounding can move a decision, it returns every admissible outcome:

* Top-p: the kernel sums exp(lt - max) per thread over ceil(V / 1024) serial terms, then over a 1024-way tree (10 levels),
  with expf within 2 ulp: its masses are within delta = (ceil(V / 1024) + 12) u z of the float64 ones (u = 2^-24).  A value
  class whose cumulative mass lies within delta of the cut may or may not pass it, so every class whose mass may pass the
  cut while the class below it may not is an admissible threshold.  A class of zero mass (-inf) never passes a positive cut.
* Top-k counts tokens: exact.
* Inverse CDF: sample_commit_kernel adds ceil(V / 1024) weights per thread, then the 1024 per-thread partials serially,
  so its running sum is within (ceil(V / 1024) + 1024 + 12) u S of the float64 CDF (S = total eligible weight).  Token t is
  admissible for the uniform x when it is eligible and C(t - 1) <= x S + d, C(t) >= x S - d.
* Posterior: orc.evaluate_posterior_sampling, run on rows already masked by the kernel's thresholds, with every uniform
  recording the acceptance probability it is compared with.  The kernel forms that probability as p / (1 - removed) in
  fp32; a uniform within 2e-5 relative of it (widened by 1 / (1 - removed) for the cancellation in 1 - removed) is
  flagged ambiguous.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import eagle_oracle as orc

U = 2.0 ** -24
CHUNKS = 1024  # threads of row_softmax_stats_kernel / sample_commit_kernel
AMBIGUOUS_REL = 2e-5


def per_thread(V: int) -> int:
    """Tokens per thread of sample_commit_kernel's contiguous split (and the serial terms of the stats' strided sums)."""
    return (V + CHUNKS - 1) // CHUNKS


def stats_delta_rel(V: int) -> float:
    """Bound on the relative error of the stats kernel's sums (of z, of a cumulative mass, of sum)."""
    return (per_thread(V) + 12) * U


def cdf_delta_rel(V: int) -> float:
    """Bound on the relative error of sample_commit_kernel's running sum against the float64 CDF."""
    return (per_thread(V) + CHUNKS + 12) * U


def top_p_on(top_p: float) -> bool:
    """The kernel's (and HF's) condition, evaluated on the fp32 value the kernel receives."""
    p = np.float32(top_p)
    return bool(p >= np.float32(1e-8) and p < np.float32(1.0))


def temperature_warp(logits: torch.Tensor, temperature: float) -> torch.Tensor:
    """lt = T(fp32(l) / fp32(temperature)) as float64; logits [..., V] in bf16 / fp16.  numpy's fp32 division is the IEEE
    one (__fdiv_rn); the fp32 -> model dtype cast is a single round to nearest even."""
    if temperature == 1.0:
        return logits.double()
    q = torch.from_numpy(logits.float().numpy() / np.float32(temperature))
    return q.to(logits.dtype).double()


class RowRef:
    """Softmax statistics of one temperature-warped row (float64 [V]) for any (top_p, top_k)."""

    def __init__(self, lt: torch.Tensor):
        self.lt = lt
        self.V = lt.numel()
        self.max = float(lt.max())
        self.e = torch.exp(lt - self.max)  # exp(-inf) = 0
        self.z = float(self.e.sum())
        self.delta = stats_delta_rel(self.V) * self.z
        # distinct values ascending (-0.0 and 0.0 compare equal: one class, as in the kernel's `lt >= thr`)
        self.vals, inv = torch.unique(lt, sorted=True, return_inverse=True)
        self.mass = torch.zeros(len(self.vals), dtype=torch.float64).index_add_(0, inv, self.e)
        self.count = torch.zeros(len(self.vals), dtype=torch.int64).index_add_(0, inv, torch.ones_like(inv))
        self.cum = torch.cumsum(self.mass, 0)                                   # mass(lt <= v_j)
        self.tail = torch.flip(torch.cumsum(torch.flip(self.mass, [0]), 0), [0])  # mass(lt >= v_j)
        self.count_ge = torch.flip(torch.cumsum(torch.flip(self.count, [0]), 0), [0])

    def top_p_thresholds(self, top_p: float) -> list[float]:
        """Admissible top-p thresholds (-inf when top-p is off), ascending."""
        if not top_p_on(top_p):
            return [-math.inf]
        cut = (1.0 - float(np.float32(top_p))) * self.z
        below = torch.cat((torch.zeros(1, dtype=torch.float64), self.cum[:-1]))
        ok = (self.cum > max(cut - self.delta, 0.0)) & (below <= cut + self.delta)
        return [float(v) for v in self.vals[ok]]

    def kth(self, top_k: int) -> float:
        """The top_k-th largest value with multiplicity (-inf when top-k is off)."""
        if not 0 < top_k < self.V:
            return -math.inf
        j = int(torch.nonzero(self.count_ge >= top_k)[-1])
        return float(self.vals[j])

    def admissible(self, top_p: float, top_k: int) -> dict[float, float]:
        """thr -> sum, for every threshold the kernel may produce."""
        kth = self.kth(top_k)
        out = {}
        for tp in self.top_p_thresholds(top_p):
            thr = max(tp, kth)
            out[thr] = self.sum_at(thr)
        return out

    def sum_at(self, thr: float) -> float:
        if thr == -math.inf:
            return self.z
        j = int(torch.searchsorted(self.vals, torch.tensor([thr], dtype=torch.float64))[0])
        return float(self.tail[j])

    def weights(self, thr: float, rejected=()) -> torch.Tensor:
        """Eligible weights exp(lt - max) under the threshold, rejected tokens zeroed."""
        w = torch.where(self.lt >= thr, self.e, torch.zeros_like(self.e))
        if len(rejected):
            w[torch.as_tensor(list(rejected), dtype=torch.long)] = 0.0
        return w


def bracket(weights: torch.Tensor, x: float, d_rel: float) -> torch.Tensor:
    """Tokens the inverse CDF may return for the uniform x: eligible (weight > 0) with C(t - 1) <= x S + d and
    C(t) >= x S - d, C the float64 CDF in index order, S its total, d = d_rel S.  Boolean mask [V]."""
    c = torch.cumsum(weights, 0)
    s = float(c[-1])
    d = d_rel * s
    return (weights > 0) & (c - weights <= x * s + d) & (c >= x * s - d)


class _Draw(float):
    """A uniform that records the acceptance probability orc.evaluate_posterior_sampling compares it with
    (`r <= gtp[xi] / 1.0`), with the fraction of its level's mass not yet rejected (1 - removed)."""

    def __new__(cls, value, level):
        self = super().__new__(cls, value)
        self.level = level
        return self

    def __le__(self, other):
        p, lv = float(other), self.level
        lv["log"].append((float(self), p, lv["keep"], lv["n"]))
        if not float(self) <= p:
            lv["keep"] *= 1.0 - p  # gtp[xi] = 0; gtp /= gtp.sum(): the next probabilities are relative to what is left
        return float(self) <= p


def posterior(lt_nodes: torch.Tensor, thr: torch.Tensor, candidates: torch.Tensor, retrieve: torch.Tensor, uniforms, draws=None):
    """utils.py:375-415 on the kernel's warped rows.

    lt_nodes: float64 [T][V] temperature-warped logits of the tree nodes; thr: [T] the stats kernel's thresholds;
    candidates / retrieve: [n_leaf][max_depth] tokens / node ids (-1 padding).  Returns best, accept_length, the bonus
    distribution (float64 [V], zero where ineligible), the number of uniforms the kernel draws (candidates tried + 1 for
    the bonus), and whether any decision was ambiguous.  draws: an optional list that receives one (level, accepted) pair
    per candidate decision, level counted from 0 for each warped row the walk evaluates."""
    masked = torch.where(lt_nodes >= thr.double()[:, None], lt_nodes, torch.full_like(lt_nodes, -math.inf))
    level = {"log": [], "keep": 1.0, "n": -1}
    it = iter(uniforms)

    def warp(row):  # called once per level, before the level's comparisons (and once more for a fresh bonus row)
        level["keep"] = 1.0
        level["n"] += 1
        return row

    best, acc, sample_p = orc.evaluate_posterior_sampling(masked[retrieve.clamp(min=0)], candidates, warp,
                                                          rand=lambda: _Draw(next(it), level))
    if draws is not None:
        draws.extend((lv, u <= a) for u, a, keep, lv in level["log"])
    ambiguous = any(abs(u - a) <= AMBIGUOUS_REL * a / max(keep, 1e-30) for u, a, keep, _ in level["log"])
    return int(best), int(acc), sample_p.double(), len(level["log"]) + 1, ambiguous

"""CPU checks of the sampling kernels' test reference (tests/sampling_ref.py): on tie-free rows it keeps what the oracle's
warpers (HF's TemperatureLogitsWarper -> TopPLogitsWarper -> TopKLogitsWarper) keep, and hand-built rows pin down the
kernels' documented policies for ties, +-0.0, -inf entries and min_tokens_to_keep.  No GPU."""
import math

import numpy as np
import pytest
import torch

from oracle import eagle_oracle as orc
from tests import sampling_ref as sr

TEMPERATURES = [1.0, 0.7, 1.3, 0.05]
TOP_PS = [0.0, 1e-8, 2e-8, 3e-8, 0.02, 0.6, 0.9, 0.999, 1.0]
INF = math.inf


def _tie_free_row(V, dtype, seed):
    """V distinct model-dtype values (no two equal after any of the temperatures either: checked by the caller)."""
    g = torch.Generator().manual_seed(seed)
    pool = torch.unique((torch.randn(8 * V, generator=g) * 2.0).to(dtype).float())
    return pool[torch.randperm(pool.numel(), generator=g)[:V]].to(dtype)


def _row(*xs, dtype=torch.bfloat16):
    return torch.tensor(xs, dtype=torch.float32).to(dtype)


def _kept(ref, thr):
    return ref.lt >= thr


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_temperature_is_the_model_dtype_division(dtype):
    """T(fp32(l) / fp32(t)): what torch computes for a model-dtype tensor divided by a Python float."""
    x = (torch.randn(4096, generator=torch.Generator().manual_seed(1)) * 4).to(dtype)
    for t in TEMPERATURES:
        assert torch.equal(sr.temperature_warp(x, t), (x / t).double())


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_kept_set_matches_the_oracle_warpers_on_tie_free_rows(dtype, seed):
    V = 300
    x = _tie_free_row(V, dtype, 10 + seed)
    for t in TEMPERATURES:
        lt = sr.temperature_warp(x, t)
        if torch.unique(lt).numel() != V:
            continue  # the division merged two values: not a tie-free row at this temperature
        ref = sr.RowRef(lt)
        for top_p in TOP_PS:
            for top_k in (0, 1, 10, 50, V - 1, V, V + 5):
                # the oracle gets the warped row in fp32 (the engine's softmax precision); its own temperature step is the
                # division checked above
                want = torch.isfinite(orc.warp_logits(lt.float()[None], 1.0, top_p, top_k)[0])
                adm = ref.admissible(top_p, top_k)
                assert any(torch.equal(_kept(ref, thr), want) for thr in adm), (t, top_p, top_k, sorted(adm))
                for thr, s in adm.items():
                    assert s == pytest.approx(float(ref.e[_kept(ref, thr)].sum()), rel=1e-12)


def test_top_p_keeps_every_tie_at_the_threshold():
    # masses 1 : 3 x e : e^2; the cut at 0.5 z lands inside the class of the three 1.0s
    ref = sr.RowRef(_row(0, 1, 1, 1, 2).double())
    assert float(ref.cum[0]) < 0.5 * ref.z < float(ref.cum[1])
    assert ref.top_p_thresholds(0.5) == [1.0]
    assert int(_kept(ref, 1.0).sum()) == 4


def test_top_k_counts_ties_with_multiplicity_and_keeps_them_all():
    ref = sr.RowRef(_row(3, 1, 2, 2, 2, 0).double())
    assert ref.kth(1) == 3.0 and ref.kth(2) == 2.0 and ref.kth(4) == 2.0 and ref.kth(5) == 1.0
    assert list(ref.admissible(0.0, 2)) == [2.0]
    assert int(_kept(ref, 2.0).sum()) == 4  # top_k = 2 keeps the whole tie class at the 2nd value


def test_signed_zeros_are_one_class():
    ref = sr.RowRef(_row(1, 0.0, -0.0, -0.0, 0.0, -1, -2).double())
    assert ref.vals.numel() == 4
    thr = ref.kth(2)
    assert thr == 0.0
    assert int(_kept(ref, thr).sum()) == 5  # 1 and all four zeros, whichever sign the kernel's threshold carries
    assert int(_kept(ref, -0.0).sum()) == int(_kept(ref, 0.0).sum())
    # top-p with the cut inside the zero class: the threshold is that class
    cut_frac = float(ref.cum[1] + ref.cum[2]) / 2 / ref.z
    assert ref.top_p_thresholds(1 - cut_frac) == [0.0]


def test_minus_inf_entries_carry_no_mass_and_count_for_top_k():
    ref = sr.RowRef(_row(0.5, -INF, 1.5, -INF, -INF, 1.0).double())
    assert float(ref.mass[0]) == 0.0
    # -inf is never a top-p threshold (a positive cut), even with top_p just below 1
    for p in (0.999, 0.9999999):
        assert -INF not in ref.top_p_thresholds(p)
    # the 5th largest is -inf: top-k keeps everything top-p kept, and sum is z
    assert ref.admissible(0.0, 5) == {-INF: ref.z}
    assert ref.admissible(0.0, 3) == {0.5: ref.z}


def test_min_tokens_to_keep_keeps_the_maximum():
    for p in (1e-8, 2e-8, 3e-8):
        # 1 - p rounds to 1 in fp32 for the first two; the maximum is kept regardless
        assert (np.float32(1.0) - np.float32(p) == np.float32(1.0)) == (p < 2.0 ** -25)
        ref = sr.RowRef(_row(0.25, 3, -1, 2, 1).double())
        assert ref.top_p_thresholds(p) == [3.0]
        # an all-equal row keeps every token
        flat = sr.RowRef(_row(*([0.5] * 7)).double())
        assert flat.top_p_thresholds(p) == [0.5] and int(_kept(flat, 0.5).sum()) == 7


def test_top_p_boundary_within_delta_admits_both_neighbours():
    # mass(lt <= 0) = 1 / z exactly at the cut: either side of it is admissible, nothing further
    ref = sr.RowRef(_row(0, 1, 2, 3).double())
    top_p = 1 - float(ref.cum[0]) / ref.z
    assert ref.top_p_thresholds(float(np.float32(top_p))) == [0.0, 1.0]
    # well inside a class: one threshold
    assert ref.top_p_thresholds(0.75) == [2.0]


def test_bracket_edges_first_and_last_eligible():
    w = torch.tensor([0.0, 1.0, 0.0, 2.0, 1.0, 0.0], dtype=torch.float64)
    assert torch.nonzero(sr.bracket(w, 0.0, 0.0)).flatten().tolist() == [1]
    assert torch.nonzero(sr.bracket(w, 1.0, 0.0)).flatten().tolist() == [4]
    # x S = 1 on the edge between tokens 1 and 3: both bracket it, the zero-weight token 2 between them never
    assert torch.nonzero(sr.bracket(w, 0.25, 0.0)).flatten().tolist() == [1, 3]
    assert torch.nonzero(sr.bracket(w, 0.5, 0.0)).flatten().tolist() == [3]
    # rejected tokens are ineligible
    ref = sr.RowRef(torch.tensor([0.0, 1.0, 2.0], dtype=torch.float64))
    assert torch.nonzero(sr.bracket(ref.weights(-INF, rejected=[2]), 1.0, 0.0)).flatten().tolist() == [1]


def test_posterior_counts_draws_and_flags_ambiguous_decisions():
    # root 0 with children 1, 2, 3 (tokens 2, 1, 2: the second 2 is a duplicate, skipped without a draw)
    lt = torch.log(torch.tensor([[0.1, 0.2, 0.3, 0.4]] * 4, dtype=torch.float64))
    retrieve = torch.tensor([[0, 1], [0, 2], [0, 3]])
    cands = torch.tensor([[7, 2], [7, 1], [7, 2]])
    thr = torch.full((4,), -INF)
    best, acc, p, used, amb = sr.posterior(lt, thr, cands, retrieve, [1.0, 1.0, 0.5])
    assert (best, acc, used, amb) == (0, 0, 3, False)
    assert p[1] == 0.0 and p[2] == 0.0 and p[0] == pytest.approx(0.2) and p[3] == pytest.approx(0.8)
    # accepted at the first candidate: one draw plus the bonus
    best, acc, p, used, amb = sr.posterior(lt, thr, cands, retrieve, [0.1, 0.5])
    assert (best, acc, used, amb) == (0, 1, 2, False)
    # u within 2e-5 of p(2) = 0.3: ambiguous; after rejecting token 2 (0.3), p(1) = 0.2 / 0.7 with the widened window
    assert sr.posterior(lt, thr, cands, retrieve, [0.3 * (1 + 1e-5), 0.5])[4]
    assert sr.posterior(lt, thr, cands, retrieve, [0.9, 0.2 / 0.7 * (1 + 2.5e-5), 0.5])[4]
    assert not sr.posterior(lt, thr, cands, retrieve, [0.9, 0.2 / 0.7 * (1 + 3e-5), 0.5])[4]

"""Draft-tree growth in isolation on the H100: tree_seed_kernel + tree_expand_kernel (eb200_k_tree_grow) on host-fed
per-level top-k tables against the plain torch reference of tests/tree_growth_ref.py (held to the CPU oracle by
tests/test_tree_growth_cpu.py), then growth -> tree_finalize -> sampling posterior as one chain.

Everything here is an integer, or a float that both sides round at the same single point (one add in fp32, one rounding
to the model dtype), so every comparison is torch.equal -- there is no tolerance.  The geometries are the ones where the
second 64-bit word of the ancestor masks is in use: more than 64 draft columns (depth * top_k up to 128)."""
import ctypes as C

import pytest
import torch

from oracle import eagle_oracle as orc
from tests import tree_growth_ref as ref
from tests.test_kernels_gpu import DT, check, lib, ptr  # noqa: F401  (lib is a fixture)

pytestmark = pytest.mark.gpu


def run_grow(lib, dtype, topk_p, topk_i, d2t, k, depth, last_row=0):
    pool, rows = k + depth * k * k, 1 + depth * k
    assert topk_p.shape == (rows, k) and topk_p.dtype == torch.float32 and topk_i.dtype == torch.int32
    out = dict(scores=torch.full((pool,), float("nan")), tokens=torch.full((pool,), -7, dtype=torch.int32),
               parents=torch.full((rows,), -7, dtype=torch.int32),
               ids=torch.full((depth + 1, k), -7, dtype=torch.int32), src=torch.full((depth + 1, k), -7, dtype=torch.int32),
               cs=torch.full((depth + 1, k), -7, dtype=torch.int32), fscores=torch.full((depth + 1, k), float("nan")),
               mask=torch.full((depth + 1, k, 2), -7, dtype=torch.int64))
    check(lib, lib.eb200_k_tree_grow(DT[dtype], ptr(topk_p.contiguous()), ptr(topk_i.contiguous()), ptr(d2t), 0 if d2t is None else d2t.numel(),
                                     k, depth, last_row, ptr(out["scores"]), ptr(out["tokens"]), ptr(out["parents"]), ptr(out["ids"]),
                                     ptr(out["src"]), ptr(out["cs"]), ptr(out["fscores"]), ptr(out["mask"])))
    return out


def same(got, want, what):
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        raise AssertionError(f"{what}: {bad.shape[0]} of {got.numel()} differ; first at {bad[:6].tolist()}: "
                             f"got {got[got != want][:6].tolist()} want {want[got != want][:6].tolist()}")


def compare(got, want, k, depth, what):
    w_scores, w_tokens, w_parents, levels = want
    same(got["parents"].long(), w_parents, f"{what}: pool parents")
    same(got["tokens"].long(), w_tokens, f"{what}: pool tokens")
    same(got["scores"], w_scores, f"{what}: pool scores")
    for slot, lv in enumerate(levels):  # slot 0 = after the seed, slot l + 1 = after level l
        where = f"{what}: frontier after " + ("the seed" if slot == 0 else f"level {slot - 1}")
        same(got["cs"][slot].long(), lv["cs"], where + " front_cs")
        same(got["src"][slot].long(), lv["src"], where + " front_src")
        same(got["ids"][slot].long(), lv["ids"], where + " front_ids")
        same(got["fscores"][slot], lv["scores"], where + " front_scores")
        same(got["mask"][slot], ref.pack_mask(lv["mask"]), where + f" front_mask words ({(slot + 1) * k} columns)")


def strided_d2t(draft_vocab=512, vocab=2048):
    from eagle_b200.synthetic import make_d2t
    return make_d2t(vocab, draft_vocab)[0]


GEOMETRIES = [
    (10, 6),   # 60 columns: word 0 only
    (10, 7),   # EaModel.from_pretrained's default: 70 columns, the last level's own columns are 60..69
    (16, 8),   # exactly 128 columns: bit 63 of word 1, and k * k = 256 candidates
    (9, 14),   # 126 columns, the deepest tree eb200_create accepts
    (8, 8),    # level 7's own columns are exactly 64..71: slot 0 of a level is bit 0 of word 1
    (13, 5),   # level 3's own columns 52..64 straddle the word boundary
    (1, 14), (1, 1),  # degenerate: a chain / a single node
    (17, 7), (32, 4),  # top_k above the engine's 16 that tree_expand still claims: 119 columns / 1024 candidates, 128 columns
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_d2t", [True, False], ids=["d2t", "nomap"])
@pytest.mark.parametrize("k,depth", GEOMETRIES)
def test_growth_is_bit_exact(lib, k, depth, with_d2t, dtype):
    topk_p, topk_i = ref.make_tables(k, depth, dtype, seed=1000 * k + depth)
    d2t = strided_d2t() if with_d2t else None
    last_row = 5 if with_d2t else 0
    want = ref.grow(topk_p, topk_i, d2t, k, depth, dtype, last_row)
    got = run_grow(lib, dtype, topk_p, topk_i, d2t, k, depth, last_row)
    compare(got, want, k, depth, f"k={k} depth={depth}")
    if depth * k > 64:  # the case is only worth its name if word 1 is really populated
        assert int((got["mask"][-1, :, 1] != 0).sum()) == k


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_natural_ties_occur_in_the_random_tables(dtype):
    """The random cases above are meant to contain equal cumulative scores (model-dtype log-probs on a coarse grid): make sure
    they do, otherwise the tie policy would only be covered by the hand-made cases below."""
    k, depth = 10, 7
    topk_p, topk_i = ref.make_tables(k, depth, dtype, seed=1000 * k + depth)
    scores, _, _, _ = ref.grow(topk_p, topk_i, None, k, depth, dtype)
    assert scores.unique().numel() < scores.numel()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("k,depth", [(10, 7), (16, 8), (3, 4)])
def test_all_candidates_tie_the_frontier_is_the_lowest_flat_indices(lib, k, depth, dtype):
    topk_p = torch.full((1 + depth * k, k), -2.0)
    topk_i = torch.arange((1 + depth * k) * k, dtype=torch.int32).view(-1, k) % 500
    got = run_grow(lib, dtype, topk_p, topk_i, None, k, depth)
    for slot in range(depth + 1):
        assert got["cs"][slot].tolist() == list(range(k)), f"slot {slot}"
        assert got["src"][slot].tolist() == [0] * k
    compare(got, ref.grow(topk_p, topk_i, None, k, depth, dtype), k, depth, "all tied")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_equal_candidates_of_different_slots_lower_flat_index_wins(lib, dtype):
    """The cut of the frontier falls inside a three-way tie between children of slots 0, 1 and 2."""
    k, depth = 4, 1
    topk_p = torch.tensor([[-1.0, -2.0, -3.0, -4.0],     # seed scores of slots 0..3
                           [-1.0, -2.0, -3.0, -6.0],     # slot 0 children: cumulative -2 -3 -4 -7
                           [-1.0, -2.0, -8.0, -9.0],     # slot 1:          -3 -4 -10 -11
                           [-1.0, -5.0, -6.0, -7.0],     # slot 2:          -4 -8 -9 -10
                           [-1.0, -5.0, -6.0, -7.0]])    # slot 3:          -5 ...
    topk_i = torch.arange(20, dtype=torch.int32).view(5, 4)
    got = run_grow(lib, dtype, topk_p, topk_i, None, k, depth)
    # -2 (flat 0), then -3 twice (flat 1 before flat 4), then -4 three times (flat 2, 5, 8): flat 2 takes the last place
    assert got["cs"][1].tolist() == [0, 1, 4, 2]
    assert got["src"][1].tolist() == [0, 0, 1, 0]
    assert got["ids"][1].tolist() == [4, 5, 8, 6]
    assert got["fscores"][1].tolist() == [-2.0, -3.0, -3.0, -4.0]
    compare(got, ref.grow(topk_p, topk_i, None, k, depth, dtype), k, depth, "cross-slot tie")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_candidates_are_ranked_by_the_rounded_sum(lib, dtype):
    """Two sums that differ in fp32 but are one model-dtype value: the kernel ranks what the reference ranks, the rounded
    value (cnets.py:740 adds in the model dtype), so they tie and the lower flat index wins although its fp32 sum is smaller."""
    k, depth = 2, 1
    eps = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10  # one ulp at 1.0; far below one ulp at 9.0
    topk_p = torch.tensor([[-1.0 - eps, -1.0],    # slot 0 scores below slot 1 by one ulp
                           [-8.0, -20.0],         # slot 0 child 0: fp32 sum -9 - eps -> rounds to -9
                           [-8.0, -20.0]])        # slot 1 child 0: fp32 sum -9 exactly
    assert float(torch.tensor(-9.0 - eps).to(dtype)) == -9.0
    topk_i = torch.arange(6, dtype=torch.int32).view(3, 2)
    got = run_grow(lib, dtype, topk_p, topk_i, None, k, depth)
    assert got["cs"][1].tolist() == [0, 2] and got["fscores"][1].tolist() == [-9.0, -9.0]
    assert got["scores"][k:].tolist() == [-9.0, -21.0, -9.0, -21.0]
    compare(got, ref.grow(topk_p, topk_i, None, k, depth, dtype), k, depth, "rounded-sum tie")


# ----------------------------------------------------------------------------------------------
# growth -> finalize -> posterior as one chain
# ----------------------------------------------------------------------------------------------
def rank_transform(scores):
    """Distinct values in the kernels' (value desc, flat index asc) order, so that orc.finalize_tree's torch.topk -- whose tie
    order is unspecified -- selects what that policy selects."""
    order = ref.stable_topk(scores, scores.numel())
    out = torch.empty_like(scores)
    out[order] = -torch.arange(scores.numel(), dtype=scores.dtype)
    return out


def finalize(lib, scores, tokens, parents, k, depth, total, sample_token, sort_rows):
    T = total
    dt = torch.zeros(T, dtype=torch.int64)
    tm = torch.zeros(T * T, dtype=torch.float32)
    tp = torch.zeros(T, dtype=torch.int64)
    ri = torch.full((T * 16,), -1, dtype=torch.int64)
    nl, md = C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_tree_finalize(0, ptr(scores.contiguous()), ptr(tokens.int().contiguous()), ptr(parents.int().contiguous()), k, depth,
                                         total, sample_token, sort_rows, ptr(dt), ptr(tm), ptr(tp), ptr(ri), C.byref(nl), C.byref(md)))
    return dt[None], ri[: nl.value * md.value].view(nl.value, md.value), tm.view(1, 1, T, T), tp


def peaked_tables(k, depth, dtype, seed, boost=14.0, draft_vocab=512):
    """Tables of a confident draft (one logit per row raised by `boost`): the best root->leaf chain runs the full depth."""
    g = torch.Generator().manual_seed(seed)
    rows = 1 + depth * k
    logits = torch.randn(rows, draft_vocab, generator=g) * 2
    logits[torch.arange(rows), torch.randint(0, draft_vocab, (rows,), generator=g)] += boost
    logp = torch.log_softmax(logits.to(dtype), dim=-1)
    order = torch.sort(logp.double(), dim=-1, descending=True, stable=True).indices[:, :k]
    return torch.gather(logp, 1, order).float().contiguous(), order.int().contiguous()


@pytest.mark.parametrize("sort_rows", [0, 1])
@pytest.mark.parametrize("k,depth,total,peaked", [(10, 6, 60, False), (10, 7, 60, False), (10, 7, 60, True), (16, 8, 64, False),
                                                  (9, 14, 64, True), (9, 14, 64, False), (8, 8, 64, True), (1, 14, 16, True), (1, 1, 2, False)])
def test_grown_pool_finalizes_to_the_oracle_tree(lib, k, depth, total, peaked, sort_rows):
    dtype = torch.bfloat16
    topk_p, topk_i = (peaked_tables if peaked else ref.make_tables)(k, depth, dtype, seed=77 + k + depth)
    d2t = strided_d2t()
    got = run_grow(lib, dtype, topk_p, topk_i, d2t, k, depth, 3)
    compare(got, ref.grow(topk_p, topk_i, d2t, k, depth, dtype, 3), k, depth, f"k={k} depth={depth}")
    # the kernel gets the pool as grown (ties and all); the oracle gets the same order with the ties resolved by the policy
    want = orc.finalize_tree(rank_transform(got["scores"]), got["tokens"].long(), got["parents"].long(), torch.tensor([777]), k, total - 1,
                             bool(sort_rows))
    mine = finalize(lib, got["scores"], got["tokens"], got["parents"], k, depth, total, 777, sort_rows)
    for a, b, name in zip(mine, want, ("draft_tokens", "retrieve_indices", "tree_mask", "tree_position_ids")):
        assert a.shape == b.shape, f"{name}: {tuple(a.shape)} vs {tuple(b.shape)}"
        same(a, b, name)
    if peaked:
        assert want[1].shape[1] == depth + 2, "a confident draft must reach the deepest retrieve row"


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("temperature,top_p,top_k", [(1.0, 0.0, 0), (0.7, 0.9, 20)])
def test_sample_posterior_on_the_deepest_tree(lib, seed, temperature, top_p, top_k):
    """eb200_k_sample_posterior on a tree grown and finalized at depth 14 with 64 nodes (16-wide retrieve rows, the sequential
    walk up to 15 levels) against orc.evaluate_posterior_sampling with the same injected uniforms."""
    g = torch.Generator().manual_seed(300 + seed)
    k, depth, total, V = 9, 14, 64, 512
    dtype = torch.bfloat16
    topk_p, topk_i = peaked_tables(k, depth, dtype, seed=500 + seed)
    pool = run_grow(lib, dtype, topk_p, topk_i, None, k, depth)
    draft_tokens, retrieve, _, _ = orc.finalize_tree(rank_transform(pool["scores"]), pool["tokens"].long(), pool["parents"].long(),
                                                     torch.tensor([3]), k, total - 1, True)
    assert retrieve.shape[1] == 16
    logits_nodes = (torch.randn(total, V, generator=g) * 1.5).to(torch.bfloat16)
    deep = max(range(retrieve.shape[0]), key=lambda r: int((retrieve[r] >= 0).sum()))
    path = retrieve[deep]
    n_planted = (15, 15, 9, 4, 15, 1)[seed]  # how many levels of the deepest path the target agrees with
    for j in range(1, min(16, 1 + n_planted)):
        logits_nodes[path[j - 1], draft_tokens[0, path[j]]] = 30.0
    uniforms = torch.rand(256, generator=g)
    it = iter(uniforms.tolist())
    warp = lambda lg: orc.warp_logits(lg, temperature, top_p, top_k)  # noqa: E731
    lg32 = logits_nodes.float()
    if temperature != 1.0:  # TemperatureLogitsWarper divides in the model dtype
        lg32 = (logits_nodes / temperature).float()
        warp = lambda lg: orc.warp_logits(lg, 1.0, top_p, top_k)  # noqa: E731
    cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
    w_best, w_acc, w_p = orc.evaluate_posterior_sampling(lg32[retrieve], cands, warp, rand=lambda: next(it))
    u_bonus = next(it)
    cdf = torch.cumsum(w_p.double(), 0)
    w_bonus = int(torch.searchsorted(cdf, torch.tensor(u_bonus * float(cdf[-1]), dtype=torch.float64)))
    best, acc, bonus, used = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_sample_posterior(0, ptr(logits_nodes.cuda()), V, ptr(draft_tokens[0].int().contiguous()),
                                            ptr(retrieve.int().contiguous()), total, retrieve.shape[0], retrieve.shape[1], temperature, top_p,
                                            top_k, ptr(uniforms.contiguous()), 256, C.byref(best), C.byref(acc), C.byref(bonus), C.byref(used)))
    assert (best.value, acc.value) == (int(w_best), int(w_acc))
    if n_planted == 15:
        assert acc.value == 15, "the planted path is accepted to the full depth: 15 levels walked"
    assert bonus.value == w_bonus or abs(float(cdf[bonus.value]) - u_bonus * float(cdf[-1])) < 1e-4

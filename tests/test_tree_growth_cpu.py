"""The torch reference the tree-growth kernels are held to (tests/tree_growth_ref.py) is itself held to the CPU oracle:
on tie-free inputs, fed the oracle's own per-level top-k tables, it must reproduce topk_generate's candidate pool, the
level ids and the dense tree mask the oracle hands to every draft forward, and so the finished tree.  Also the host-side
argument checks of eb200_k_tree_grow, which run before any CUDA call.  No GPU."""
import ctypes as C

import pytest
import torch

from oracle import eagle_oracle as orc
from tests import tree_growth_ref as ref
from tests.fixtures import fixture_models, to_cfg


def _fp64(W):
    return {k: (v.double() if v.dtype.is_floating_point else v) for k, v in W.items()}


@pytest.mark.parametrize("fx", ["e3_rand_bf16", "e1_rand_bf16"])  # EAGLE-3 with a d2t map / EAGLE-1 without
@pytest.mark.parametrize("total,depth,k", [(60, 7, 10), (64, 8, 16), (64, 14, 9), (17, 1, 16), (2, 1, 1)])
def test_reference_reproduces_the_oracle_on_tie_free_inputs(fx, total, depth, k):
    tcfg, tW, hcfg, hW, eagle3, _, _ = fixture_models(fx)
    # float64 model: its cumulative scores do not tie (a near-uniform random head ties even in fp32 a few levels down), so
    # torch.topk's unspecified tie order cannot matter
    tW, hW = _fp64(tW), _fp64(hW)
    head = orc.DraftHead(to_cfg(hcfg), hW, eagle3, total, depth, k)
    g = torch.Generator().manual_seed(depth * 100 + k)
    P = 23
    feat = (3 if eagle3 else 1) * tcfg["hidden_size"]
    hidden = torch.randn(1, P, feat, generator=g, dtype=torch.float64) * 0.5
    ids = torch.randint(0, tcfg["vocab_size"] - 200, (1, P + 1), generator=g)
    seen = []
    inner = head.forward

    def spy(h, input_ids, past_kv=None, position_ids=None, tree_mask=None, **kw):
        if tree_mask is not None:
            seen.append((input_ids.clone(), tree_mask.clone()))
        return inner(h, input_ids, past_kv=past_kv, position_ids=position_ids, tree_mask=tree_mask, **kw)

    head.forward = spy
    head.trace = {}
    want_tree = head.topk_generate(hidden, ids, tW["lm_head.weight"], False)
    tr = head.trace
    assert len(seen) == depth and len(tr["level_logp"]) == depth + 1
    tops = [torch.topk(lp, k, dim=-1) for lp in tr["level_logp"]]  # the oracle's own tables
    topk_p = torch.cat([t.values.reshape(-1, k) for t in tops])
    topk_i = torch.cat([t.indices.reshape(-1, k) for t in tops])
    d2t = hW.get("d2t") if eagle3 and hcfg.get("draft_vocab_size", hcfg["vocab_size"]) != hcfg["vocab_size"] else None
    assert (d2t is not None) == (fx == "e3_rand_bf16")
    scores, tokens, parents, levels = ref.grow(topk_p, topk_i, d2t, k, depth, torch.float64, last_row=P - 1)
    # tie-free where a tie could matter: the best k + 1 candidates of every level, and the cut of the global rerank
    exact = tr["scores_flat"]
    assert exact.dtype == torch.float64
    for lvl in range(depth):
        cu = exact[k + lvl * k * k: k + (lvl + 1) * k * k].sort(descending=True).values[: k + 1]
        assert cu.unique().numel() == cu.numel(), f"level {lvl}: tied frontier candidates, the comparison would be ill-defined"
    ranked = exact.sort(descending=True).values
    assert total - 1 >= ranked.numel() or ranked[total - 2] > ranked[total - 1]
    assert torch.equal(scores, exact.float())
    assert torch.equal(tokens, tr["tokens_flat"])
    assert torch.equal(parents, tr["parents_flat"])
    for lvl, (level_ids, tree_mask) in enumerate(seen):  # what the oracle fed to the draft forward of level `lvl`
        assert torch.equal(levels[lvl]["ids"], level_ids.reshape(-1)), f"level {lvl} ids"
        assert torch.equal(levels[lvl]["mask"], tree_mask[0, 0].bool()), f"level {lvl} tree mask"
        assert levels[lvl]["mask"].shape == (k, (lvl + 1) * k)
    got_tree = orc.finalize_tree(exact, tokens, parents, ids[:, -1], k, total - 1, False)
    for a, b in zip(got_tree, want_tree):
        assert torch.equal(a, b)


def test_stable_topk_orders_ties_by_index():
    v = torch.tensor([-1.0, -2.0, -1.0, -3.0, -2.0, -1.0])
    assert ref.stable_topk(v, 5).tolist() == [0, 2, 5, 1, 4]


def test_pack_mask_word_boundaries():
    dense = torch.zeros(3, 128, dtype=torch.bool)
    dense[0, 0] = dense[0, 63] = True
    dense[1, 64] = True
    dense[2, 127] = True
    assert ref.pack_mask(dense).tolist() == [[1 - (1 << 63), 0], [0, 1], [0, -(1 << 63)]]


@pytest.mark.parametrize("kw,msg", [
    (dict(k=33, depth=2), "top_k must be in [1, 32]"),
    (dict(k=0, depth=2), "top_k must be in [1, 32]"),
    (dict(k=4, depth=15), "depth must be in [1, 14]"),
    (dict(k=4, depth=0), "depth must be in [1, 14]"),
    (dict(k=13, depth=10), "depth * top_k must be <= 128"),
    (dict(k=4, depth=2, dtype=2), "dtype must be bf16 or fp16"),
    (dict(k=4, depth=2, last_row=-1), "last_row must be >= 0"),
    (dict(k=4, depth=2, bad_index=True), "out of range"),
])
def test_tree_grow_refuses_bad_arguments_on_the_host(kw, msg):
    """Out-of-range geometries are refused with a message before anything is launched (so this needs no device)."""
    from eagle_b200 import _lib
    lib = _lib.load()
    k, depth = kw["k"], kw["depth"]
    rows = 1 + max(depth, 0) * max(k, 1)
    p = torch.zeros(rows * max(k, 1), dtype=torch.float32)
    i = torch.zeros(rows * max(k, 1), dtype=torch.int32)
    d2t = torch.zeros(8, dtype=torch.int64)
    if kw.get("bad_index"):
        i[5] = 8  # == d2t_len
    rc = lib.eb200_k_tree_grow(kw.get("dtype", 0), C.c_void_p(p.data_ptr()), C.c_void_p(i.data_ptr()), C.c_void_p(d2t.data_ptr()), 8,
                               k, depth, kw.get("last_row", 0), None, None, None, None, None, None, None, None)
    assert rc != 0 and msg in lib.eb200_last_error().decode()

"""Engines at the draft-tree geometries no named fixture reaches: EaModel.from_pretrained's default (total_token 60,
depth 7, top_k 10 -- 70 draft columns, the second 64-bit word of every ancestor mask in use) and the limits eb200_create
accepts (128 columns, 64 verify rows, depth 14 with 16-wide retrieve rows and 16-row commits, the smallest engine).

The reference is the CPU oracle on the same seeded weights with the same total_token / depth / top_k (pinned to the
unmodified reference at depth 7 and at 128 columns by tests/golden/e3_corr_bf16_D7.pt / _D8K16.pt, tests/test_oracle_golden.py).
Integer results (ids, accept lengths, committed tokens, verify arg-max of shared nodes, tree structure) are exact; the draft
logits carry the tolerance of tests/test_fullshape_gpu.py (1e-3 + one ulp of the model dtype), stated where it is used.
"""
import pytest
import torch

from eagle_b200 import synthetic as syn
from eagle_b200.synthetic import FIXTURES, fixture_models, make_prompt
from oracle import eagle_oracle as orc
from tests import test_e2e_gpu as e2e
from tests.fixtures import load_golden, report, to_cfg
from tests.test_e2e_gpu import node_map

pytestmark = pytest.mark.gpu

ULP = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}

DEFAULT = dict(total_token=60, depth=7, top_k=10)    # EaModel.from_pretrained without tree arguments: 70 draft columns
WIDE = dict(total_token=64, depth=8, top_k=16)       # 128 columns exactly, 16-row draft tile and 64-row verify tile full
DEEP = dict(total_token=64, depth=14, top_k=9)       # retrieve rows 16 wide, 126 columns
NARROW = dict(total_token=32, depth=12, top_k=4)     # most nodes on long chains
SMALLEST = dict(total_token=2, depth=1, top_k=1)
SHALLOW = dict(total_token=17, depth=1, top_k=16)    # pool k + k*k much larger than the tree


def tid(tree):
    return f"T{tree['total_token']}-d{tree['depth']}-k{tree['top_k']}"


def weights(base, corrupt_frac=None):
    """The named fixture's weights; corrupt_frac replaces the EAGLE-3 copy head of e3_corr_bf16 by one that is wrong on that
    fraction of rows (0.0: a draft that is always right, so every cycle accepts the full depth)."""
    tcfg, tW, hcfg, hW, eagle3, dtype, _ = fixture_models(base)
    if corrupt_frac is not None:
        assert base == "e3_corr_bf16"
        hW = syn.make_copy_head_eagle3_(syn.make_head_weights(hcfg, tW, True, 3, dtype), tW, hcfg, corrupt_frac=corrupt_frac)
    return tcfg, tW, hcfg, hW, eagle3, dtype


def engine(w, tree, max_length=512, **kw):
    from eagle_b200 import EaModel
    tcfg, tW, hcfg, hW, eagle3, dtype = w
    return EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=max_length, **dict(tree, **kw))


def oracle(w, tree):
    tcfg, tW, hcfg, hW, eagle3, dtype = w
    return orc.OracleEaModel(to_cfg(tcfg), tW, to_cfg(hcfg), hW, eagle3, **tree)


def prompt_of(base, w, n=None):
    plen, pseed, _, _ = FIXTURES[base]
    return make_prompt(w[0]["vocab_size"], n or plen, pseed)


def check_tree(dt, ri, tm, tp, tree, what):
    """Structure every correct draft tree has, whatever order tied siblings come in."""
    T, D = tree["total_token"], tree["depth"] + 2
    assert dt.shape == (1, T) and tm.shape == (1, 1, T, T) and tp.shape == (T,), what
    m = tm[0, 0] > 0
    assert set(tm.unique().tolist()) <= {0.0, 1.0}, what
    assert bool(m.diagonal().all()) and bool(m[:, 0].all()), f"{what}: diagonal / root column of the tree mask"
    assert not bool(torch.triu(m, 1).any()), f"{what}: a node sees a later node"
    depth_of = m.sum(-1) - 1
    assert torch.equal(tp, depth_of), f"{what}: tree_position_ids != mask.sum(-1) - 1"
    assert int(depth_of.max()) + 1 == ri.shape[1] <= D, f"{what}: max_depth"
    parent = [0] * T
    for i in range(1, T):
        anc = [j for j in range(i) if m[i, j]]
        p = max(anc, key=lambda j: int(depth_of[j]))
        assert int(depth_of[p]) == int(depth_of[i]) - 1, f"{what}: node {i} has no parent one level up"
        own = torch.zeros(T, dtype=torch.bool)
        own[i] = True
        assert torch.equal(m[i], m[p] | own), f"{what}: ancestors of node {i} are not its parent's plus itself"
        parent[i] = p
    leaves = sorted(set(range(T)) - set(parent[1:])) if T > 1 else [0]
    assert ri.shape[0] == len(leaves), f"{what}: n_leaf {ri.shape[0]} but {len(leaves)} nodes have no child"
    ends = []
    for r in range(ri.shape[0]):
        row = ri[r].tolist()
        n = sum(1 for x in row if x >= 0)
        assert n >= 1 and all(x >= 0 for x in row[:n]) and all(x == -1 for x in row[n:]), f"{what}: retrieve row {r} padding {row}"
        assert row[0] == 0, f"{what}: retrieve row {r} does not start at the root"
        assert row[:n] == [j for j in range(T) if m[row[n - 1], j]], f"{what}: retrieve row {r} is not the root->leaf path of the mask"
        ends.append(row[n - 1])
    assert sorted(ends) == leaves, f"{what}: retrieve rows end in {sorted(ends)}, the leaves are {leaves}"


def frontier_logits_bar(got, want, dtype):
    """Last-level draft logits [k, V] of the engine (got) against the oracle's (want).  Rows belong to the k frontier nodes; tied
    low-probability filler may be fed different tokens by the two implementations (torch.topk orders ties arbitrarily), so rows
    are paired by distance (median error below 0.05) and only rows of the same node are compared, element-wise against
    1e-3 + one ulp of the model dtype.  Returns (pairs, elements beyond the bar, elements compared, worst error / bar)."""
    k = got.shape[0]
    d = (got[:, None, :] - want[None, :, :]).abs().median(-1).values
    used, pairs = set(), []
    for i in range(k):
        j = min((jj for jj in range(want.shape[0]) if jj not in used), key=lambda jj: float(d[i, jj]))
        if float(d[i, j]) < 0.05:
            used.add(j)
            pairs.append((i, j))
    n_bad, n_all, worst = 0, 0, 0.0
    for i, j in pairs:
        err = (got[i] - want[j]).abs()
        tol = 1e-3 + ULP[dtype] * want[j].abs()
        n_bad += int((err > tol).sum())
        n_all += err.numel()
        worst = max(worst, float((err / tol).max()))
    return pairs, n_bad, n_all, worst


def compare_cycles(m, ref, prompt, tree, what, new_tokens=48, max_length=512, min_shared=None):
    """Whole call, then cycle by cycle against the oracle's log.  Returns (accept lengths, shared verify nodes compared)."""
    ref.cycle_log = []
    want, w_new, w_idx = ref.eagenerate(prompt, max_new_tokens=new_tokens, max_length=max_length, log=True)
    log, ref.cycle_log = ref.cycle_log, None
    ids, new_token, idx = m.eagenerate(prompt.cuda(), max_new_tokens=new_tokens, max_length=max_length, log=True)
    assert ids.cpu().tolist() == want.tolist(), f"{what}: generated ids"
    assert (new_token, idx) == (w_new, w_idx), f"{what}: (new_token, idx)"
    first = m.prefill(prompt.cuda())
    assert first == int(want[0, prompt.shape[1]])
    T = tree["total_token"]
    floor = min(8, T) if min_shared is None else min_shared
    n_cmp, committed = 0, prompt.shape[1]
    for c, rec in enumerate(log):
        dt, ri, tm, tp = m.get_tree()
        check_tree(dt, ri, tm, tp, tree, f"{what} cycle {c}")
        toks, nxt = m.step()
        am, best, acc, n = m.get_verify()
        wt = torch.cat((rec["draft_tokens"], torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, rec["retrieve"]]
        assert toks == wt[rec["best"], : rec["accept_length"] + 1].tolist(), f"{what} cycle {c}: committed tokens differ"
        assert acc == rec["accept_length"] and nxt == rec["bonus"], f"{what} cycle {c}: accept length / bonus token"
        committed += acc + 1
        assert n == committed, f"{what} cycle {c}: committed length {n}, expected {committed}"
        shared = [(i, j) for i, j in node_map(dt, tm, rec["draft_tokens"], rec["tree_mask"]).items() if j is not None]
        assert len(shared) >= floor, f"{what} cycle {c}: the two draft trees share only {len(shared)} of {T} nodes"
        for i, j in shared:
            assert int(am[i]) == int(rec["node_argmax"][j]), f"{what} cycle {c}: verify arg-max of node {i} differs"
        n_cmp += len(shared)
    accs = [rec["accept_length"] for rec in log]
    report(f"tree geometry {what}: {len(log)} cycles identical to the oracle, accept lengths {accs}, {n_cmp} verify nodes compared")
    return accs, n_cmp


GREEDY_CASES = [
    ("e3_corr_bf16", DEFAULT), ("e1_corr_fp16", DEFAULT), ("e3_gqa_bf16", DEFAULT),
    ("e3_corr_bf16", WIDE), ("e1_corr_fp16", WIDE),
    ("e3_corr_bf16", DEEP), ("e3_gqa_bf16", DEEP),
    ("e3_corr_bf16", NARROW), ("e3_corr_bf16", SMALLEST), ("e1_corr_fp16", SMALLEST), ("e3_corr_bf16", SHALLOW),
]


@pytest.mark.parametrize("base,tree", GREEDY_CASES, ids=[f"{b}-{tid(t)}" for b, t in GREEDY_CASES])
def test_greedy_generation_identical_to_the_oracle(base, tree):
    w = weights(base)
    accs, n_cmp = compare_cycles(engine(w, tree), oracle(w, tree), prompt_of(base, w), tree, f"{base} {tid(tree)}")
    if base.startswith("e3") and tree["depth"] >= 7 and tree["top_k"] > 1:  # the EAGLE-1 copy head is never wrong: all accepts are full
        assert max(accs) >= 8 and min(accs) == 0, f"the fixture must exercise long and empty accepts: {accs}"
    if base.startswith("e1") and tree["top_k"] > 1:
        assert min(accs) == tree["depth"] + 1, f"an always-right head accepts the full depth every cycle: {accs}"


@pytest.mark.parametrize("fx", ["e3_corr_bf16_D7", "e3_corr_bf16_D8K16"])
def test_identical_to_the_reference_goldens(fx):
    """The two geometries that have vectors from the unmodified reference: the bodies of the reference-golden tests of
    tests/test_e2e_gpu.py, run on the new fixture names."""
    e2e.test_correlated_fixture_identical_to_reference(fx, 0)
    e2e.test_first_tree_and_stepwise_state(fx)
    g = load_golden(fx)
    assert max(c["accept_length"] for c in g["cycles"]) == g["tree"]["depth"] + 1, "the golden run contains a full-depth accept"


@pytest.mark.parametrize("tree", [DEFAULT, WIDE], ids=tid)
@pytest.mark.parametrize("base", ["e3_rand_bf16", "e1_rand_bf16"])
def test_random_weights_speculative_equals_vanilla_greedy(base, tree):
    """Losslessness where nothing is peaked: near-uniform logits, cumulative scores that tie all over the tree."""
    w = weights(base)
    m = engine(w, tree)
    prompt = prompt_of(base, w).cuda()
    ids = m.eagenerate(prompt, max_new_tokens=40, max_length=512).cpu()
    naive = m.naivegenerate(prompt, max_new_tokens=40, max_length=512).cpu()
    n = min(ids.shape[1], naive.shape[1])
    assert n > prompt.shape[1] + 40 and ids[0, :n].tolist() == naive[0, :n].tolist(), "speculative output differs from vanilla greedy"
    m.prefill(prompt)
    for c in range(4):
        check_tree(*m.get_tree(), tree, f"{base} {tid(tree)} cycle {c}")
        m.step()


@pytest.mark.parametrize("tree", [DEFAULT, WIDE], ids=tid)
def test_last_level_draft_logits_within_1e3_of_the_oracle(tree):
    """The last level's draft forward attends over columns 64.. of the draft tree: a missing or extra ancestor bit in the second
    mask word changes these logits far beyond an ulp while the generated text stays lossless.  Tolerance as in
    tests/test_fullshape_gpu.py: 1e-3 absolute plus one ulp of the model dtype (the spacing of the tensor the reference itself
    materialises); the kernels accumulate in fp32 like the reference, so only summation order differs."""
    base = "e3_corr_bf16"
    w = weights(base)
    m, ref, prompt = engine(w, tree), oracle(w, tree), prompt_of(base, w)
    ref.head.trace = {}
    ref.eagenerate(prompt, max_new_tokens=0, max_length=512, log=True)  # prefill + one cycle: the trace holds the tree grown after it
    want = ref.head.trace["level_raw"][-1].float()
    ref.head.trace = None
    k = tree["top_k"]
    assert want.shape[0] == k
    m.prefill(prompt.cuda())
    m.step()
    got = m.debug_read("draft_logits")[:k]
    assert got.shape == want.shape
    pairs, n_bad, n_all, worst = frontier_logits_bar(got, want, w[5])
    assert len(pairs) >= 3, f"only {len(pairs)} of {k} frontier rows are fed the same node in both implementations"
    report(f"tree geometry {tid(tree)}: last-level draft logits over {(tree['depth']) * k} columns, {len(pairs)} comparable rows, "
           f"{n_bad}/{n_all} beyond 1e-3 + 1 ulp, worst {worst:.2f} x tolerance")
    assert n_bad <= n_all * 1e-3 and worst <= 3.0, f"{n_bad}/{n_all} draft logits beyond 1e-3 + 1 ulp; worst {worst:.2f}x"


@pytest.mark.parametrize("tree", [DEEP, DEFAULT], ids=tid)
def test_full_depth_accepts_commit_every_row(tree):
    """A draft that is always right: every cycle accepts depth + 1 draft tokens and commits depth + 2 rows (16 at depth 14: every
    row kv_compact_kernel has).  After such a cycle the committed target KV must be what the oracle holds, and what a second
    engine holds that prefilled the same ids from scratch."""
    base = "e3_corr_bf16"
    w = weights(base, corrupt_frac=0.0)
    m, ref, prompt = engine(w, tree), oracle(w, tree), prompt_of(base, w)
    accs, _ = compare_cycles(m, ref, prompt, tree, f"always-right head {tid(tree)}", new_tokens=60)
    full = tree["depth"] + 1
    assert accs and all(a == full for a in accs), f"every cycle of the oracle must accept the full depth {full}: {accs}"
    # replay two cycles and look at the KV cache
    P = prompt.shape[1]
    ids = [int(x) for x in prompt[0]]
    m.prefill(prompt.cuda())
    for _ in range(2):
        toks, _ = m.step()
        assert len(toks) == full + 1
        ids += toks
    n = len(ids)
    assert n == P + 2 * (full + 1) == m.get_verify()[3]
    tcfg = w[0]
    L, nkv = tcfg["num_hidden_layers"], tcfg["num_key_value_heads"]
    kv = m.debug_read("target_kv").view(L * 2 * nkv, -1, 128)[:, :n]
    # the oracle's cache after the same two cycles: planes 2l (K) / 2l+1 (V) of [1, nkv, max_length, 128]
    ref.cycle_log = None
    okv = oracle(w, tree)
    okv.eagenerate(prompt, max_new_tokens=2 * (full + 1) - 1, max_length=512)
    want = okv.kv.data[:, 0, :, :n].float()  # [2L, nkv, n, 128]
    want = torch.stack([want[2 * l + s, h] for l in range(L) for s in range(2) for h in range(nkv)])
    fresh = engine(w, tree)
    fresh.prefill(torch.tensor([ids]).cuda())
    kv2 = fresh.debug_read("target_kv").view(L * 2 * nkv, -1, 128)[:, :n]

    def row_err(a, b):  # relative L2 distance per (plane, row)
        return (a - b).norm(dim=-1) / b.norm(dim=-1).clamp_min(1e-6)

    # A row left uncompacted holds another node's K/V: relative distance ~1.  Rounding differences between the verify pass, the
    # prefill and the CPU oracle (different summation orders through 8 layers) stay far below the 5% bar; the first layer's planes
    # have three rounding points (RMSNorm, GEMM, RoPE) and are held to 2 ulp + 1e-3 element-wise against the oracle.
    e_or, e_fr = row_err(kv, want), row_err(kv, kv2)
    report(f"tree geometry {tid(tree)}: target KV after two {full + 1}-row commits: worst row distance {float(e_or.max()):.4f} to the "
           f"oracle, {float(e_fr.max()):.4f} to a fresh prefill (bit-identical: {bool(torch.equal(kv, kv2))})")
    assert float(e_or.max()) < 0.05, f"committed KV rows differ from the oracle: {(e_or >= 0.05).nonzero()[:8].tolist()}"
    assert float(e_fr.max()) < 0.05, f"committed KV rows differ from a fresh prefill: {(e_fr >= 0.05).nonzero()[:8].tolist()}"
    first_layer = slice(0, 2 * nkv)
    err = (kv[first_layer] - want[first_layer]).abs()
    tol = 1e-3 + 2 * ULP[w[5]] * want[first_layer].abs()
    assert bool((err <= tol).all()), f"layer-0 K/V: {int((err > tol).sum())} elements beyond 2 ulp, max {float(err.max()):.4g}"


@pytest.mark.parametrize("tree", [DEFAULT, DEEP], ids=tid)
@pytest.mark.parametrize("gen", [dict(temperature=1.0), dict(temperature=0.7, top_p=0.9, top_k=20)], ids=["T1", "T07-p09-k20"])
def test_sampling_is_reproducible_and_follows_the_peaked_target(tree, gen):
    """Sampling sorts the retrieve rows (tree_finalize's sort_rows branch, limited to depth + 2 <= 16) and walks the posterior
    level by level.  Seeded runs repeat; with top_p = 0.9 the large-margin target (p(top-1) ~ 0.997) keeps only its top-1 token,
    so that sample is the greedy continuation (at plain temperature 1 a 40-token sample leaves it about one time in ten)."""
    base = "e3_corr_bf16"
    w = weights(base)
    m = engine(w, tree)
    prompt = prompt_of(base, w)
    greedy = m.eagenerate(prompt.cuda(), max_new_tokens=40, max_length=512).cpu()
    torch.manual_seed(7)
    a = m.eagenerate(prompt.cuda(), max_new_tokens=40, max_length=512, **gen).cpu()
    torch.manual_seed(7)
    b = m.eagenerate(prompt.cuda(), max_new_tokens=40, max_length=512, **gen).cpu()
    assert a.tolist() == b.tolist() and a.shape[1] > prompt.shape[1] + 40
    if "top_p" in gen:
        n = min(a.shape[1], greedy.shape[1])
        assert a[0, :n].tolist() == greedy[0, :n].tolist()
    m.prefill(prompt.cuda())
    check_tree(*m.get_tree(), tree, f"sampling {tid(tree)}")


@pytest.mark.parametrize("tree", [DEFAULT, DEEP], ids=tid)
def test_sampling_posterior_is_lossless_monte_carlo(tree):
    """tests/test_e2e_gpu.py's Monte-Carlo check at these geometries: first token pinned, the second generated token -- decided by
    the speculative-sampling posterior -- must follow the target's own next-token distribution (chi-square over 16 equal-mass
    buckets, df = 15, bound 45 as there: p < 1e-4 for a correct sampler)."""
    base = "e3_rand_bf16"
    w = weights(base)
    m, ref = engine(w, tree), oracle(w, tree)
    prompt = prompt_of(base, w)
    P = prompt.shape[1]
    m.set_uniforms([0.5])
    torch.manual_seed(0)
    t1 = int(m.eagenerate(prompt.cuda(), temperature=1.0, max_new_tokens=0, max_length=512)[0, P])
    hidden, _ = ref.target.forward(torch.cat((prompt, torch.tensor([[t1]])), dim=1), ref._kv(512))
    p2 = torch.softmax(ref.target.lm_head(hidden)[0, -1].float(), dim=-1)
    order = torch.argsort(p2, descending=True)
    n_buckets, n_trials = 16, 1600
    cum = torch.cumsum(p2[order], 0)
    bucket_of = torch.empty_like(order)
    bucket_of[order] = torch.clamp((cum * n_buckets).long(), max=n_buckets - 1)
    expected = torch.zeros(n_buckets).index_add_(0, bucket_of, p2) * n_trials
    counts = torch.zeros(n_buckets)
    dev_prompt = prompt.cuda()
    for i in range(n_trials):
        m.set_uniforms([0.5])
        torch.manual_seed(1000 + i)
        ids = m.eagenerate(dev_prompt, temperature=1.0, max_new_tokens=1, max_length=512)
        assert int(ids[0, P]) == t1
        counts[bucket_of[int(ids[0, P + 1])]] += 1
    chi2 = float(((counts - expected) ** 2 / expected).sum())
    report(f"tree geometry {tid(tree)}: sampling losslessness chi2={chi2:.1f} over {n_buckets} equal-mass buckets, {n_trials} trials")
    assert chi2 < 45.0, f"second-token histogram deviates from the target distribution: chi2={chi2:.1f} (df=15)"


def test_int8_twin_at_the_default_geometry():
    from tests.test_w8_gpu import run_cycles, same, twins
    m8, mb, prompt, gen_kw, _ = twins("e3_corr_bf16", **DEFAULT)
    a = m8.eagenerate(prompt.cuda(), log=True, **gen_kw)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    n = a[2] + 1
    ca, cb = run_cycles(m8, prompt, n), run_cycles(mb, prompt, n)
    for c in range(n + 1):
        assert same(ca[c], cb[c]), f"cycle {c - 1}: int8 engine and its model-dtype twin differ"


def test_static_tree_next_to_a_wide_dynamic_engine():
    """A fixed tree is untouched by the dynamic-tree geometry of another engine in the same process."""
    from eagle_b200 import static_trees
    base = "e3_corr_bf16"
    w = weights(base)
    wide = engine(w, WIDE)
    prompt = prompt_of(base, w)
    wide.eagenerate(prompt.cuda(), max_new_tokens=16, max_length=512)
    tcfg, tW, hcfg, hW, eagle3, dtype = w
    m = engine(w, dict(top_k=10), tree_choices=static_trees.mc_sim_7b_63)
    o = orc.OracleEaModel(to_cfg(tcfg), tW, to_cfg(hcfg), hW, eagle3, top_k=10, tree_choices=[list(c) for c in static_trees.mc_sim_7b_63])
    want = o.eagenerate(prompt, max_new_tokens=40, max_length=512, log=True)
    got = m.eagenerate(prompt.cuda(), max_new_tokens=40, max_length=512, log=True)
    assert got[0].cpu().tolist() == want[0].tolist() and got[1:] == want[1:]


def test_kv_bucket_crossing_with_a_128_column_tree():
    """The attention strips (and the captured cycle graph) are sized in 256-row buckets of committed + total_token + depth + 2 +
    depth * top_k + 8 rows.  At 64 / 8 / 16 that is committed + 210: a 230-token prompt starts in the 512-row bucket and leaves it
    once 303 tokens are committed, so this generation re-captures the graph while the draft tree is 128 columns wide."""
    base = "e3_corr_bf16"
    w = weights(base)
    prompt = prompt_of(base, w, n=230)
    m, ref = engine(w, WIDE, max_length=640), oracle(w, WIDE)
    accs, _ = compare_cycles(m, ref, prompt, WIDE, f"bucket crossing {tid(WIDE)}", new_tokens=110, max_length=640)
    assert 230 + 210 + 64 <= 512 < 230 + sum(a + 1 for a in accs) + 210, "the run must start inside the 512-row bucket and leave it"


BAD_GEOMETRIES = [
    (dict(total_token=1), r"total_token must be in \[2, 64\]"), (dict(total_token=65), r"total_token must be in \[2, 64\]"),
    (dict(top_k=0), r"top_k must be in \[1, 16\]"), (dict(top_k=17, depth=4), r"top_k must be in \[1, 16\]"),
    (dict(depth=0), r"depth must be in \[1, 14\]"), (dict(depth=15, top_k=4), r"depth must be in \[1, 14\]"),
    (dict(depth=13, top_k=10), r"depth \* top_k must be <= 128"),
    (dict(total_token=12, depth=2, top_k=2), "candidate pool smaller than total_token - 1"),  # pool 2 + 2 * 4 = 10 < 11
]


@pytest.mark.parametrize("kw,msg", BAD_GEOMETRIES, ids=[str(sorted(k.items())) for k, _ in BAD_GEOMETRIES])
def test_create_refuses_geometries_outside_the_limits(kw, msg):
    from eagle_b200 import EaModel, _lib
    tcfg, tW, hcfg, hW, eagle3, dtype = weights("e3_corr_bf16")
    with pytest.raises(_lib.EngineError, match=msg):
        EaModel(tcfg, hcfg, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, **dict(DEFAULT, **kw))


def test_set_total_token_refuses_above_capacity():
    from eagle_b200 import _lib
    base = "e3_corr_bf16"
    w = weights(base)
    m = engine(w, dict(total_token=40, depth=7, top_k=10))
    lib = _lib.load()
    with pytest.raises(_lib.EngineError, match=r"total_token must be in \[2, 40\]"):
        _lib.check(lib.eb200_set_total_token(m._h, 41))
    with pytest.raises(_lib.EngineError, match=r"total_token must be in \[2, 40\]"):
        _lib.check(lib.eb200_set_total_token(m._h, 1))
    _lib.check(lib.eb200_set_total_token(m._h, 24))
    m._cfg.total_token = 24
    m.ea_layer.total_tokens = 23
    tree = dict(total_token=24, depth=7, top_k=10)
    compare_cycles(m, oracle(w, tree), prompt_of(base, w), tree, "set_total_token 40 -> 24")

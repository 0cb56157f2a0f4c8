"""Tree attention at the engine's launch geometry, on the H100, against the rounding-aware float64 reference of
tests/attention_ref.py.

The engine sizes the score strip from its KV bucket (max_kv = min(cap, kv_bucket)), not from the live length, so cluster
ranks with no or only some live KV tiles, strips wider than the live columns, one head per CTA under GQA and row / prefix
counts read from the device state are the usual case.  eb200_k_attention_ex launches the kernel exactly that way.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import eagle_oracle as orc
from tests import attention_ref as ar
from tests.fixtures import report

pytestmark = pytest.mark.gpu

DT = {torch.bfloat16: 0, torch.float16: 1}
MAX_KV = 16896  # largest score strip the kernel holds (DESIGN.md); engines need max_length + 128 + depth * top_k <= it
BIG = {torch.bfloat16: 1e30, torch.float16: 6e4}  # large finite cache garbage


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _mask_tensor(masks):
    if masks is None:
        return None
    flat = []
    for lo, hi in masks:
        flat += [lo - (1 << 64) if lo >= (1 << 63) else lo, hi - (1 << 64) if hi >= (1 << 63) else hi]
    return torch.tensor(flat, dtype=torch.int64, device="cuda")


def launch(lib, dtype, q, kc, vc, max_kv, n_ctx, n_tree, masks, out=None, st=None, rows_idx=-1, n_ctx_idx=-1, hpc_cap=0,
           kvs_cap=0):
    """q [rows, nh, 128], kc / vc [nkv, cap, 128] on the GPU.  Returns (rc, out [rows, nh, 128])."""
    rows, nh, _ = q.shape
    nkv, cap, _ = kc.shape
    if out is None:
        out = torch.zeros(rows, nh * 128, dtype=dtype, device="cuda")
    m = _mask_tensor(masks)
    torch.cuda.synchronize()
    rc = lib.eb200_k_attention_ex(DT[dtype], _ptr(q), _ptr(kc), _ptr(vc), _ptr(out), rows, nh, nkv, cap, max_kv, _ptr(st), rows_idx,
                                  n_ctx_idx, n_ctx, n_tree, _ptr(m), hpc_cap, kvs_cap, None)
    return rc, out[:rows].view(rows, nh, 128)


def ok(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def tree_masks(n_tree, rows, seed):
    """Ancestor masks of `rows` nodes of a real draft tree of n_tree nodes (orc.finalize_tree over a random candidate pool,
    cnets.py:760-827), as (word0, word1) pairs."""
    if n_tree == 1:
        return [(1, 0)] * rows
    k = 10
    depth = 1 + max(0, -(-(n_tree - 1 - k) // (k * k)))
    g = torch.Generator().manual_seed(seed)
    scores = [F.log_softmax(torch.randn(k, generator=g) * 2, -1)]
    front, parents, cs = scores[0].clone(), [torch.zeros(1, dtype=torch.long)], torch.arange(k)
    for i in range(depth):
        parents.append(cs + 1 + k * k * max(0, i - 1) + (k if i > 0 else 0))
        cu = F.log_softmax(torch.randn(k, k, generator=g) * 2, -1) + front[:, None]
        scores.append(cu)
        top = torch.topk(cu.view(-1), k)
        cs, front = top.indices, top.values
    s = torch.cat([x.reshape(-1) for x in scores])
    tokens = torch.randint(0, 1000, (s.numel(),), generator=g)
    _, _, tm, _ = orc.finalize_tree(s, tokens, torch.cat(parents), torch.zeros(1, dtype=torch.long), k, n_tree - 1, False)
    tm = tm[0, 0].bool()
    sel = torch.linspace(0, n_tree - 1, rows).round().long() if rows <= n_tree else torch.arange(rows) % n_tree
    out = []
    for r in sel.tolist():
        b = sum(1 << j for j in range(n_tree) if tm[r, j])
        out.append((b & (2 ** 64 - 1), b >> 64))
    return out


def straddle_masks(n_tree, rows, seed):
    """Masks that cross the word boundary: bits 62..65, bit 63 alone, bit 64 alone, the last column, everything."""
    g = torch.Generator().manual_seed(seed)
    pats = [(1 << 63) | (1 << 64), 1 << 64, 1 << 63, 0b1111 << 62, 1 << (n_tree - 1), (1 << n_tree) - 1, 1]
    out = []
    for r in range(rows):
        b = pats[r % len(pats)] | (int(torch.randint(0, 2 ** 62, (1,), generator=g)) if r % 3 == 0 else 0)
        b &= (1 << n_tree) - 1
        out.append((b & (2 ** 64 - 1), b >> 64))
    return out


def inputs(dtype, rows, nh, nkv, cap, kv_len, temp, seed):
    """q, K with S / sqrt(d) of standard deviation `temp` (peaked softmaxes for temp >> 1), V ~ N(0, 1); cache rows beyond
    kv_len hold large finite garbage."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = math.sqrt(temp)
    q = (torch.randn(rows, nh, 128, generator=g, device="cuda") * s).to(dtype)
    kc = (torch.randn(nkv, cap, 128, generator=g, device="cuda") * s).to(dtype)
    vc = torch.randn(nkv, cap, 128, generator=g, device="cuda").to(dtype)
    kc[:, kv_len:] = BIG[dtype]
    vc[:, kv_len:] = -BIG[dtype]
    return q, kc, vc


# (dtype, nh, nkv, max_kv, kv_len, rows, n_tree, masks, temp).  max_kv: engine buckets for max_length 512 (256, the target
# cap 576, the draft cap 700), 2048 (768, 1024, 2304) and 8192 (8192, the draft cap 8380), the largest accepted strip, and
# small strips without a KV split.  kv_len leaves cluster ranks idle or partly live, or fills the strip.
BF, FP = torch.bfloat16, torch.float16
SWEEP = [
    (BF, 32, 8, 768, 640, 60, 60, "tree", 1.0),
    (FP, 32, 8, 1024, 833, 10, 63, "tree", 4.0),
    (BF, 8, 1, 1024, 447, 17, 65, "straddle", 9.0),
    (FP, 20, 20, 576, 576, 64, 64, "causal", 1.0),
    (BF, 32, 32, 700, 700, 16, 128, "tree", 4.0),
    (FP, 2, 1, 256, 129, 1, 1, "tree", 9.0),
    (BF, 2, 1, 2304, 2240, 8, 8, "tree", 1.0),
    (FP, 8, 1, 8192, 5000, 16, 127, "straddle", 4.0),
    (BF, 32, 8, 8380, 8380, 60, 60, "tree", 9.0),
    (FP, 32, 8, MAX_KV, MAX_KV, 8, 8, "tree", 1.0),
    (BF, 8, 1, MAX_KV, 9000, 64, 128, "tree", 4.0),
    (FP, 20, 20, 2304, 1087, 17, 60, "tree", 9.0),
    (BF, 32, 32, 256, 64, 64, 64, "causal", 4.0),
    (FP, 2, 1, 192, 130, 60, 128, "straddle", 1.0),
    (BF, 32, 8, 8192, 8192, 10, 65, "straddle", 4.0),
    (BF, 8, 1, 256, 100, 10, 8, "tree", 9.0),
    (FP, 20, 20, 128, 70, 8, 8, "tree", 4.0),
    (FP, 40, 40, 768, 620, 60, 60, "tree", 4.0),  # Llama-2-13B's verify pass: fp16, 40 query / 40 kv heads
]


def _id(c):
    return f"{'bf16' if c[0] == BF else 'fp16'}-{c[1]}x{c[2]}-kv{c[3]}-len{c[4]}-r{c[5]}-t{c[6]}-{c[7]}-T{c[8]:g}"


def _masks(kind, n_tree, rows, seed):
    return None if kind == "causal" else (tree_masks if kind == "tree" else straddle_masks)(n_tree, rows, seed)


@pytest.mark.parametrize("case", SWEEP, ids=[_id(c) for c in SWEEP])
def test_engine_geometry_sweep(lib, case):
    dtype, nh, nkv, max_kv, kv_len, rows, n_tree, kind, temp = case
    geo, err = ar.attention_plan(lib, max_kv, nh, nkv)
    assert err is None, err
    hpc, kvs, stride, _ = geo
    tiles_per = (stride - 8) // 64
    n_ctx = kv_len - n_tree
    cap = max_kv + 24
    seed = max_kv + kv_len + rows
    q, kc, vc = inputs(dtype, rows, nh, nkv, cap, kv_len, temp, seed)
    masks = _masks(kind, n_tree, rows, seed)
    rc, got = launch(lib, dtype, q, kc, vc, max_kv, n_ctx, n_tree, masks)
    ok(lib, rc)
    o, bound, st = ar.tree_attention_ref(q, kc, vc, n_ctx, n_tree, masks, dtype, kv_len,
                                         ar.kernel_error_model(kv_len, kvs, tiles_per))
    live = -(-kv_len // 64)
    report(f"attention {_id(case)}: hpc {hpc} kvs {kvs}, live tiles per rank "
           f"{[max(0, min(live - r * tiles_per, tiles_per)) for r in range(kvs)]} of {tiles_per}; {st}")
    ar.check_against(got, o, bound, _id(case))


def test_sweep_covers_every_geometry_with_idle_ranks(lib):
    seen = set()
    for dtype, nh, nkv, max_kv, kv_len, *_ in SWEEP:
        hpc, kvs, stride, _ = ar.attention_plan(lib, max_kv, nh, nkv)[0]
        tiles_per = (stride - 8) // 64
        if kvs == 1 or -(-kv_len // 64) <= (kvs - 1) * tiles_per:  # the last rank has no live tile
            seen.add((hpc, kvs))
    assert seen >= {(h, k) for h in (1, 2) for k in (1, 2, 4)}, seen


# ----------------------------------------------------------------------------------------------
# exact addressing: one dominant column per head dimension, V encodes the column
# ----------------------------------------------------------------------------------------------
def _v_code(nkv, cap, dtype):
    c = torch.arange(cap)[None, :, None]
    g = torch.arange(nkv)[:, None, None]
    j = torch.arange(128)[None, None, :]
    v = ((c * 31 + j * 17 + g * 7) % 120 + 1) * (1 - 2 * (j % 2))
    v = v.expand(nkv, cap, 128).clone()
    v[:, :, 0] = (c[..., 0] >> 7) + 1
    v[:, :, 1] = (c[..., 0] & 127) + 1
    v[:, :, 2] = g[..., 0] + 1
    return v.to(dtype)  # integers of magnitude <= 133: exact in bf16 and fp16, never 0


@pytest.mark.parametrize("dtype,nh,nkv,max_kv,kv_len,n_tree,rows", [
    (BF, 8, 2, 1024, 900, 100, 64), (FP, 32, 8, MAX_KV, 12345, 128, 16), (BF, 4, 4, 700, 700, 64, 17), (FP, 2, 1, 192, 150, 65, 10),
    (FP, 8, 1, 8380, 8300, 60, 60),
])
def test_exact_addressing(lib, dtype, nh, nkv, max_kv, kv_len, n_tree, rows):
    """q(r, h) = 8 e_d; K = noise of at most 2^-7 plus K[t_d, d] = 40 (S / sqrt(d) ~ 28, a gap of ~28 to every other visible
    column) and a decoy K[u_d, d] = 48 on a column the row must not see (masked tree column, or beyond kv_len).  Then
    P[t_d] rounds to 1, every other P to ~e^-28, and the output must be V[t_d] bit for bit, for every (row, head)."""
    geo, err = ar.attention_plan(lib, max_kv, nh, nkv)
    assert err is None, err
    tiles_per = (geo[2] - 8) // 64
    n_ctx = kv_len - n_tree
    cap = max(max_kv, kv_len + 64) + 8
    n_rep = nh // nkv
    g = torch.Generator().manual_seed(kv_len + nh)
    masks = [((b | 1) & ((1 << n_tree) - 1) & (2 ** 64 - 1), ((b | 1) & ((1 << n_tree) - 1)) >> 64)
             for b in (int(torch.randint(0, 2 ** 62, (1,), generator=g)) | (int(torch.randint(0, 2 ** 62, (1,), generator=g)) << 62)
                       for _ in range(rows))]
    vis = ar.visible_mask(rows, n_ctx, n_tree, cap, masks)  # columns >= kv_len are never visible
    vis[:, kv_len:] = False
    special = [0, 63, 64, 65, n_ctx - 1, n_ctx, n_ctx + 63, n_ctx + 64, kv_len - 1, kv_len - 2]
    for r in range(1, geo[1]):
        special += [r * tiles_per * 64 - 1, r * tiles_per * 64]
    special += [t * 64 + o for t in range(0, -(-kv_len // 64), max(1, kv_len // 64 // 8)) for o in (0, 63)]
    kc = ((torch.randint(-2, 3, (nkv, cap, 128), generator=g)).double() * 2.0 ** -8).to(dtype)
    vc = _v_code(nkv, cap, dtype)
    q = torch.zeros(rows, nh, 128, dtype=dtype)
    want = torch.zeros(rows, nh, 128, dtype=dtype)
    for kvh in range(nkv):
        perm = torch.randperm(kv_len, generator=g).tolist()
        cand = [c for c in dict.fromkeys(special + perm) if 0 <= c < kv_len]
        targets = cand[:128]
        decoys = []
        for d in range(128):
            if d % 2 == 0:  # beyond kv_len (read by the last tile, or not at all)
                decoys.append(kv_len + (d * 7) % (cap - kv_len))
            else:  # a tree column, invisible to some rows
                decoys.append(n_ctx + (d * 13) % n_tree)
        for d in range(128):
            kc[kvh, targets[d], d] = 40
        for d in range(128):
            if decoys[d] not in targets:
                kc[kvh, decoys[d], d] = 48
        for r in range(rows):
            for hh in range(n_rep):
                h = kvh * n_rep + hh
                for i in range(128):
                    d = (r * 37 + h * 11 + i) % 128
                    u = decoys[d]
                    if vis[r, targets[d]] and (u in targets or not vis[r, u]):
                        break
                else:
                    pytest.fail(f"no usable dimension for row {r} head {h}")
                q[r, h, d] = 8
                want[r, h] = vc[kvh, targets[d]]
    rc, got = launch(lib, dtype, q.cuda(), kc.cuda(), vc.cuda(), max_kv, n_ctx, n_tree, masks)
    ok(lib, rc)
    got = got.cpu()
    bad = (got != want).any(-1)
    assert not bool(bad.any()), f"{int(bad.sum())} (row, head) pairs read the wrong column; first {bad.nonzero()[:6].tolist()}"


# ----------------------------------------------------------------------------------------------
# row count and prefix length from the device state (the draft stable pass: rows = D, st[S_ACC] valid, causal)
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF, FP])
def test_dynamic_rows_and_prefix(lib, dtype):
    D, nh, nkv, max_kv, n_ctx = 8, 8, 2, 1024, 777
    cap = max_kv + 8
    sentinel = -7.0
    q, kc, vc = inputs(dtype, D, nh, nkv, cap, n_ctx + D, 4.0, 11)
    for acc in range(1, D + 1):
        add = 3 * acc
        st = torch.tensor([n_ctx - add, acc, 0, 0], dtype=torch.int32, device="cuda")
        out = torch.full((D + 2, nh * 128), sentinel, dtype=dtype, device="cuda")
        rc, _ = launch(lib, dtype, q, kc, vc, max_kv, add, D, None, out=out, st=st, rows_idx=1, n_ctx_idx=0)
        ok(lib, rc)
        o, bound, _ = ar.tree_attention_ref(q[:acc], kc, vc, n_ctx, D, None, dtype)
        ar.check_against(out[:acc].view(acc, nh, 128), o, bound, f"acc {acc}")
        assert bool((out[acc:] == sentinel).all()), f"acc {acc}: rows at or beyond the valid count were written"


# ----------------------------------------------------------------------------------------------
# contract: what the kernel must not read or write
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF, FP])
def test_cache_rows_beyond_kv_len_and_other_planes_do_not_matter(lib, dtype):
    nh, nkv, kv_len, n_tree, rows = 8, 2, 1000, 60, 60
    cap = 1010  # the last 64-row tile of kv head 0 runs 14 rows into head 1's plane
    max_kv = cap
    masks = tree_masks(n_tree, rows, 5)
    q, kc, vc = inputs(dtype, rows, nh, nkv, cap, kv_len, 4.0, 5)
    kz, vz = kc.clone(), vc.clone()
    kz[:, kv_len:] = 0
    vz[:, kv_len:] = 0
    sentinel = -7.0
    out = torch.full((rows + 2, nh * 128), sentinel, dtype=dtype, device="cuda")
    ok(lib, launch(lib, dtype, q, kz, vz, max_kv, kv_len - n_tree, n_tree, masks, out=out)[0])
    assert bool((out[rows:] == sentinel).all()) and bool(torch.isfinite(out[:rows]).all())
    ref = out[:rows].clone()
    # rows [kv_len, cap) of every plane: large finite values instead of zeros
    rc, got = launch(lib, dtype, q, kc, vc, max_kv, kv_len - n_tree, n_tree, masks)
    ok(lib, rc)
    assert torch.equal(got.reshape(rows, -1), ref)
    # head 1's plane all garbage: the heads of kv head 0 do not change
    kh, vh = kz.clone(), vz.clone()
    kh[1] = BIG[dtype]
    vh[1] = -BIG[dtype]
    rc, got = launch(lib, dtype, q, kh, vh, max_kv, kv_len - n_tree, n_tree, masks)
    ok(lib, rc)
    assert torch.equal(got.reshape(rows, -1)[:, : nh // nkv * 128], ref[:, : nh // nkv * 128])
    # deterministic: the same call twice, bit for bit
    rc, again = launch(lib, dtype, q, kz, vz, max_kv, kv_len - n_tree, n_tree, masks)
    ok(lib, rc)
    assert torch.equal(again.reshape(rows, -1), ref)


# ----------------------------------------------------------------------------------------------
# every geometry the caps allow
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF, FP])
def test_forced_geometry(lib, dtype):
    nh, nkv, max_kv, kv_len, n_tree, rows = 8, 2, 448, 300, 65, 17  # 7 strip tiles, 5 live: idle / partial ranks at kvs 2 and 4
    n_ctx = kv_len - n_tree
    q, kc, vc = inputs(dtype, rows, nh, nkv, max_kv + 8, kv_len, 4.0, 21)
    masks = tree_masks(n_tree, rows, 21)
    o, bound, _ = ar.tree_attention_ref(q, kc, vc, n_ctx, n_tree, masks, dtype)
    ran = set()
    for hpc in (1, 2, 4):
        for kvs in (1, 2, 4):
            geo, err = ar.attention_plan(lib, max_kv, nh, nkv, hpc, kvs)
            assert err is None, err
            if geo[:2] != (hpc, kvs):
                continue
            rc, got = launch(lib, dtype, q, kc, vc, max_kv, n_ctx, n_tree, masks, hpc_cap=hpc, kvs_cap=kvs)
            ok(lib, rc)
            ar.check_against(got, o, bound, f"hpc {hpc} kvs {kvs}")
            ran.add((hpc, kvs))
    assert len(ran) == 9, ran


def test_strip_beyond_the_limit_is_refused(lib):
    dtype = BF
    q, kc, vc = inputs(dtype, 8, 2, 1, MAX_KV + 72, 100, 1.0, 3)
    rc, _ = launch(lib, dtype, q, kc, vc, MAX_KV + 1, 92, 8, None)
    assert rc != 0 and str(MAX_KV) in lib.eb200_last_error().decode()
    rc, _ = launch(lib, dtype, q, kc, vc, MAX_KV, 92, 8, None)
    ok(lib, rc)


# ----------------------------------------------------------------------------------------------
# engine at the limit
# ----------------------------------------------------------------------------------------------
def test_engine_max_length_limit():
    from eagle_b200 import EaModel
    from eagle_b200.synthetic import fixture_models, make_prompt
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models("e3_corr_bf16")
    longest = MAX_KV - 128 - tree["depth"] * tree["top_k"]
    with pytest.raises(Exception, match="max_length"):
        EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=longest + 1, **tree)
    m = EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=longest, **tree)
    prompt = make_prompt(tcfg["vocab_size"], longest - 150, 7).cuda()
    ids, new, idx = m.eagenerate(prompt, max_new_tokens=1000, max_length=longest, log=True)
    want, w_new, _ = m.naivegenerate(prompt, max_new_tokens=1000, max_length=longest, log=True)
    report(f"engine at max_length {longest}: {new} new tokens in {idx + 1} cycles")
    assert new > 60
    # the two loops stop at different lengths near max_length (ea_model.py:250, :298): compare what both generated
    n = min(ids.shape[1], want.shape[1])
    assert n >= prompt.shape[1] + 60
    assert ids[0, :n].cpu().tolist() == want[0, :n].cpu().tolist(), "speculative output differs from vanilla greedy"


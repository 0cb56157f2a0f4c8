"""CPU checks of the tree attention's test reference (tests/attention_ref.py) and of its launch geometry
(eb200_k_attention_plan, host only)."""
import math
import os

import pytest
import torch

from oracle import eagle_oracle as orc
from tests import attention_ref as ar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]


def _t(*xs):
    return torch.tensor(xs, dtype=torch.float64)


# ----------------------------------------------------------------------------------------------
# round to nearest even, float64 -> bf16 / fp16
# ----------------------------------------------------------------------------------------------
def test_rne_bf16_ties_and_double_rounding():
    e = 2.0 ** -8  # half an ulp of bf16 at 1
    x = _t(1 + e, 1 + 3 * e, 1 + e + 2.0 ** -30, -(1 + e + 2.0 ** -30), 1 + e - 2.0 ** -30, 2 - e / 2)
    want = _t(1.0, 1 + 4 * e, 1.0078125, -1.0078125, 1.0, 2.0)
    assert torch.equal(ar.rne(x, torch.bfloat16), want)
    # torch's cast rounds 1 + 2^-8 + 2^-30 to float32 first (-> the tie 1 + 2^-8), then the tie to even: 1.0
    assert float(ar.rne(_t(1 + e + 2.0 ** -30), torch.bfloat16)) != float(_t(1 + e + 2.0 ** -30).to(torch.bfloat16))


def test_rne_fp16_ties_and_double_rounding():
    e = 2.0 ** -11
    x = _t(1 + e, 1 + 3 * e, 1 + e + 2.0 ** -40, -(1 + e + 2.0 ** -40), 2048 + 1, 2048 + 3)
    want = _t(1.0, 1 + 4 * e, 1 + 2 * e, -(1 + 2 * e), 2048.0, 2052.0)
    assert torch.equal(ar.rne(x, torch.float16), want)


def test_rne_range_edges():
    # fp16: largest finite 65504, the tie 65520 goes to the even neighbour 65536 = overflow; subnormal spacing 2^-24
    got = ar.rne(_t(65519.99, 65520.0, -65520.0, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -25 + 2.0 ** -60, 0.0), torch.float16)
    assert torch.equal(got, _t(65504.0, math.inf, -math.inf, 0.0, 2.0 ** -23, 2.0 ** -24, 0.0))
    # bf16: largest finite (2 - 2^-7) 2^127, subnormal spacing 2^-133
    mx = float.fromhex("0x1.fep127")
    got = ar.rne(_t(mx + 2.0 ** 119, mx + 2.0 ** 119 - 2.0 ** 100, 2.0 ** -134, 3 * 2.0 ** -134), torch.bfloat16)
    assert torch.equal(got, _t(math.inf, mx, 0.0, 2.0 ** -132))


@pytest.mark.parametrize("dtype", DTYPES)
def test_rne_is_the_nearest_value(dtype):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(200000, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-20, 12, (200000,), generator=g).double())
    r = ar.rne(x, dtype)
    assert torch.equal(r.to(dtype).to(torch.float64), r), "not a value of the dtype"
    u = ar.ulp(x, dtype)
    err = (x - r).abs()
    assert bool((err <= u / 2).all())
    tie = err == u / 2
    assert bool(((r[tie] / ar.ulp(r[tie], dtype)) % 2 == 0).all()), "ties must go to the even neighbour"
    # from float32 a single rounding is what torch's own cast does
    x32 = x.float().double()
    assert torch.equal(ar.rne(x32, dtype), x32.to(dtype).double())


# ----------------------------------------------------------------------------------------------
# the reference against the oracle's eager attention
# ----------------------------------------------------------------------------------------------
def _masks(rows, n_tree, g):
    out = []
    for _ in range(rows):
        b = int(torch.randint(0, 2 ** 62, (1,), generator=g)) | (int(torch.randint(0, 2 ** 62, (1,), generator=g)) << 62)
        b = (b | 1) & ((1 << n_tree) - 1)
        out.append((b & (2 ** 64 - 1), b >> 64))
    return out


def _eager(q, kc, vc, n_ctx, n_tree, masks):
    rows, nh, _ = q.shape
    kv_len = n_ctx + n_tree
    vis = ar.visible_mask(rows, n_ctx, n_tree, kv_len, masks)
    m = torch.where(vis, 0.0, torch.finfo(torch.float32).min)
    out = orc.eager_attention(q.transpose(0, 1)[None], kc[None, :, :kv_len], vc[None, :, :kv_len], m[None, None], nh // kc.shape[0])
    return out[0].transpose(0, 1)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,nh,nkv,n_ctx,n_tree,temp,causal", [
    (10, 4, 2, 37, 10, 1.0, False), (16, 2, 1, 100, 70, 3.0, False), (8, 2, 2, 0, 8, 2.0, True), (5, 4, 1, 200, 128, 4.0, False),
])
def test_reference_agrees_with_eager_attention(rows, nh, nkv, n_ctx, n_tree, temp, causal, dtype):
    g = torch.Generator().manual_seed(rows * 31 + n_ctx)
    kv_len = n_ctx + n_tree
    q = (torch.randn(rows, nh, 128, generator=g) * math.sqrt(temp)).to(dtype)
    kc = (torch.randn(nkv, kv_len, 128, generator=g) * math.sqrt(temp)).to(dtype)
    vc = torch.randn(nkv, kv_len, 128, generator=g).to(dtype)
    masks = None if causal else _masks(rows, n_tree, g)
    got = _eager(q, kc, vc, n_ctx, n_tree, masks)
    # the eager path sums sequentially in fp32 on the CPU: its accumulation chains are the full reduction lengths
    model = dict(qk_err=2 * 128 * ar.U, pv_err=2 * kv_len * ar.U, sum_depth=kv_len, kvs=1)
    o, bound, st = ar.tree_attention_ref(q, kc, vc, n_ctx, n_tree, masks, dtype, model=model)
    ar.check_against(got, o, bound, "eager attention")
    # and the nominal chain rounds to the eager result almost everywhere
    same = ar.rne(o, dtype) == got.double()
    assert float(same.float().mean()) > 0.97, f"only {float(same.float().mean()):.3f} identical; {st}"
    # the CPU's sequential fp32 chains are 16 x longer than the kernel's MMA chains: fp16 scores are then often ambiguous
    assert st["median_ulps"] < (1.5 if dtype == torch.bfloat16 else 4.0), st


def test_reference_bound_rejects_a_wrong_column():
    """The bound is tight enough that attending one wrong column (a shifted tile) is out of bounds."""
    dtype = torch.bfloat16
    g = torch.Generator().manual_seed(5)
    rows, nh, n_ctx, n_tree = 8, 2, 150, 8
    q = (torch.randn(rows, nh, 128, generator=g) * 2).to(dtype)
    kc = (torch.randn(1, n_ctx + n_tree + 64, 128, generator=g) * 2).to(dtype)
    vc = torch.randn(1, n_ctx + n_tree + 64, 128, generator=g).to(dtype)
    o, bound, _ = ar.tree_attention_ref(q, kc, vc, n_ctx, n_tree, None, dtype)
    shifted = _eager(q, kc[:, 64:], vc[:, 64:], n_ctx, n_tree, None)  # every column read one tile late
    with pytest.raises(AssertionError):
        ar.check_against(shifted, o, bound)
    bad_mask = _eager(q, kc, vc, n_ctx, n_tree, [((1 << (r + 2)) - 1, 0) for r in range(rows)])  # one extra tree column
    with pytest.raises(AssertionError):
        ar.check_against(bad_mask, o, bound)


# ----------------------------------------------------------------------------------------------
# launch geometry (host only)
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    if os.environ.get("EB200_ATTN_HPC") or os.environ.get("EB200_ATTN_KVS"):
        pytest.skip("the attention tuning knobs change the default geometry")
    import __graft_entry__ as ge
    if not os.path.exists(os.path.join(ROOT, "eagle_b200", "libeagle_b200.so")):
        ge.build()
    from eagle_b200 import _lib
    return _lib.load()


def plan(lib, max_kv, nh, nkv, hpc_cap=0, kvs_cap=0):
    return ar.attention_plan(lib, max_kv, nh, nkv, hpc_cap, kvs_cap)


MAX_KV = 16896  # largest strip that fits in 220 KiB of shared memory (one head per CTA, 4-way KV split, 66 tiles per CTA)


# engine buckets (multiples of 256 rows) -> (kvs, 64-row tiles per cluster rank)
BUCKETS = {256: (2, 2), 512: (4, 2), 768: (4, 3), 1024: (4, 4), 1280: (4, 5), 1536: (4, 6), 1792: (4, 7), 2048: (4, 8),
           2304: (4, 9)}


@pytest.mark.parametrize("max_kv", sorted(BUCKETS))
def test_plan_at_engine_buckets(lib, max_kv):
    g, err = plan(lib, max_kv, 32, 8)
    assert err is None, err
    hpc, kvs, stride, smem = g
    assert (kvs, (stride - 8) // 64) == BUCKETS[max_kv] and stride % 64 == 8
    assert hpc == 2 and smem <= 220 * 1024


def test_plan_small_strips_do_not_split(lib):
    for max_kv, kvs in ((64, 1), (192, 1), (193, 2), (384, 2), (385, 4)):
        g, err = plan(lib, max_kv, 2, 1)
        assert err is None and g[1] == kvs, (max_kv, g, err)


def test_plan_hpc_switch_and_limit(lib):
    assert plan(lib, 8192, 32, 8)[0][0] == 2
    assert plan(lib, 8193, 32, 8)[0][0] == 1  # the 2-head strip no longer fits: Llama-3-8B falls back to one head per CTA
    assert plan(lib, 8192, 20, 20)[0][0] == 1  # no GQA: one head per CTA at any length
    g, err = plan(lib, MAX_KV, 32, 8)
    assert err is None and g[:3] == (1, 4, 66 * 64 + 8) and g[3] <= 220 * 1024
    g, err = plan(lib, MAX_KV + 1, 32, 8)
    assert g is None and str(MAX_KV) in err


def test_plan_caps(lib):
    assert plan(lib, 1024, 32, 8, hpc_cap=4)[0][0] == 4
    assert plan(lib, 1024, 32, 8, hpc_cap=1)[0][0] == 1
    assert plan(lib, 1024, 32, 8, kvs_cap=1)[0][1:3] == (1, 16 * 64 + 8)
    assert plan(lib, 1024, 32, 8, kvs_cap=2)[0][1] == 2
    assert plan(lib, 1024, 20, 20, hpc_cap=4)[0][0] == 1  # 4 heads per CTA need n_rep % 4 == 0
    assert plan(lib, 4096, 32, 8, hpc_cap=4)[0][0] == 2  # the 4-head strip of 1032 columns does not fit
    for bad in ((3, 0), (0, 8), (-1, 0)):
        g, err = plan(lib, 1024, 32, 8, *bad)
        assert g is None and err, bad
    assert plan(lib, 1024, 32, 6)[0] is None  # heads must be a multiple of kv heads

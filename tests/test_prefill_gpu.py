"""Prompt prefill through the 256-row path against the CPU oracle and against the 64-row path.

On one GPU the engine runs a prompt through the target in 256-row chunks: the GEMMs launch 256 activation rows (wgmma N = 256)
and causal attention runs in four 64-row blocks per chunk.  Everything a later cycle reads comes out of this pass: the target
KV cache, the first token and, through the EAGLE-3 feature taps, the draft head's stable KV.  The prompt lengths put the chunk
boundaries where they bite: 65 (smallest 256-row chunk), 129, 256 (one full chunk), 257 (a 1-row second chunk, 16-row launch),
321 (a 65-row second chunk, 256-row launch again) and 700 (chunks of 256, 256 and 188).

Bars against the oracle (as tests/test_tree_geometry_gpu.py's committed-KV check): every K/V row within relative L2 distance
0.05, and the first layer's K/V (three rounding points: RMSNorm, GEMM, RoPE) within 1e-3 + 2 ulp element-wise; for the target's
layer-0 K that bar adds two ulp of each RoPE product (see kv_bars), which only matters where the products cancel.  Against the
engine built with EB200_PREFILL_ROWS=64 -- the path the kernel and end-to-end tests cover, one 64-row chunk at a time -- the
prefill must be bit-identical: the 256-row GEMM sums every output element in the same order as the 64-row launches
(tests/test_kernels_gpu.py::test_256_rows_equal_64_row_launches_bit_for_bit), and the attention blocks see the same columns.
"""
import pytest
import torch
import torch.nn.functional as F

from eagle_b200.synthetic import make_prompt
from oracle import eagle_oracle as orc
from tests.fixtures import report
from tests.test_tree_geometry_gpu import DEFAULT, ULP, compare_cycles, engine, oracle, prompt_of, weights

pytestmark = pytest.mark.gpu

MAX_LEN = 1024
BASES = ["e3_corr_bf16", "e1_corr_fp16", "e3_gqa_bf16"]
LENGTHS = [65, 129, 256, 257, 321, 700]


@pytest.fixture(scope="module")
def engines():
    """Per fixture: (weights, 256-row engine, 64-row engine, oracle), built once and reused across prompt lengths."""
    cache = {}

    def get(base):
        if base not in cache:
            w = weights(base)
            m256 = engine(w, DEFAULT, max_length=MAX_LEN)
            with pytest.MonkeyPatch.context() as mp:
                mp.setenv("EB200_PREFILL_ROWS", "64")  # read when the engine is created
                m64 = engine(w, DEFAULT, max_length=MAX_LEN)
            cache[base] = (w, m256, m64, oracle(w, DEFAULT))
        return cache[base]

    return get


def planes(m, what, P):
    """Rows [0, P) of the engine's K/V planes ("target_kv" / "draft_kv"): [planes, P, 128], plane (2 * layer + k/v) * nkv + head."""
    t = m.debug_read(what)
    return t.view(t.shape[0], -1, 128)[:, :P]


def oracle_prefill(ref, prompt):
    """(first token, target KV [2L * nkv, P, 128], draft stable KV after the first tree [2 * layers * nkv, P, 128])."""
    P = prompt.shape[1]
    kv = ref._kv(MAX_LEN)
    hidden, taps = ref.target.forward(prompt, kv)
    first = int(torch.argmax(ref.target.lm_head(hidden)[0, -1]))
    ref.head.reset_kv()
    ref._tree(ref._features(hidden, taps), torch.cat((prompt, torch.tensor([[first]])), dim=1), False)
    tkv = kv.data[:, 0, :, :P].float()
    dkv = torch.cat([t[0].float() for layer in ref.head.stable_kv for t in layer])
    assert dkv.shape[1] == P
    return first, tkv.reshape(-1, P, 128), dkv


def target_rope_terms(ref, prompt):
    """|k c| + |rotate_half(k) s| of the oracle's layer-0 K before RoPE, zeros for the V planes: [2 * nkv, P, 128].  A one-ulp
    flip of the projection k moves the rotated value by an ulp of these products; where they cancel (a long K sum at H = 4096,
    large angles) that is many ulps of the result."""
    tgt, P = ref.target, prompt.shape[1]
    cfg, W = tgt.cfg, tgt.W
    h = orc.rms_norm(F.embedding(prompt, W["model.embed_tokens.weight"]), W["model.layers.0.input_layernorm.weight"], cfg.rms_norm_eps)
    k = F.linear(h, W["model.layers.0.self_attn.k_proj.weight"]).view(P, cfg.num_key_value_heads, cfg.head_dim).transpose(0, 1).float()
    c, s = tgt.cos[:P].float(), tgt.sin[:P].float()
    terms = (k * c).abs() + (orc._rotate_half(k) * s).abs()
    return torch.cat((terms, torch.zeros_like(terms)))


def kv_bars(got, want, n_first, dtype, what, terms=None):
    """The oracle bars on K/V planes [planes, P, 128]: (failure messages, worst row distance per row [P], worst layer-0
    element error as a multiple of its tolerance).  terms: target_rope_terms for the layer-0 planes, or None."""
    d = (got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-6)
    fails = []
    if float(d.max()) >= 0.05:
        fails.append(f"{what}: {int((d >= 0.05).sum())} rows beyond relative distance 0.05, first (plane, row) {(d >= 0.05).nonzero()[:8].tolist()}")
    err = (got[:n_first] - want[:n_first]).abs()
    tol = 1e-3 + 2 * ULP[dtype] * (want[:n_first].abs() + (0 if terms is None else terms))
    worst = float((err / tol).max())
    if worst > 1.0:
        fails.append(f"{what}: layer-0 K/V: {int((err > tol).sum())} elements beyond 1e-3 + 2 ulp, worst {worst:.2f} x tolerance")
    return fails, d.max(0).values, worst


def by_block(rows_worst):
    """Worst row distance for each 64-row block position (0..3) of a 256-row chunk."""
    blk = (torch.arange(rows_worst.numel()) % 256) // 64
    return [round(float(rows_worst[blk == b].max()), 4) if bool((blk == b).any()) else None for b in range(4)]


@pytest.mark.parametrize("P", LENGTHS)
@pytest.mark.parametrize("base", BASES)
def test_prefill_matches_the_oracle_and_the_64_row_path(engines, base, P):
    w, m256, m64, ref = engines(base)
    tcfg, _, hcfg, _, _, dtype = w
    prompt = prompt_of(base, w, P)
    first, tkv_want, dkv_want = oracle_prefill(ref, prompt)
    got = {}
    for name, m in (("256", m256), ("64", m64)):
        tok = m.prefill(prompt.cuda())
        got[name] = (tok, planes(m, "target_kv", P), planes(m, "draft_kv", P))
    tok, tkv, dkv = got["256"]
    f_t, rows_t, worst_t = kv_bars(tkv, tkv_want, 2 * tcfg["num_key_value_heads"], dtype, "target KV", target_rope_terms(ref, prompt))
    f_d, rows_d, worst_d = kv_bars(dkv, dkv_want, 2 * hcfg["num_key_value_heads"], dtype, "draft KV")
    same = [tok == got["64"][0], torch.equal(tkv, got["64"][1]), torch.equal(dkv, got["64"][2])]
    report(f"prefill {base} P={P}: worst row distance to the oracle per 64-row block of a 256-row chunk: target {by_block(rows_t)}, "
           f"draft {by_block(rows_d)}; layer-0 worst {worst_t:.2f} / {worst_d:.2f} x (1e-3 + 2 ulp); "
           f"bit-identical to the 64-row path (first token, target KV, draft KV): {same}")
    assert tok == first, f"first token {tok}, the oracle's {first}"
    assert not f_t + f_d, "; ".join(f_t + f_d)
    assert all(same), f"the 256-row prefill differs from the 64-row prefill (first token, target KV, draft KV): {same}"


@pytest.mark.parametrize("P", [321, 700])
def test_eagle3_draft_kv_carries_the_feature_taps(P):
    """The EAGLE-3 copy heads of the fixtures have fc = 0, so their draft KV depends on the prompt tokens alone.  With a random
    fc the V planes carry norm(fc(taps)): the target's residual stream at three layers, written at every row of every chunk.
    Bars: the oracle's row distance, and bit identity with the 64-row path."""
    base = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype = weights(base)
    g = torch.Generator().manual_seed(5)
    fc = hW["fc.weight"]
    hW = dict(hW, **{"fc.weight": (torch.randn(fc.shape, generator=g) / fc.shape[1] ** 0.5).to(fc.dtype)})
    w = (tcfg, tW, hcfg, hW, eagle3, dtype)
    m = engine(w, DEFAULT, max_length=MAX_LEN)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("EB200_PREFILL_ROWS", "64")
        m64 = engine(w, DEFAULT, max_length=MAX_LEN)
    prompt = prompt_of(base, w, P)
    first, _, want = oracle_prefill(oracle(w, DEFAULT), prompt)
    assert m.prefill(prompt.cuda()) == first == m64.prefill(prompt.cuda())
    got = planes(m, "draft_kv", P)
    fails, rows, worst = kv_bars(got, want, got.shape[0], dtype, "draft KV")
    report(f"prefill EAGLE-3 draft KV with a random fc, P={P}: worst row distance to the oracle per 64-row block of a 256-row "
           f"chunk {by_block(rows)}; worst element {worst:.2f} x (1e-3 + 2 ulp)")
    assert not [f for f in fails if "relative distance" in f], fails
    assert torch.equal(got, planes(m64, "draft_kv", P)), "the draft KV differs from the 64-row prefill's"


def test_a_reused_engine_prefills_like_a_fresh_one():
    """A 700-token prefill leaves its rows in the 256-row activation buffers and the caches; a shorter prompt prefilled next
    must not see any of them."""
    base = "e3_corr_bf16"
    w = weights(base)
    long_prompt = prompt_of(base, w, 700)
    short = make_prompt(w[0]["vocab_size"], 300, 99)
    m, fresh = engine(w, DEFAULT, max_length=MAX_LEN), engine(w, DEFAULT, max_length=MAX_LEN)
    m.prefill(long_prompt.cuda())
    tok, tok_fresh = m.prefill(short.cuda()), fresh.prefill(short.cuda())
    assert tok == tok_fresh
    for what in ("target_kv", "draft_kv"):
        assert torch.equal(planes(m, what, 300), planes(fresh, what, 300)), f"{what} after a 700-token prefill differs from a fresh engine's"
    for a, b in zip(m.get_tree(), fresh.get_tree()):
        assert torch.equal(a, b), "the first draft tree differs from a fresh engine's"


def test_generation_after_a_321_token_prompt_identical_to_the_oracle():
    """A 65-row second chunk, then cycles that attend over all 321 prompt rows."""
    base = "e3_corr_bf16"
    w = weights(base)
    compare_cycles(engine(w, DEFAULT, max_length=MAX_LEN), oracle(w, DEFAULT), prompt_of(base, w, 321), DEFAULT, "321-token prompt",
                   new_tokens=32, max_length=MAX_LEN)

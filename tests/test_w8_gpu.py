"""`load_in_8bit` on the H100: int8 target projections (EB200_FLAG_TARGET_INT8) through the W8A16 GEMM.

The contract (eagle_b200/quant.py) makes an int8 engine compute exactly what a model-dtype engine loaded with
W' = dequantize_int8_rowwise(q, SCB) computes, so every comparison here is bit for bit against that twin: the kernel against
the model-dtype kernel on W', and whole generations (trees, verify results, committed tokens, KV) against a bf16 / fp16
engine built from W'.
"""
import ctypes as C

import pytest
import torch

from eagle_b200 import quant, static_trees
from eagle_b200.synthetic import FIXTURES, base_fixture, fixture_models, make_prompt
from oracle import eagle_oracle as orc
from tests.fixtures import report, to_cfg

pytestmark = pytest.mark.gpu

DT = {torch.bfloat16: 0, torch.float16: 1}
EPI = {"store": 0, "residual": 1, "swiglu": 5}


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def engine_splitk(N, K):
    """The engine's split-K policy (engine.cu pick_splitk): smallest power of two giving >= 100 CTAs, >= 4 k-blocks each."""
    tiles, kb, sk = (N + 127) // 128, (K + 63) // 64, 1
    while sk < 8 and tiles * sk < 100:
        sk *= 2
    while sk > 1 and kb // sk < 4:
        sk //= 2
    return sk


def quantized(N, K, seed, dtype, device="cuda"):
    """(q, scb, W') of a random weight with an all-zero row and rows whose absmax is on either sign (q = +-127)."""
    g = torch.Generator(device=device).manual_seed(seed)
    w = (torch.randn(N, K, generator=g, device=device) * 0.02).to(dtype)
    w[min(5, N - 1)] = 0
    w[0, 3] = 0.5
    w[N - 1, K - 1] = -0.5
    q, scb = quant.quantize_int8_rowwise(w)
    return q, scb, quant.dequantize_int8_rowwise(q, scb, dtype)


# ----------------------------------------------------------------------------------------------
# 1. the kernel: eb200_k_gemm_w8 == eb200_k_gemm (cluster split-K) on W', bit for bit
# ----------------------------------------------------------------------------------------------
SHAPES = {  # N (output rows; SwiGLU: output columns over a [2N, K] interleaved weight), K
    "store": [(256, 256), (200, 320), (6144, 4096)],          # tiny, N % 128 != 0, Llama-3-8B qkv
    "residual": [(384, 768), (4096, 4096), (4096, 14336)],   # o_proj, down_proj
    "swiglu": [(320, 256), (14336, 4096)],                   # gate/up
}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("epi", ["store", "residual", "swiglu"])
def test_w8_gemm_bitwise_equal_to_the_gemm_on_dequantized_weights(lib, epi, dtype):
    n_cmp = 0
    for N, K in SHAPES[epi]:
        rows = 2 * N if epi == "swiglu" else N
        q, scb, wd = quantized(rows, K, N + K, dtype)
        g = torch.Generator(device="cuda").manual_seed(K)
        X = (torch.randn(256, K, generator=g, device="cuda") * 0.5).to(dtype)  # 256 rows: the prefill launch reads them all
        bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(dtype) if epi == "store" else None
        res = torch.randn(256, N, generator=g, device="cuda").to(dtype) if epi == "residual" else None
        torch.cuda.synchronize()
        for M in (1, 10, 16, 60, 64) + (() if epi == "store" else (65, 200, 256)):  # > 64: the prompt prefill's 256-row launch
            for sk in sorted({1, engine_splitk(rows, K)}):
                outs = []
                for w8 in (True, False):
                    out = res.clone() if res is not None else torch.zeros(256, N, dtype=dtype, device="cuda")
                    torch.cuda.synchronize()
                    rp = C.c_void_p(out.data_ptr()) if res is not None else None
                    bp = C.c_void_p(bias.data_ptr()) if bias is not None else None
                    if w8:
                        rc = lib.eb200_k_gemm_w8(DT[dtype], EPI[epi], C.c_void_p(q.data_ptr()), C.c_void_p(scb.data_ptr()),
                                                 C.c_void_p(X.data_ptr()), C.c_void_p(out.data_ptr()), rp, bp, M, N, K, sk, None)
                    else:
                        rc = lib.eb200_k_gemm(DT[dtype], 2, EPI[epi], C.c_void_p(wd.data_ptr()), None, C.c_void_p(X.data_ptr()),
                                              C.c_void_p(out.data_ptr()), rp, bp, M, N, K, sk, None)
                    check(lib, rc)
                    outs.append(out)
                a, b = outs
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{epi} M={M} N={N} K={K} splitk={sk}"
                want = res[M:] if res is not None else torch.zeros_like(a[M:])
                assert torch.equal(a[M:].view(torch.int16), want.view(torch.int16))  # rows beyond M are never written
                n_cmp += 1
    assert n_cmp >= 10


def test_w8_gemm_rejects_what_it_does_not_run(lib):
    q = torch.zeros(128, 64, dtype=torch.int8, device="cuda")
    scb = torch.zeros(128, device="cuda")
    X = torch.zeros(64, 64, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(64, 128, dtype=torch.bfloat16, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.eb200_k_gemm_w8(0, 2, p(q), p(scb), p(X), p(out), None, None, 4, 128, 64, 1, None) != 0  # two-matrix SwiGLU
    assert lib.eb200_k_gemm_w8(0, 0, p(q), p(scb), p(X), p(out), None, None, 65, 128, 64, 1, None) != 0  # store at 256 rows
    assert lib.eb200_k_gemm_w8(0, 1, p(q), p(scb), p(X), p(out), p(out), None, 257, 128, 64, 1, None) != 0  # M > 256
    assert lib.eb200_k_gemm_w8(0, 0, p(q), None, p(X), p(out), None, None, 4, 128, 64, 1, None) != 0  # no scales


# ----------------------------------------------------------------------------------------------
# 2. whole generations: int8 engine == model-dtype engine on W'
# ----------------------------------------------------------------------------------------------
def split_weights(tW, dtype):
    """(int8 state dict: q + SCB for the projections, W' state dict: the dequantized projections); other tensors shared."""
    t8, tp = {}, {}
    for k, v in tW.items():
        if quant.is_target_projection(k):
            q, scb = quant.quantize_int8_rowwise(v.to(dtype))
            t8[k], t8[k[: -len("weight")] + "SCB"] = q, scb
            tp[k] = quant.dequantize_int8_rowwise(q, scb, dtype)
        else:
            t8[k] = tp[k] = v
    return t8, tp


def twins(fx, max_length=512, quantize_at_load=False, **kw):
    """(int8 engine, model-dtype engine on W', prompt, gen kwargs, sampling seed) for a named fixture."""
    from eagle_b200 import EaModel
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(base_fixture(fx))
    tree = dict(tree, **kw)
    t8, tp = split_weights(tW, dtype)
    common = dict(use_eagle3=eagle3, torch_dtype=dtype, max_length=max_length, **tree)
    m8 = EaModel.from_state_dicts(tcfg, tW if quantize_at_load else t8, hcfg, hW, load_in_8bit=True, **common)
    mb = EaModel.from_state_dicts(tcfg, tp, hcfg, hW, **common)
    plen, pseed, gen_kw, seed = FIXTURES[fx]
    return m8, mb, make_prompt(tcfg["vocab_size"], plen, pseed), gen_kw, seed


def run_cycles(m, prompt, n):
    first = m.prefill(prompt.cuda())
    out = [first]
    for _ in range(n):
        dt, ri, tm, tp = m.get_tree()
        toks, nxt = m.step()
        am, best, acc, committed = m.get_verify()
        out.append((dt, ri, tm, tp, toks, nxt, am, best, acc, committed))
    return out


def same(a, b):
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("fx,static", [("e3_rand_bf16", False), ("e3_corr_bf16", False), ("e3_gqa_bf16", False),
                                       ("e1_corr_fp16", False), ("e3_corr_bf16", True)])
def test_int8_engine_identical_to_the_engine_on_dequantized_weights(fx, static):
    kw = dict(tree_choices=static_trees.mc_sim_7b_63) if static else {}
    m8, mb, prompt, gen_kw, _ = twins(fx, quantize_at_load=(fx == "e3_gqa_bf16"), **kw)
    a = m8.eagenerate(prompt.cuda(), log=True, **gen_kw)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    n = a[2] + 1
    ca, cb = run_cycles(m8, prompt, n), run_cycles(mb, prompt, n)
    assert ca[0] == cb[0]
    for c in range(1, n + 1):
        assert same(ca[c], cb[c]), f"cycle {c - 1}: tree / verify / committed tokens differ"
    if fx == "e3_corr_bf16" and not static:
        accs = [c[8] for c in ca[1:]]
        assert max(accs) >= 3 and min(accs) == 0, f"the fixture must exercise long and empty accepts: {accs}"
    want = mb.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    got = m8.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:]
    for gen in ("ea_generate", "naive_generate"):
        ga = [t.cpu().tolist() for t in getattr(m8, gen)(prompt.cuda(), **gen_kw)]
        gb = [t.cpu().tolist() for t in getattr(mb, gen)(prompt.cuda(), **gen_kw)]
        assert ga == gb, gen
    report(f"int8 {fx}{' static tree' if static else ''}: {a[1]} tokens in {a[2] + 1} cycles, identical to the W' twin")


@pytest.mark.parametrize("fx", ["e3_corr_bf16_T1", "e3_corr_bf16_T07"])
def test_int8_sampling_identical_to_the_engine_on_dequantized_weights(fx):
    m8, mb, prompt, gen_kw, seed = twins(fx)
    torch.manual_seed(seed)
    a = m8.eagenerate(prompt.cuda(), log=True, **gen_kw)
    torch.manual_seed(seed)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    torch.manual_seed(seed)
    a = m8.naivegenerate(prompt.cuda(), **gen_kw)
    torch.manual_seed(seed)
    b = mb.naivegenerate(prompt.cuda(), **gen_kw)
    assert a.cpu().tolist() == b.cpu().tolist()


def test_int8_prefill_of_a_long_prompt_uses_the_256_row_path():
    """A 300-token prompt is prefilled in 256-row chunks (MPAD 256): the target KV cache after prefill is identical."""
    m8, mb, _, gen_kw, _ = twins("e3_corr_bf16")
    prompt = make_prompt(m8.vocab_size, 300, 31)
    assert m8.prefill(prompt.cuda()) == mb.prefill(prompt.cuda())
    ka, kb = m8.debug_read("target_kv"), mb.debug_read("target_kv")
    assert torch.equal(ka, kb) and float(ka.abs().sum()) > 0
    a = m8.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    b = mb.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]


# ----------------------------------------------------------------------------------------------
# 3. oracle anchor: the CPU oracle on W' gives the int8 engine's tokens
# ----------------------------------------------------------------------------------------------
ULP = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}


def test_int8_engine_matches_the_oracle_on_dequantized_weights():
    from eagle_b200 import EaModel
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    t8, tp = split_weights(tW, dtype)
    m8 = EaModel.from_state_dicts(tcfg, t8, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, load_in_8bit=True, **tree)
    plen, pseed, gen_kw, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed)
    ids = m8.eagenerate(prompt.cuda(), **gen_kw).cpu()
    ref = orc.OracleEaModel(to_cfg(tcfg), {k: v.cpu() for k, v in tp.items()}, to_cfg(hcfg), hW, eagle3, **tree)
    want = ref.eagenerate(prompt, **gen_kw)
    k = min(ids.shape[1], want.shape[1])
    agree = int((ids[0, :k] == want[0, :k]).long().cumprod(0).sum())
    # margin-aware bar (tests/test_e2e_gpu.py): every generated token up to the oracle's first sub-2-ulp top-2 decision
    hidden, _ = ref.target.forward(want[:, : k - 1], ref._kv(512))
    logits = ref.target.lm_head(hidden)[0, plen - 1:].float()
    top2 = logits.topk(2, dim=-1).values
    spacing = torch.exp2(torch.floor(torch.log2(top2[:, 0].abs().clamp_min(1e-30)))) * ULP[dtype]
    fragile = ((top2[:, 0] - top2[:, 1]) / spacing < 2.0).nonzero().flatten()
    must = int(fragile[0]) if fragile.numel() else k - plen
    report(f"int8 vs oracle on W': identical generated prefix {agree - plen}/{k - plen}, first fragile decision at {must}")
    assert agree - plen >= must


# ----------------------------------------------------------------------------------------------
# 4. Llama-3-8B width (8 layers): identical generation and draft logits, and the device memory saved
# ----------------------------------------------------------------------------------------------
def test_int8_at_llama3_8b_width_identical_and_smaller():
    from eagle_b200 import EaModel, synthetic as syn
    dtype = torch.bfloat16
    tree = dict(total_token=60, depth=6, top_k=10)
    tcfg, tW, hcfg, hW = syn.correlated_llama3_eagle3(8, dtype, "cuda")
    t8, tp = split_weights(tW, dtype)
    proj_bf16 = sum(v.numel() * 2 for k, v in tW.items() if quant.is_target_projection(k))
    del tW
    used = syn.draft_vocab_ids(tcfg["vocab_size"], hcfg["draft_vocab_size"])
    prompt = used[torch.randint(0, used.numel(), (700,), generator=torch.Generator().manual_seed(77))][None]

    def build(sd, **kw):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        m = EaModel.from_state_dicts(tcfg, sd, hcfg, hW, use_eagle3=True, torch_dtype=dtype, max_length=1100, **tree, **kw)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return m, free0 - torch.cuda.mem_get_info()[0]

    m8, used8 = build(t8, load_in_8bit=True)
    mb, usedb = build(tp)
    report(f"int8 at Llama-3-8B width, 8 layers: create + load takes {used8 / 1e9:.3f} GB vs {usedb / 1e9:.3f} GB in bf16 "
           f"(target projections {proj_bf16 / 1e9:.3f} GB in bf16)")
    assert proj_bf16 == 8 * 218103808 * 2
    assert usedb - used8 >= 0.4 * proj_bf16
    a = m8.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    b = mb.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    assert a[0].shape[1] > 832, "generation must cross the 1024-row KV bucket"
    assert m8.prefill(prompt.cuda()) == mb.prefill(prompt.cuda())
    for c in range(a[2] + 1):
        sa, sb = m8.step(), mb.step()
        va, vb = m8.get_verify(), mb.get_verify()
        assert sa == sb and va[2] == vb[2], f"cycle {c}: committed tokens / accept length differ"
        if c == 0:
            assert torch.equal(m8.debug_read("draft_logits"), mb.debug_read("draft_logits"))


# ----------------------------------------------------------------------------------------------
# 5. loading: from_pretrained(load_in_8bit=True) on bf16 and on bitsandbytes-8-bit directories; refused combinations
# ----------------------------------------------------------------------------------------------
def test_from_pretrained_load_in_8bit(tmp_path):
    from eagle_b200 import EaModel
    from eagle_b200.checkpoint import save_head_checkpoint, save_target_checkpoint
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    t8, _ = split_weights(tW, dtype)
    plen, pseed, gen_kw, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed).cuda()
    want = EaModel.from_state_dicts(tcfg, t8, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, load_in_8bit=True,
                                    **tree).eagenerate(prompt, log=True, **gen_kw)
    hdir = str(tmp_path / "head")
    save_head_checkpoint(hdir, hcfg, hW)
    bf16_dir, int8_dir = str(tmp_path / "bf16"), str(tmp_path / "int8")
    save_target_checkpoint(bf16_dir, tcfg, tW)
    stored = dict(t8)
    for k in list(stored):
        if k.endswith(".SCB"):
            stored[k[: -len("SCB")] + "weight_format"] = torch.tensor(0, dtype=torch.uint8)
    save_target_checkpoint(int8_dir, dict(tcfg, quantization_config={"quant_method": "bitsandbytes", "load_in_8bit": True}), stored)
    for d, kw in ((bf16_dir, dict(load_in_8bit=True)), (int8_dir, {})):
        m = EaModel.from_pretrained(use_eagle3=eagle3, base_model_path=d, ea_model_path=hdir, torch_dtype=dtype, max_length=512, **kw, **tree)
        assert m.load_in_8bit
        got = m.eagenerate(prompt, log=True, **gen_kw)
        assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:], d


def test_int8_loader_refuses_mismatched_tensors():
    from eagle_b200 import EaModel, _lib
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models("e3_corr_bf16")
    t8, _ = split_weights(tW, dtype)
    m = EaModel(tcfg, hcfg, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, load_in_8bit=True, **tree)
    with pytest.raises(_lib.EngineError, match="int8"):  # model-dtype data for an int8 projection
        m._load("model.layers.0.mlp.down_proj.weight", tW["model.layers.0.mlp.down_proj.weight"])
    with pytest.raises(_lib.EngineError, match="only for the target decoder projections"):
        m._load("lm_head.weight", t8["model.layers.0.mlp.down_proj.weight"])
    with pytest.raises(_lib.EngineError, match="SCB row scales missing"):
        m.load_target_state_dict({k: v for k, v in t8.items() if k != "model.layers.1.self_attn.k_proj.SCB"})
        m.load_head_state_dict(hW)
        m.finalize()
    mb = EaModel(tcfg, hcfg, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, **tree)
    with pytest.raises(_lib.EngineError, match="without EB200_FLAG_TARGET_INT8"):
        mb._load("model.layers.0.mlp.down_proj.weight", t8["model.layers.0.mlp.down_proj.weight"])

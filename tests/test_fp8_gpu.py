"""FP8 target weights on the H100: transformers' fine-grained e4m3 projections (EB200_FLAG_TARGET_FP8) through the W8A16 GEMM.

The contract (eagle_b200/quant.py) makes an FP8 engine compute exactly what a model-dtype engine loaded with
W' = dequantize_fp8_block(q, scale_inv) computes, so every comparison here is bit for bit against that twin: the kernel against the
model-dtype kernel on W', and whole generations (trees, verify results, committed tokens, draft logits, KV) against a bf16 / fp16
engine built from W'.  The model-width cases run in subprocesses so that no module fixture holds their memory.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from eagle_b200 import quant, static_trees
from eagle_b200.synthetic import FIXTURES, base_fixture, fixture_models, make_prompt
from oracle import eagle_oracle as orc
from tests.fixtures import report, to_cfg
from tests.test_w8_gpu import ULP, engine_splitk, run_cycles, same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {torch.bfloat16: 0, torch.float16: 1}
EPI = {"store": 0, "residual": 1, "swiglu": 5}
FP8 = {"quant_method": "fp8", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def coded(N, K, seed, dtype):
    """(q, scale_inv, W') with every finite e4m3 byte in block (0, 0), an all-zero block, and a block whose products include model-dtype
    subnormals (its scale times the small e4m3 codes)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    codes = torch.randint(0, 256, (N, K), generator=g, device="cuda", dtype=torch.int32)
    codes.view(-1)[:256] = torch.arange(256, device="cuda")  # the first rows of block (0, 0)
    codes[(codes & 0x7F) == 0x7F] = 0x7E  # the two NaN encodings
    codes[-128:, -128:] = 0
    q = codes.to(torch.uint8).view(torch.float8_e4m3fn)
    scale = torch.exp2(torch.randint(-11, -6, (N // 128, K // 128), generator=g, device="cuda").float())
    scale *= 1 + torch.rand(N // 128, K // 128, generator=g, device="cuda")
    scale[0, 0] = 2e-38 if dtype == torch.bfloat16 else 1e-6
    wd = quant.dequantize_fp8_block(q, scale, dtype)
    tiny = torch.finfo(dtype).tiny
    assert bool(((wd[:128, :128].float().abs() < tiny) & (wd[:128, :128] != 0)).any())
    return q, scale, wd


# ----------------------------------------------------------------------------------------------
# 1. the kernel: eb200_k_gemm_fp8 == eb200_k_gemm (cluster split-K) on W', bit for bit
# ----------------------------------------------------------------------------------------------
SHAPES = {  # N (output rows; SwiGLU: output columns over a [2N, K] interleaved weight), K
    "store": [(256, 256), (384, 128), (6144, 4096), (10240, 8192)],         # tiny, K = 128, 8B / 70B qkv
    "residual": [(384, 768), (4096, 4096), (4096, 14336), (8192, 8192)],   # 8B o / down, 70B o
    "swiglu": [(320, 256), (14336, 4096), (28672, 8192)],                   # 8B / 70B gate/up
}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("epi", ["store", "residual", "swiglu"])
def test_fp8_gemm_bitwise_equal_to_the_gemm_on_dequantized_weights(lib, epi, dtype):
    n_cmp = 0
    for N, K in SHAPES[epi]:
        rows = 2 * N if epi == "swiglu" else N
        q, scale, wd = coded(rows, K, N + K, dtype)
        g = torch.Generator(device="cuda").manual_seed(K)
        X = (torch.randn(256, K, generator=g, device="cuda") * 0.5).to(dtype)  # 256 rows: the prefill launch reads them all
        bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(dtype) if epi == "store" else None
        res = torch.randn(256, N, generator=g, device="cuda").to(dtype) if epi == "residual" else None
        torch.cuda.synchronize()
        for M in (1, 10, 16, 60, 64) + (() if epi == "store" else (65, 200, 256)):  # > 64: the prompt prefill's 256-row launch
            for sk in sorted({1, engine_splitk(rows, K)}):
                outs = []
                for f8 in (True, False):
                    out = res.clone() if res is not None else torch.zeros(256, N, dtype=dtype, device="cuda")
                    torch.cuda.synchronize()
                    rp = C.c_void_p(out.data_ptr()) if res is not None else None
                    bp = C.c_void_p(bias.data_ptr()) if bias is not None else None
                    if f8:
                        rc = lib.eb200_k_gemm_fp8(DT[dtype], EPI[epi], C.c_void_p(q.data_ptr()), C.c_void_p(scale.data_ptr()),
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
    assert n_cmp >= 15


def test_fp8_gemm_rejects_what_it_does_not_run(lib):
    q = torch.zeros(128, 128, dtype=torch.uint8, device="cuda")
    s = torch.ones(1, 1, device="cuda")
    X = torch.zeros(64, 256, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(64, 256, dtype=torch.bfloat16, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.eb200_k_gemm_fp8(0, 2, p(q), p(s), p(X), p(out), None, None, 4, 128, 128, 1, None) != 0  # two-matrix SwiGLU
    assert lib.eb200_k_gemm_fp8(0, 0, p(q), p(s), p(X), p(out), None, None, 65, 128, 128, 1, None) != 0  # store at 256 rows
    assert lib.eb200_k_gemm_fp8(0, 1, p(q), p(s), p(X), p(out), p(out), None, 257, 128, 128, 1, None) != 0  # M > 256
    assert lib.eb200_k_gemm_fp8(0, 0, p(q), None, p(X), p(out), None, None, 4, 128, 128, 1, None) != 0  # no scales
    assert lib.eb200_k_gemm_fp8(0, 0, p(q), p(s), p(X), p(out), None, None, 4, 128, 192, 1, None) != 0  # K % 128 != 0
    assert lib.eb200_k_gemm_fp8(0, 0, p(q), p(s), p(X), p(out), None, None, 4, 192, 128, 1, None) != 0  # N % 128 != 0


# ----------------------------------------------------------------------------------------------
# 2. whole generations: FP8 engine == model-dtype engine on W'
# ----------------------------------------------------------------------------------------------
def split_weights(tW, dtype):
    """(FP8 state dict: e4m3 + weight_scale_inv for the projections, W' state dict: the dequantized projections); others shared."""
    t8, tp = {}, {}
    for k, v in tW.items():
        if quant.is_target_projection(k):
            q, s = quant.quantize_fp8_block(v.to(dtype))
            t8[k], t8[k[: -len("weight")] + "weight_scale_inv"] = q, s
            tp[k] = quant.dequantize_fp8_block(q, s, dtype)
        else:
            t8[k] = tp[k] = v
    return t8, tp


def twins(fx, max_length=512, quantize_at_load=False, **kw):
    """(FP8 engine, model-dtype engine on W', prompt, gen kwargs, sampling seed) for a named fixture."""
    from eagle_b200 import EaModel
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(base_fixture(fx))
    tree = dict(tree, **kw)
    t8, tp = split_weights(tW, dtype)
    common = dict(use_eagle3=eagle3, torch_dtype=dtype, max_length=max_length, **tree)
    m8 = EaModel.from_state_dicts(tcfg, tW if quantize_at_load else t8, hcfg, hW, quantization_config=FP8, **common)
    mb = EaModel.from_state_dicts(tcfg, tp, hcfg, hW, **common)
    plen, pseed, gen_kw, seed = FIXTURES[fx]
    return m8, mb, make_prompt(tcfg["vocab_size"], plen, pseed), gen_kw, seed


@pytest.mark.parametrize("fx,static", [("e3_rand_bf16", False), ("e3_corr_bf16", False), ("e3_gqa_bf16", False), ("e1_corr_fp16", False),
                                       ("e3_corr_bf16", True)])
def test_fp8_engine_identical_to_the_engine_on_dequantized_weights(fx, static):
    kw = dict(tree_choices=static_trees.mc_sim_7b_63) if static else {}
    m8, mb, prompt, gen_kw, _ = twins(fx, quantize_at_load=(fx == "e3_gqa_bf16"), **kw)
    a = m8.eagenerate(prompt.cuda(), log=True, **gen_kw)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    assert torch.equal(m8.debug_read("target_kv"), mb.debug_read("target_kv"))
    n = a[2] + 1
    ca, cb = run_cycles(m8, prompt, n), run_cycles(mb, prompt, n)
    assert ca[0] == cb[0]
    for c in range(1, n + 1):
        assert same(ca[c], cb[c]), f"cycle {c - 1}: tree / verify / committed tokens differ"
    assert torch.equal(m8.debug_read("draft_logits"), mb.debug_read("draft_logits"))
    want = mb.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    got = m8.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:]
    report(f"fp8 {fx}{' static tree' if static else ''}: {a[1]} tokens in {a[2] + 1} cycles, identical to the W' twin")


def test_fp8_sampling_identical_to_the_engine_on_dequantized_weights():
    m8, mb, prompt, gen_kw, seed = twins("e3_corr_bf16_T1")
    torch.manual_seed(seed)
    a = m8.eagenerate(prompt.cuda(), log=True, **gen_kw)
    torch.manual_seed(seed)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]


def test_fp8_prefill_of_a_long_prompt_uses_the_256_row_path():
    """A 300-token prompt is prefilled in 256-row chunks (MPAD 256): the target KV cache after prefill is identical."""
    m8, mb, _, gen_kw, _ = twins("e3_corr_bf16")
    prompt = make_prompt(m8.vocab_size, 300, 31)
    assert m8.prefill(prompt.cuda()) == mb.prefill(prompt.cuda())
    ka, kb = m8.debug_read("target_kv"), mb.debug_read("target_kv")
    assert torch.equal(ka, kb) and float(ka.abs().sum()) > 0
    a = m8.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    b = mb.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]


def test_fp8_engine_matches_the_oracle_on_dequantized_weights():
    from eagle_b200 import EaModel
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    t8, tp = split_weights(tW, dtype)
    m8 = EaModel.from_state_dicts(tcfg, t8, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, quantization_config=FP8, **tree)
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
    report(f"fp8 vs oracle on W': identical generated prefix {agree - plen}/{k - plen}, first fragile decision at {must}")
    assert agree - plen >= must


# ----------------------------------------------------------------------------------------------
# 3. loading: from_pretrained with quantization_config and on a stored FP8 directory; refusals of the engine
# ----------------------------------------------------------------------------------------------
def test_from_pretrained_fp8(tmp_path):
    from eagle_b200 import EaModel
    from eagle_b200.checkpoint import save_head_checkpoint, save_target_checkpoint
    from transformers import FineGrainedFP8Config
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    plen, pseed, gen_kw, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed).cuda()
    hdir = str(tmp_path / "head")
    save_head_checkpoint(hdir, hcfg, hW)
    t8, _ = split_weights(tW, dtype)
    want = EaModel.from_state_dicts(tcfg, t8, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, quantization_config=FP8,
                                    **tree).eagenerate(prompt, log=True, **gen_kw)
    common = dict(use_eagle3=eagle3, ea_model_path=hdir, torch_dtype=dtype, max_length=512, **tree)
    bf16_dir, fp8_dir = str(tmp_path / "bf16"), str(tmp_path / "fp8")
    save_target_checkpoint(bf16_dir, tcfg, tW)
    save_target_checkpoint(fp8_dir, tcfg, {k: v.to(dtype) for k, v in tW.items()}, fp8=True)
    for kw in (dict(base_model_path=bf16_dir, quantization_config=FineGrainedFP8Config()), dict(base_model_path=fp8_dir),
               dict(base_model_path=fp8_dir, quantization_config=FP8)):
        m = EaModel.from_pretrained(**kw, **common)
        assert m.quant_fp8
        got = m.eagenerate(prompt, log=True, **gen_kw)
        assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:], kw


def test_engine_refusals_with_fp8_weights():
    from eagle_b200 import EaModel, _lib
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models("e3_corr_bf16")
    t8, _ = split_weights(tW, dtype)
    common = dict(use_eagle3=eagle3, torch_dtype=dtype, max_length=512, **tree)
    with pytest.raises(_lib.EngineError, match="EB200_FLAG_SIMT_GEMM"):
        EaModel.from_state_dicts(tcfg, t8, hcfg, hW, quantization_config=FP8, flags=_lib.FLAG_SIMT_GEMM, **common)
    for other in (_lib.FLAG_TARGET_INT8, _lib.FLAG_TARGET_NF4, _lib.FLAG_TARGET_FP4):
        with pytest.raises(_lib.EngineError, match="exclude each other"):
            EaModel(tcfg, hcfg, flags=_lib.FLAG_TARGET_FP8 | other, **common)
    gcfg, _, ghcfg, _, g3, gdt, gtree = fixture_models("e3_gqa_bf16")
    with pytest.raises(_lib.EngineError, match="tensor parallelism"):
        EaModel(gcfg, ghcfg, use_eagle3=g3, torch_dtype=gdt, max_length=512, tp_size=2, quantization_config=FP8, **gtree)
    m = EaModel(tcfg, hcfg, quantization_config=FP8, **common)
    name = "model.layers.0.mlp.down_proj.weight"
    sname = "model.layers.0.mlp.down_proj.weight_scale_inv"
    with pytest.raises(_lib.EngineError, match="in FP8"):  # model-dtype data for an FP8 projection
        m._load(name, tW[name])
    with pytest.raises(_lib.EngineError, match="only for the target decoder projections"):
        m._load("lm_head.weight", t8[name])
    with pytest.raises(_lib.EngineError, match="shape mismatch"):
        m._load(name, t8[name][:, :-128].contiguous())
    with pytest.raises(_lib.EngineError, match="shape mismatch"):
        m._load(sname, t8[sname][:, :-1].contiguous())
    with pytest.raises(_lib.EngineError, match="weight_scale_inv must be fp32"):
        m._load(sname, t8[sname].to(torch.bfloat16))
    with pytest.raises(_lib.EngineError, match="block scales missing"):
        m.load_target_state_dict({k: v for k, v in t8.items() if k != "model.layers.1.self_attn.k_proj.weight_scale_inv"})
        m.load_head_state_dict(hW)
        m.finalize()
    mb = EaModel(tcfg, hcfg, **common)
    with pytest.raises(_lib.EngineError, match="without EB200_FLAG_TARGET_FP8"):
        mb._load(name, t8[name])
    with pytest.raises(_lib.EngineError, match="without EB200_FLAG_TARGET_FP8"):
        mb._load(sname, t8[sname])


# ----------------------------------------------------------------------------------------------
# 4. model widths, in subprocesses: EB200_L2_PREFETCH on / off, 8-layer Llama-3-8B / 70B widths against their W' twins with the
#    measured footprint, full Llama-3-70B shapes + EAGLE-3 head on one H100
# ----------------------------------------------------------------------------------------------
def run_case(name, *args, env=None, timeout=1500):
    code = f"import json, sys; from tests.test_fp8_gpu import {name}; print('RESULT ' + json.dumps({name}(*sys.argv[1:])))"
    torch.cuda.synchronize()
    torch.cuda.empty_cache()  # what this process's allocator caches is not available to the child
    p = subprocess.run([sys.executable, "-s", "-c", code, *[str(a) for a in args]], cwd=ROOT, env=dict(os.environ, **(env or {})),
                       capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])


def case_prefetch():
    """Cycles and ids of an 8-layer Llama-3-8B-width FP8 engine (run with EB200_L2_PREFETCH=0 / 1)."""
    from eagle_b200 import EaModel, synthetic as syn
    tcfg, tW, hcfg, hW = syn.correlated_llama3_eagle3(8, torch.bfloat16, "cuda")
    m = EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=True, torch_dtype=torch.bfloat16, max_length=1100, total_token=60, depth=6,
                                 top_k=10, quantization_config=FP8)
    used = syn.draft_vocab_ids(tcfg["vocab_size"], hcfg["draft_vocab_size"])
    prompt = used[torch.randint(0, used.numel(), (300,), generator=torch.Generator().manual_seed(0))][None].cuda()
    out = {"first": m.prefill(prompt), "cycles": []}
    for _ in range(16):
        dt, ri, tm, tp = m.get_tree()
        toks, nxt = m.step()
        am, best, acc, n = m.get_verify()
        out["cycles"].append([dt.tolist(), ri.tolist(), tm.flatten().nonzero().flatten().tolist(), tp.tolist(), am.tolist(), best, acc, toks, nxt])
    ids, new_token, idx = m.eagenerate(prompt, max_new_tokens=96, max_length=1100, log=True)
    out["ids"], out["new_token"], out["idx"] = ids.tolist(), int(new_token), int(idx)
    return out


@pytest.mark.timeout(1800)
def test_l2_prefetch_on_and_off_identical():
    off, on = run_case("case_prefetch", env={"EB200_L2_PREFETCH": "0"}), run_case("case_prefetch", env={"EB200_L2_PREFETCH": "1"})
    assert max(c[6] for c in off["cycles"]) >= 2, "the fixture must accept drafts"
    assert on == off


def proj_fp8_bytes(tcfg):
    """Shape-computed device bytes of the FP8 projections: N*K e4m3 plus 16 B of block scales per 128 x 128 block."""
    H, I, L = tcfg["hidden_size"], tcfg["intermediate_size"], tcfg["num_hidden_layers"]
    kv = tcfg["num_key_value_heads"] * 128
    return L * sum(n * k + 16 * (n // 128) * (k // 128) for n, k in ((H + 2 * kv, H), (H, H), (2 * I, H), (H, I)))


def case_width(model):
    """An 8-layer model at the width of `model` (llama3-8b: the correlated pair; llama3-70b: random weights): FP8 engine against
    its W' twin -- ids, per-cycle committed tokens and accept lengths, draft logits -- and the measured footprints."""
    from eagle_b200 import EaModel, synthetic as syn
    dtype = torch.bfloat16
    tree = dict(total_token=60, depth=6, top_k=10)
    if model == "llama3-8b":
        tcfg, tW, hcfg, hW = syn.correlated_llama3_eagle3(8, dtype, "cuda")
        used = syn.draft_vocab_ids(tcfg["vocab_size"], hcfg["draft_vocab_size"])
        prompt = used[torch.randint(0, used.numel(), (700,), generator=torch.Generator().manual_seed(77))][None]
    else:
        tcfg = dict(syn.target_config(model), num_hidden_layers=8)
        hcfg = syn.head_config(model, True, draft_vocab_size=32000)
        tW = syn.make_target_weights(tcfg, 5, dtype, device="cuda")
        hW = syn.make_head_weights(hcfg, tW, True, 6, dtype, device="cuda")
        prompt = make_prompt(tcfg["vocab_size"], 300, 3)
    t8, tp = split_weights(tW, dtype)
    proj_bf16 = sum(v.numel() * 2 for k, v in tW.items() if quant.is_target_projection(k))
    del tW

    def build(sd, **kw):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        m = EaModel.from_state_dicts(tcfg, sd, hcfg, hW, use_eagle3=True, torch_dtype=dtype, max_length=1100, **tree, **kw)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return m, free0 - torch.cuda.mem_get_info()[0]

    m8, used8 = build(t8, quantization_config=FP8)
    mb, usedb = build(tp)
    a = m8.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    b = mb.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    same_ids = a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    cycles_equal, logits_equal = m8.prefill(prompt.cuda()) == mb.prefill(prompt.cuda()), True
    for c in range(a[2] + 1):
        sa, sb = m8.step(), mb.step()
        va, vb = m8.get_verify(), mb.get_verify()
        cycles_equal &= sa == sb and va[2] == vb[2]
        if c == 0:
            logits_equal = torch.equal(m8.debug_read("draft_logits"), mb.debug_read("draft_logits"))
    return {"same_ids": same_ids, "cycles_equal": cycles_equal, "logits_equal": logits_equal, "used8": used8, "usedb": usedb,
            "proj_bf16": proj_bf16, "proj_fp8": proj_fp8_bytes(tcfg), "new_token": a[1], "cycles": a[2] + 1}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("model", ["llama3-8b", "llama3-70b"])
def test_fp8_at_model_width_identical_and_smaller(model):
    r = run_case("case_width", model)
    report(f"fp8 at {model} width, 8 layers: create + load {r['used8'] / 1e9:.3f} GB vs {r['usedb'] / 1e9:.3f} GB in bf16 "
           f"(projections {r['proj_bf16'] / 1e9:.3f} GB in bf16, {r['proj_fp8'] / 1e9:.3f} GB in FP8); "
           f"{r['new_token']} tokens in {r['cycles']} cycles")
    assert r["same_ids"] and r["cycles_equal"] and r["logits_equal"]
    # the difference of the two footprints is the projections' bf16 bytes minus their FP8 bytes (allocation granularity aside)
    saved = r["usedb"] - r["used8"]
    assert abs(saved - (r["proj_bf16"] - r["proj_fp8"])) <= 0.02 * r["proj_bf16"], (saved, r["proj_bf16"], r["proj_fp8"])


def case_llama3_70b_full():
    """Llama-3-70B shapes (80 layers, random weights quantized per tensor on the device) + an EAGLE-3 head on one H100."""
    from eagle_b200 import EaModel, synthetic as syn
    dtype = torch.bfloat16
    tcfg = syn.target_config("llama3-70b")
    hcfg = syn.head_config("llama3-70b", True, draft_vocab_size=32000)
    H, I, V, L = tcfg["hidden_size"], tcfg["intermediate_size"], tcfg["vocab_size"], tcfg["num_hidden_layers"]
    kv = tcfg["num_key_value_heads"] * 128
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    m = EaModel(tcfg, hcfg, use_eagle3=True, torch_dtype=dtype, max_length=2048, total_token=60, depth=6, top_k=10, quantization_config=FP8)
    g = torch.Generator(device="cuda").manual_seed(70)

    def rnd(n, k):  # normal(0, 0.02) in the model dtype, 8192 rows at a time: the engine leaves a few GB for temporaries
        out = torch.empty(n, k, dtype=dtype, device="cuda")
        for r in range(0, n, 8192):
            out[r: r + 8192] = (torch.randn(min(8192, n - r), k, generator=g, device="cuda") * 0.02).to(dtype)
        return out

    m._load("model.embed_tokens.weight", rnd(V, H))
    m._load("lm_head.weight", rnd(V, H))
    # the head embeds with the target's table (load_head_state_dict skips its embed_tokens)
    hW = syn.make_head_weights(hcfg, {"model.embed_tokens.weight": torch.empty(0)}, True, 71, dtype, device="cuda")
    m.load_head_state_dict(hW)
    del hW
    torch.cuda.empty_cache()
    for i in range(L):
        p = f"model.layers.{i}."
        for name, shape in (("self_attn.q_proj", (H, H)), ("self_attn.k_proj", (kv, H)), ("self_attn.v_proj", (kv, H)), ("self_attn.o_proj", (H, H)),
                            ("mlp.gate_proj", (I, H)), ("mlp.up_proj", (I, H)), ("mlp.down_proj", (H, I))):
            m._load_target(p + name + ".weight", rnd(*shape))
        m._load(p + "input_layernorm.weight", torch.ones(H, dtype=dtype, device="cuda"))
        m._load(p + "post_attention_layernorm.weight", torch.ones(H, dtype=dtype, device="cuda"))
        torch.cuda.empty_cache()
    m._load("model.norm.weight", torch.ones(H, dtype=dtype, device="cuda"))
    m.finalize()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    used = free0 - torch.cuda.mem_get_info()[0]
    prompt = make_prompt(V, 512, 7).cuda()
    ids, new_token, idx = m.eagenerate(prompt, max_new_tokens=64, max_length=2048, log=True)
    naive = m.naivegenerate(prompt, max_new_tokens=64, max_length=2048)
    n = min(ids.shape[1], naive.shape[1])
    return {"used": used, "proj_fp8": proj_fp8_bytes(tcfg), "embed_head": 2 * V * H * 2, "lossless": ids[0, :n].tolist() == naive[0, :n].tolist(),
            "n": n, "new_token": int(new_token), "cycles": int(idx) + 1, "name": torch.cuda.get_device_name()}


@pytest.mark.timeout(2700)
def test_llama3_70b_fp8_on_one_h100():
    r = run_case("case_llama3_70b_full", timeout=2400)
    report(f"fp8 Llama-3-70B + EAGLE-3 on one {r['name']}: {r['used'] / 1e9:.2f} GB on the device (FP8 projections "
           f"{r['proj_fp8'] / 1e9:.2f} GB, embeddings + lm_head {r['embed_head'] / 1e9:.2f} GB); {r['new_token']} tokens in {r['cycles']} cycles")
    # the rest is the EAGLE-3 head (~2.8 GB + its own embedding copy), the KV cache and the work buffers
    assert r["proj_fp8"] + r["embed_head"] < r["used"] < r["proj_fp8"] + r["embed_head"] + 8e9
    assert r["lossless"] and r["n"] >= 512 + 64

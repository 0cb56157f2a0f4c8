"""4-bit target weights on the H100: bitsandbytes nf4 / fp4 projections (EB200_FLAG_TARGET_NF4 / _FP4) through the W4A16 GEMM.

The contract (eagle_b200/quant.py) makes a 4-bit engine compute exactly what a model-dtype engine loaded with
W' = dequantize_4bit(packed, absmax) computes, so every comparison here is bit for bit against that twin: the kernel against the
model-dtype kernel on W', and whole generations (trees, verify results, committed tokens, KV) against a bf16 / fp16 engine built
from W'.  The model-width cases run in subprocesses so that no module fixture holds their memory.
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
QT = {"nf4": 0, "fp4": 1}


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def quantized(N, K, seed, dtype, qt):
    """(packed, absmax, W') of a random weight with an all-zero block, a block of subnormal absmax and all 16 codes present."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
    w[min(5, N - 1), :64] = 0
    packed, absmax = quant.quantize_4bit(w, qt)
    absmax[N - 1, 0] = 3e-39 if dtype == torch.bfloat16 else 2e-7  # model-dtype subnormal products
    codes = quant.unpack_4bit(packed)
    assert codes.unique().numel() == 16
    return packed, absmax, quant.dequantize_4bit(packed, absmax, qt, dtype)


# ----------------------------------------------------------------------------------------------
# 1. the kernel: eb200_k_gemm_w4 == eb200_k_gemm (cluster split-K) on W', bit for bit
# ----------------------------------------------------------------------------------------------
SHAPES = {  # N (output rows; SwiGLU: output columns over a [2N, K] interleaved weight), K
    "store": [(256, 256), (200, 320), (130, 64), (6144, 4096), (10240, 8192)],   # tiny, ragged N, K = 64, 8B / 70B qkv
    "residual": [(384, 768), (4096, 4096), (4096, 14336), (8192, 8192)],         # 8B o / down, 70B o
    "swiglu": [(320, 256), (14336, 4096), (28672, 8192)],                         # 8B / 70B gate/up
}


@pytest.mark.parametrize("qt", ["nf4", "fp4"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("epi", ["store", "residual", "swiglu"])
def test_w4_gemm_bitwise_equal_to_the_gemm_on_dequantized_weights(lib, epi, dtype, qt):
    n_cmp = 0
    for N, K in SHAPES[epi]:
        rows = 2 * N if epi == "swiglu" else N
        packed, absmax, wd = quantized(rows, K, N + K, dtype, qt)
        g = torch.Generator(device="cuda").manual_seed(K)
        X = (torch.randn(256, K, generator=g, device="cuda") * 0.5).to(dtype)  # 256 rows: the prefill launch reads them all
        bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(dtype) if epi == "store" else None
        res = torch.randn(256, N, generator=g, device="cuda").to(dtype) if epi == "residual" else None
        torch.cuda.synchronize()
        for M in (1, 10, 16, 60, 64) + (() if epi == "store" else (65, 200, 256)):  # > 64: the prompt prefill's 256-row launch
            for sk in sorted({1, engine_splitk(rows, K)}):
                outs = []
                for w4 in (True, False):
                    out = res.clone() if res is not None else torch.zeros(256, N, dtype=dtype, device="cuda")
                    torch.cuda.synchronize()
                    rp = C.c_void_p(out.data_ptr()) if res is not None else None
                    bp = C.c_void_p(bias.data_ptr()) if bias is not None else None
                    if w4:
                        rc = lib.eb200_k_gemm_w4(DT[dtype], QT[qt], EPI[epi], C.c_void_p(packed.data_ptr()), C.c_void_p(absmax.data_ptr()),
                                                 C.c_void_p(X.data_ptr()), C.c_void_p(out.data_ptr()), rp, bp, M, N, K, sk, None)
                    else:
                        rc = lib.eb200_k_gemm(DT[dtype], 2, EPI[epi], C.c_void_p(wd.data_ptr()), None, C.c_void_p(X.data_ptr()),
                                              C.c_void_p(out.data_ptr()), rp, bp, M, N, K, sk, None)
                    check(lib, rc)
                    outs.append(out)
                a, b = outs
                assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{qt} {epi} M={M} N={N} K={K} splitk={sk}"
                want = res[M:] if res is not None else torch.zeros_like(a[M:])
                assert torch.equal(a[M:].view(torch.int16), want.view(torch.int16))  # rows beyond M are never written
                n_cmp += 1
    assert n_cmp >= 15


def test_w4_gemm_rejects_what_it_does_not_run(lib):
    q = torch.zeros(128, 32, dtype=torch.uint8, device="cuda")
    am = torch.zeros(128, 1, device="cuda")
    X = torch.zeros(64, 96, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(64, 128, dtype=torch.bfloat16, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.eb200_k_gemm_w4(0, 0, 2, p(q), p(am), p(X), p(out), None, None, 4, 128, 64, 1, None) != 0  # two-matrix SwiGLU
    assert lib.eb200_k_gemm_w4(0, 0, 0, p(q), p(am), p(X), p(out), None, None, 65, 128, 64, 1, None) != 0  # store at 256 rows
    assert lib.eb200_k_gemm_w4(0, 0, 1, p(q), p(am), p(X), p(out), p(out), None, 257, 128, 64, 1, None) != 0  # M > 256
    assert lib.eb200_k_gemm_w4(0, 0, 0, p(q), None, p(X), p(out), None, None, 4, 128, 64, 1, None) != 0  # no absmax
    assert lib.eb200_k_gemm_w4(0, 2, 0, p(q), p(am), p(X), p(out), None, None, 4, 128, 64, 1, None) != 0  # unknown code table
    assert lib.eb200_k_gemm_w4(0, 0, 0, p(q), p(am), p(X), p(out), None, None, 4, 128, 96, 1, None) != 0  # K % 64 != 0


# ----------------------------------------------------------------------------------------------
# 2. whole generations: 4-bit engine == model-dtype engine on W'
# ----------------------------------------------------------------------------------------------
def split_weights(tW, dtype, qt):
    """(4-bit state dict: codes + absmax for the projections, W' state dict: the dequantized projections); others shared."""
    t4, tp = {}, {}
    for k, v in tW.items():
        if quant.is_target_projection(k):
            packed, absmax = quant.quantize_4bit(v.to(dtype), qt)
            t4[k], t4[k + ".absmax"] = packed, absmax
            tp[k] = quant.dequantize_4bit(packed, absmax, qt, dtype)
        else:
            t4[k] = tp[k] = v
    return t4, tp


def qc(qt):
    return {"load_in_4bit": True, "bnb_4bit_quant_type": qt}


def twins(fx, qt="nf4", max_length=512, quantize_at_load=False, **kw):
    """(4-bit engine, model-dtype engine on W', prompt, gen kwargs, sampling seed) for a named fixture."""
    from eagle_b200 import EaModel
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(base_fixture(fx))
    tree = dict(tree, **kw)
    t4, tp = split_weights(tW, dtype, qt)
    common = dict(use_eagle3=eagle3, torch_dtype=dtype, max_length=max_length, **tree)
    m4 = EaModel.from_state_dicts(tcfg, tW if quantize_at_load else t4, hcfg, hW, quantization_config=qc(qt), **common)
    mb = EaModel.from_state_dicts(tcfg, tp, hcfg, hW, **common)
    plen, pseed, gen_kw, seed = FIXTURES[fx]
    return m4, mb, make_prompt(tcfg["vocab_size"], plen, pseed), gen_kw, seed


@pytest.mark.parametrize("fx,qt,static", [("e3_rand_bf16", "nf4", False), ("e3_corr_bf16", "nf4", False), ("e3_gqa_bf16", "fp4", False),
                                          ("e1_corr_fp16", "fp4", False), ("e3_corr_bf16", "fp4", True)])
def test_4bit_engine_identical_to_the_engine_on_dequantized_weights(fx, qt, static):
    kw = dict(tree_choices=static_trees.mc_sim_7b_63) if static else {}
    m4, mb, prompt, gen_kw, _ = twins(fx, qt, quantize_at_load=(fx == "e3_gqa_bf16"), **kw)
    a = m4.eagenerate(prompt.cuda(), log=True, **gen_kw)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    n = a[2] + 1
    ca, cb = run_cycles(m4, prompt, n), run_cycles(mb, prompt, n)
    assert ca[0] == cb[0]
    for c in range(1, n + 1):
        assert same(ca[c], cb[c]), f"cycle {c - 1}: tree / verify / committed tokens differ"
    want = mb.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    got = m4.naivegenerate(prompt.cuda(), log=True, **gen_kw)
    assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:]
    for gen in ("ea_generate", "naive_generate"):
        ga = [t.cpu().tolist() for t in getattr(m4, gen)(prompt.cuda(), **gen_kw)]
        gb = [t.cpu().tolist() for t in getattr(mb, gen)(prompt.cuda(), **gen_kw)]
        assert ga == gb, gen
    report(f"{qt} {fx}{' static tree' if static else ''}: {a[1]} tokens in {a[2] + 1} cycles, identical to the W' twin")


def test_4bit_sampling_identical_to_the_engine_on_dequantized_weights():
    m4, mb, prompt, gen_kw, seed = twins("e3_corr_bf16_T1", "nf4")
    torch.manual_seed(seed)
    a = m4.eagenerate(prompt.cuda(), log=True, **gen_kw)
    torch.manual_seed(seed)
    b = mb.eagenerate(prompt.cuda(), log=True, **gen_kw)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    torch.manual_seed(seed)
    a = m4.naivegenerate(prompt.cuda(), **gen_kw)
    torch.manual_seed(seed)
    b = mb.naivegenerate(prompt.cuda(), **gen_kw)
    assert a.cpu().tolist() == b.cpu().tolist()


def test_4bit_prefill_of_a_long_prompt_uses_the_256_row_path():
    """A 300-token prompt is prefilled in 256-row chunks (MPAD 256): the target KV cache after prefill is identical."""
    m4, mb, _, gen_kw, _ = twins("e3_corr_bf16", "fp4")
    prompt = make_prompt(m4.vocab_size, 300, 31)
    assert m4.prefill(prompt.cuda()) == mb.prefill(prompt.cuda())
    ka, kb = m4.debug_read("target_kv"), mb.debug_read("target_kv")
    assert torch.equal(ka, kb) and float(ka.abs().sum()) > 0
    a = m4.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    b = mb.eagenerate(prompt.cuda(), log=True, max_new_tokens=32, max_length=512)
    assert a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]


def test_4bit_engine_matches_the_oracle_on_dequantized_weights():
    from eagle_b200 import EaModel
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    t4, tp = split_weights(tW, dtype, "nf4")
    m4 = EaModel.from_state_dicts(tcfg, t4, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, quantization_config=qc("nf4"),
                                  **tree)
    plen, pseed, gen_kw, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed)
    ids = m4.eagenerate(prompt.cuda(), **gen_kw).cpu()
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
    report(f"nf4 vs oracle on W': identical generated prefix {agree - plen}/{k - plen}, first fragile decision at {must}")
    assert agree - plen >= must


# ----------------------------------------------------------------------------------------------
# 3. loading: from_pretrained with quantization_config and on stored 4-bit directories; refusals of the engine
# ----------------------------------------------------------------------------------------------
def test_from_pretrained_4bit(tmp_path):
    from eagle_b200 import EaModel
    from eagle_b200.checkpoint import iter_4bit_triples, save_head_checkpoint, save_target_checkpoint
    fx = "e3_corr_bf16"
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    plen, pseed, gen_kw, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed).cuda()
    hdir = str(tmp_path / "head")
    save_head_checkpoint(hdir, hcfg, hW)
    bf16_dir = str(tmp_path / "bf16")
    save_target_checkpoint(bf16_dir, tcfg, tW)
    common = dict(use_eagle3=eagle3, ea_model_path=hdir, torch_dtype=dtype, max_length=512, **tree)
    for qt in ("nf4", "fp4"):
        t4, _ = split_weights(tW, dtype, qt)
        want = EaModel.from_state_dicts(tcfg, t4, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, quantization_config=qc(qt),
                                        **tree).eagenerate(prompt, log=True, **gen_kw)
        m = EaModel.from_pretrained(base_model_path=bf16_dir, quantization_config=dict(qc(qt), bnb_4bit_compute_dtype=torch.bfloat16), **common)
        assert m.quant_4bit == qt
        got = m.eagenerate(prompt, log=True, **gen_kw)
        assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:], qt
    for dq in (False, True):  # stored nf4, plain and double-quantized: the engine equals a from_state_dicts engine on the stored codes
        d = str(tmp_path / f"nf4_dq{int(dq)}")
        save_target_checkpoint(d, dict(tcfg, torch_dtype="bfloat16"), tW, load_in_4bit="nf4", double_quant=dq)
        stored = {k: v for k, v, a in iter_4bit_triples(d, "nf4", dtype) for k, v in ([(k, v)] + ([(k + ".absmax", a)] if a is not None else []))}
        want = EaModel.from_state_dicts(tcfg, stored, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512,
                                        quantization_config=qc("nf4"), **tree).eagenerate(prompt, log=True, **gen_kw)
        m = EaModel.from_pretrained(base_model_path=d, **common)
        assert m.quant_4bit == "nf4"
        got = m.eagenerate(prompt, log=True, **gen_kw)
        assert got[0].cpu().tolist() == want[0].cpu().tolist() and got[1:] == want[1:], d


def test_engine_refusals_with_4bit_weights():
    from eagle_b200 import EaModel, _lib
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models("e3_corr_bf16")
    t4, _ = split_weights(tW, dtype, "nf4")
    t8 = {k: quant.quantize_int8_rowwise(v)[0] for k, v in tW.items() if k.endswith("down_proj.weight")}
    common = dict(use_eagle3=eagle3, torch_dtype=dtype, max_length=512, **tree)
    with pytest.raises(_lib.EngineError, match="EB200_FLAG_SIMT_GEMM"):
        EaModel.from_state_dicts(tcfg, t4, hcfg, hW, quantization_config=qc("nf4"), flags=_lib.FLAG_SIMT_GEMM, **common)
    with pytest.raises(_lib.EngineError, match="exclude each other"):
        EaModel(tcfg, hcfg, flags=_lib.FLAG_TARGET_NF4 | _lib.FLAG_TARGET_FP4, **common)
    # the 4-bit loader places whole tensors: tensor parallelism is refused when the engine is created, before any load
    gcfg, _, ghcfg, _, g3, gdt, gtree = fixture_models("e3_gqa_bf16")
    for q in ("nf4", "fp4"):
        with pytest.raises(_lib.EngineError, match="tensor parallelism"):
            EaModel(gcfg, ghcfg, use_eagle3=g3, torch_dtype=gdt, max_length=512, tp_size=2, quantization_config=qc(q), **gtree)
    m = EaModel(tcfg, hcfg, quantization_config=qc("nf4"), **common)
    name = "model.layers.0.mlp.down_proj.weight"
    with pytest.raises(_lib.EngineError, match="4 bits"):  # model-dtype data for a 4-bit projection
        m._load(name, tW[name])
    with pytest.raises(_lib.EngineError, match=r"int8 data \(load_in_8bit format\)"):
        m._load(name, t8[name])
    with pytest.raises(_lib.EngineError, match="only for the target decoder projections"):
        m._load("lm_head.weight", t4[name])
    with pytest.raises(_lib.EngineError, match="shape mismatch"):
        m._load(name, t4[name][:, :-16].contiguous())
    with pytest.raises(_lib.EngineError, match="absmax must be fp32"):
        m._load(name + ".absmax", t4[name + ".absmax"].to(torch.bfloat16))
    with pytest.raises(_lib.EngineError, match="block absmax missing"):
        m.load_target_state_dict({k: v for k, v in t4.items() if k != "model.layers.1.self_attn.k_proj.weight.absmax"})
        m.load_head_state_dict(hW)
        m.finalize()
    mb = EaModel(tcfg, hcfg, **common)
    with pytest.raises(_lib.EngineError, match="without EB200_FLAG_TARGET_NF4"):
        mb._load(name, t4[name])
    m8 = EaModel(tcfg, hcfg, load_in_8bit=True, **common)
    with pytest.raises(_lib.EngineError, match="without EB200_FLAG_TARGET_NF4"):
        m8._load(name + ".absmax", t4[name + ".absmax"])


# ----------------------------------------------------------------------------------------------
# 4. model widths, in subprocesses: EB200_L2_PREFETCH on / off, 8-layer Llama-3-8B / 70B widths against their W' twins with the
#    measured footprint, full Llama-3-70B shapes + EAGLE-3 head on one H100
# ----------------------------------------------------------------------------------------------
def run_case(name, *args, env=None, timeout=1500):
    code = f"import json, sys; from tests.test_w4_gpu import {name}; print('RESULT ' + json.dumps({name}(*sys.argv[1:])))"
    torch.cuda.synchronize()
    torch.cuda.empty_cache()  # what this process's allocator caches is not available to the child
    p = subprocess.run([sys.executable, "-s", "-c", code, *[str(a) for a in args]], cwd=ROOT, env=dict(os.environ, **(env or {})),
                       capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])


def case_prefetch():
    """Cycles and ids of an 8-layer Llama-3-8B-width nf4 engine (run with EB200_L2_PREFETCH=0 / 1)."""
    from eagle_b200 import EaModel, synthetic as syn
    tcfg, tW, hcfg, hW = syn.correlated_llama3_eagle3(8, torch.bfloat16, "cuda")
    m = EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=True, torch_dtype=torch.bfloat16, max_length=1100, total_token=60, depth=6,
                                 top_k=10, quantization_config=qc("nf4"))
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


def proj_4bit_bytes(tcfg):
    """Shape-computed device bytes of the 4-bit projections: N*K/2 nibbles + 4*N*K/64 absmax per projection (N padded to 128)."""
    H, I, L = tcfg["hidden_size"], tcfg["intermediate_size"], tcfg["num_hidden_layers"]
    kv = tcfg["num_key_value_heads"] * 128
    pad = lambda n: (n + 127) // 128 * 128  # noqa: E731
    per = sum(pad(n) * k // 2 + pad(n) * (k // 64) * 4 for n, k in ((H + 2 * kv, H), (H, H), (2 * I, H), (H, I)))
    return L * per


def case_width(model, qt):
    """An 8-layer model at the width of `model` (llama3-8b: the correlated pair; llama3-70b: random weights): 4-bit engine against
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
    t4, tp = split_weights(tW, dtype, qt)
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

    m4, used4 = build(t4, quantization_config=qc(qt))
    mb, usedb = build(tp)
    a = m4.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    b = mb.eagenerate(prompt.cuda(), max_new_tokens=150, max_length=1100, log=True)
    same_ids = a[0].cpu().tolist() == b[0].cpu().tolist() and a[1:] == b[1:]
    cycles_equal, logits_equal = m4.prefill(prompt.cuda()) == mb.prefill(prompt.cuda()), True
    for c in range(a[2] + 1):
        sa, sb = m4.step(), mb.step()
        va, vb = m4.get_verify(), mb.get_verify()
        cycles_equal &= sa == sb and va[2] == vb[2]
        if c == 0:
            logits_equal = torch.equal(m4.debug_read("draft_logits"), mb.debug_read("draft_logits"))
    return {"same_ids": same_ids, "cycles_equal": cycles_equal, "logits_equal": logits_equal, "used4": used4, "usedb": usedb,
            "proj_bf16": proj_bf16, "proj_4bit": proj_4bit_bytes(tcfg), "new_token": a[1], "cycles": a[2] + 1}


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("model,qt", [("llama3-8b", "nf4"), ("llama3-70b", "fp4")])
def test_4bit_at_model_width_identical_and_smaller(model, qt):
    r = run_case("case_width", model, qt)
    report(f"{qt} at {model} width, 8 layers: create + load {r['used4'] / 1e9:.3f} GB vs {r['usedb'] / 1e9:.3f} GB in bf16 "
           f"(projections {r['proj_bf16'] / 1e9:.3f} GB in bf16, {r['proj_4bit'] / 1e9:.3f} GB in 4 bits); "
           f"{r['new_token']} tokens in {r['cycles']} cycles")
    assert r["same_ids"] and r["cycles_equal"] and r["logits_equal"]
    # the difference of the two footprints is the projections' bf16 bytes minus their 4-bit bytes (allocation granularity aside)
    saved = r["usedb"] - r["used4"]
    assert abs(saved - (r["proj_bf16"] - r["proj_4bit"])) <= 0.02 * r["proj_bf16"], (saved, r["proj_bf16"], r["proj_4bit"])


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
    m = EaModel(tcfg, hcfg, use_eagle3=True, torch_dtype=dtype, max_length=2048, total_token=60, depth=6, top_k=10, quantization_config=qc("nf4"))
    g = torch.Generator(device="cuda").manual_seed(70)
    rnd = lambda *s: (torch.randn(*s, generator=g, device="cuda") * 0.02).to(dtype)  # noqa: E731
    embed = rnd(V, H)
    m._load("model.embed_tokens.weight", embed)
    for i in range(L):
        p = f"model.layers.{i}."
        for name, shape in (("self_attn.q_proj", (H, H)), ("self_attn.k_proj", (kv, H)), ("self_attn.v_proj", (kv, H)), ("self_attn.o_proj", (H, H)),
                            ("mlp.gate_proj", (I, H)), ("mlp.up_proj", (I, H)), ("mlp.down_proj", (H, I))):
            m._load_target(p + name + ".weight", rnd(*shape))
        m._load(p + "input_layernorm.weight", torch.ones(H, dtype=dtype, device="cuda"))
        m._load(p + "post_attention_layernorm.weight", torch.ones(H, dtype=dtype, device="cuda"))
    m._load("model.norm.weight", torch.ones(H, dtype=dtype, device="cuda"))
    m._load("lm_head.weight", rnd(V, H))
    hW = syn.make_head_weights(hcfg, {"model.embed_tokens.weight": embed}, True, 71, dtype, device="cuda")
    del embed
    m.load_head_state_dict(hW)
    del hW
    m.finalize()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    used = free0 - torch.cuda.mem_get_info()[0]
    prompt = make_prompt(V, 512, 7).cuda()
    ids, new_token, idx = m.eagenerate(prompt, max_new_tokens=64, max_length=2048, log=True)
    naive = m.naivegenerate(prompt, max_new_tokens=64, max_length=2048)
    n = min(ids.shape[1], naive.shape[1])
    return {"used": used, "proj_4bit": proj_4bit_bytes(tcfg), "embed_head": 2 * V * H * 2, "lossless": ids[0, :n].tolist() == naive[0, :n].tolist(),
            "n": n, "new_token": int(new_token), "cycles": int(idx) + 1, "name": torch.cuda.get_device_name()}


@pytest.mark.timeout(2700)
def test_llama3_70b_4bit_on_one_h100():
    r = run_case("case_llama3_70b_full", timeout=2400)
    report(f"nf4 Llama-3-70B + EAGLE-3 on one {r['name']}: {r['used'] / 1e9:.2f} GB on the device (4-bit projections "
           f"{r['proj_4bit'] / 1e9:.2f} GB, embeddings + lm_head {r['embed_head'] / 1e9:.2f} GB); {r['new_token']} tokens in {r['cycles']} cycles")
    assert r["used"] < 60e9
    # the rest is the EAGLE-3 head (~2.8 GB + its own embedding copy), the KV cache and the work buffers
    assert r["proj_4bit"] + r["embed_head"] < r["used"] < r["proj_4bit"] + r["embed_head"] + 8e9
    assert r["lossless"] and r["n"] >= 512 + 64

"""Synthetic (random-init / correlated) weights of the named shapes.

There is no network for checkpoints, so the benchmark and the parity fixtures use
random-init weights of the reference's architectures (HF default init: normal(0, 0.02),
RMSNorm weights 1.0 -- SURVEY.md 8d).  The dicts use the reference's own state-dict keys
(HF Llama names for the target; cnets.py:486-541 / cnets1.py:480-528 names for the head),
so the same dict loads into the reference model, the CPU oracle and the CUDA engine.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

SHAPES = {
    # name: (V, H, I, L, heads, kv_heads, eps, rope_theta, max_pos)
    "llama3-8b": (128256, 4096, 14336, 32, 32, 8, 1e-5, 500000.0, 8192),
    "llama3-70b": (128256, 8192, 28672, 80, 64, 8, 1e-5, 500000.0, 8192),
    "vicuna-7b": (32000, 4096, 11008, 32, 32, 32, 1e-5, 10000.0, 4096),
    "llama2-13b": (32000, 5120, 13824, 40, 40, 40, 1e-5, 10000.0, 4096),
    # tiny fixtures (head_dim stays 128 like every real target)
    "tiny": (1024, 256, 512, 8, 2, 1, 1e-5, 500000.0, 2048),
    "tiny-mha": (1024, 256, 512, 6, 2, 2, 1e-5, 10000.0, 2048),
    "tiny-gqa4": (1024, 512, 1024, 8, 4, 2, 1e-5, 500000.0, 2048),  # 4 query / 2 kv heads: shardable 2-way
    "tiny-h8": (1024, 1024, 2048, 8, 8, 8, 1e-5, 500000.0, 2048),    # 8 query / 8 kv heads: shardable 2-, 4-, 8-way
}


def target_config(name: str) -> dict:
    V, H, I, L, nh, nkv, eps, theta, maxpos = SHAPES[name]
    return dict(vocab_size=V, hidden_size=H, intermediate_size=I, num_hidden_layers=L,
                num_attention_heads=nh, num_key_value_heads=nkv, rms_norm_eps=eps,
                rope_theta=theta, max_position_embeddings=maxpos)


def head_config(name: str, eagle3: bool, draft_vocab_size: Optional[int] = None,
                num_key_value_heads: Optional[int] = None) -> dict:
    """Head config.json fields (EConfig, configs.py:77-124; extras read at cnets.py:486-534)."""
    c = target_config(name)
    c["num_hidden_layers"] = 1
    if num_key_value_heads is not None:
        c["num_key_value_heads"] = num_key_value_heads
    if eagle3:
        c["draft_vocab_size"] = draft_vocab_size or c["vocab_size"]
    else:
        c["bias"] = True  # ea_model.py:49-54: missing key -> True
    # traineagle3/config.json carries no rope_theta -> cnets.py:216-223 falls back to 10000;
    # train/EAGLE-LLaMA3-Instruct-8B carries 500000.  We state it explicitly.
    return c


def _normal(shape, std, gen, dtype, device):
    if device is not None and torch.device(device).type == "cuda":
        return (torch.randn(shape, generator=gen, device=device, dtype=torch.float32) * std).to(dtype)
    return (torch.randn(shape, generator=gen, dtype=torch.float32) * std).to(dtype)


def make_target_weights(cfg: dict, seed: int, dtype: torch.dtype, device=None, std: float = 0.02) -> Dict[str, torch.Tensor]:
    dev = torch.device(device) if device is not None else torch.device("cpu")
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    H, I, V, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"], cfg["num_hidden_layers"]
    d = H // cfg["num_attention_heads"]
    kvd = cfg["num_key_value_heads"] * d
    W = {"model.embed_tokens.weight": _normal((V, H), std, gen, dtype, dev)}
    for i in range(L):
        p = f"model.layers.{i}."
        W[p + "self_attn.q_proj.weight"] = _normal((H, H), std, gen, dtype, dev)
        W[p + "self_attn.k_proj.weight"] = _normal((kvd, H), std, gen, dtype, dev)
        W[p + "self_attn.v_proj.weight"] = _normal((kvd, H), std, gen, dtype, dev)
        W[p + "self_attn.o_proj.weight"] = _normal((H, H), std, gen, dtype, dev)
        W[p + "mlp.gate_proj.weight"] = _normal((I, H), std, gen, dtype, dev)
        W[p + "mlp.up_proj.weight"] = _normal((I, H), std, gen, dtype, dev)
        W[p + "mlp.down_proj.weight"] = _normal((H, I), std, gen, dtype, dev)
        W[p + "input_layernorm.weight"] = torch.ones(H, dtype=dtype, device=dev)
        W[p + "post_attention_layernorm.weight"] = torch.ones(H, dtype=dtype, device=dev)
    W["model.norm.weight"] = torch.ones(H, dtype=dtype, device=dev)
    W["lm_head.weight"] = _normal((V, H), std, gen, dtype, dev)
    return W


def make_d2t(vocab_size: int, draft_vocab_size: int, device=None):
    """A fixed strided draft->target map in the reference's format: target = draft + d2t[draft]
    (traineagle3/cnets.py:671-676: d2t[i] = used[i] - i, t2d = membership mask)."""
    stride = vocab_size // draft_vocab_size
    used = torch.arange(draft_vocab_size, dtype=torch.long) * stride
    d2t = used - torch.arange(draft_vocab_size, dtype=torch.long)
    t2d = torch.zeros(vocab_size, dtype=torch.bool)
    t2d[used] = True
    if device is not None:
        d2t, t2d = d2t.to(device), t2d.to(device)
    return d2t, t2d


def make_head_weights(hcfg: dict, target_W: Dict[str, torch.Tensor], eagle3: bool, seed: int, dtype: torch.dtype,
                      device=None, std: float = 0.02, target_hidden: Optional[int] = None) -> Dict[str, torch.Tensor]:
    dev = torch.device(device) if device is not None else torch.device("cpu")
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    H, I, V = hcfg["hidden_size"], hcfg["intermediate_size"], hcfg["vocab_size"]
    d = H // hcfg["num_attention_heads"]
    kvd = hcfg["num_key_value_heads"] * d
    W = {"embed_tokens.weight": target_W["model.embed_tokens.weight"].clone()}  # load_emb (cnets.py:488-519)
    if eagle3:
        Vd = hcfg.get("draft_vocab_size") or V
        th = target_hidden or H
        W["fc.weight"] = _normal((H, 3 * th), std, gen, dtype, dev)
        p = "midlayer."
        qk_in = 2 * H
        W["norm.weight"] = torch.ones(H, dtype=dtype, device=dev)
        W["lm_head.weight"] = _normal((Vd, H), std, gen, dtype, dev)
        W[p + "hidden_norm.weight"] = torch.ones(H, dtype=dtype, device=dev)
        W[p + "input_layernorm.weight"] = torch.ones(H, dtype=dtype, device=dev)
        if Vd != V:
            W["d2t"], W["t2d"] = make_d2t(V, Vd, dev)
    else:
        W["fc.weight"] = _normal((H, 2 * H), std, gen, dtype, dev)
        if hcfg.get("bias", True):
            W["fc.bias"] = _normal((H,), std, gen, dtype, dev)
        p = "layers.0."
        qk_in = H
    W[p + "self_attn.q_proj.weight"] = _normal((H, qk_in), std, gen, dtype, dev)
    W[p + "self_attn.k_proj.weight"] = _normal((kvd, qk_in), std, gen, dtype, dev)
    W[p + "self_attn.v_proj.weight"] = _normal((kvd, qk_in), std, gen, dtype, dev)
    W[p + "self_attn.o_proj.weight"] = _normal((H, H), std, gen, dtype, dev)
    W[p + "mlp.gate_proj.weight"] = _normal((I, H), std, gen, dtype, dev)
    W[p + "mlp.up_proj.weight"] = _normal((I, H), std, gen, dtype, dev)
    W[p + "mlp.down_proj.weight"] = _normal((H, I), std, gen, dtype, dev)
    W[p + "post_attention_layernorm.weight"] = torch.ones(H, dtype=dtype, device=dev)
    return W


# --------------------------------------------------------------------------------------
# correlated fixtures (SURVEY.md 7.3 H1): a "bigram-dominant" target and a head that
# reproduces the target's next-token choice, so accept_length > 0 paths are exercised.
# --------------------------------------------------------------------------------------
@torch.no_grad()
def make_bigram_target_(W: Dict[str, torch.Tensor], cfg: dict, residual_eps: float = 0.0,
                        emb_scale: float = 50.0, head_scale: float = 0.05, seed: int = 1234,
                        closed_set: Optional[torch.Tensor] = None):
    """In place: a "permutation bigram" target with LARGE arg-max margins in the model dtype.
    embed *= 50 (about unit-RMS rows); lm_head row perm[t] = head_scale * emb[t], so after token t the logit of
    perm[t] is ~ head_scale * |emb[t]|^2 (about 13) while every other logit is ~ N(0, 0.8): a top-2 margin of ~80
    bf16 ulps, far above summation-order noise (plain random weights have margins of 0-2 ulps: see DESIGN.md).
    Every o_proj / down_proj *= residual_eps keeps the residual stream close to emb(token).
    closed_set (sorted token ids, e.g. the draft vocabulary of an EAGLE-3 head with d2t): the permutation maps the set onto
    itself (and its complement onto itself), so a continuation that starts inside the set stays inside it."""
    W["model.embed_tokens.weight"].mul_(emb_scale)
    E = W["model.embed_tokens.weight"]
    V = E.shape[0]
    g = torch.Generator()
    g.manual_seed(seed)
    if closed_set is None:
        perm = torch.randperm(V, generator=g).to(E.device)
    else:
        inside = closed_set.cpu().long()
        mask = torch.ones(V, dtype=torch.bool)
        mask[inside] = False
        outside = mask.nonzero().flatten()
        perm = torch.empty(V, dtype=torch.long)
        perm[inside] = inside[torch.randperm(inside.numel(), generator=g)]
        perm[outside] = outside[torch.randperm(outside.numel(), generator=g)]
        perm = perm.to(E.device)
    lm = torch.empty_like(W["lm_head.weight"])
    lm[perm] = (E.float() * head_scale).to(E.dtype)
    W["lm_head.weight"] = lm
    for i in range(cfg["num_hidden_layers"]):
        W[f"model.layers.{i}.self_attn.o_proj.weight"].mul_(residual_eps)
        W[f"model.layers.{i}.mlp.down_proj.weight"].mul_(residual_eps)
    return W


@torch.no_grad()
def make_copy_head_eagle1_(hW: Dict[str, torch.Tensor], tW: Dict[str, torch.Tensor]):
    """EAGLE-1 "copy head": fc = [I | 0], bias 0, o_proj = down_proj = 0, so the head's output feature
    is emb(tok_{j+1}) whose target-lm_head argmax equals the bigram target's own choice."""
    H = hW["fc.weight"].shape[0]
    hW["embed_tokens.weight"] = tW["model.embed_tokens.weight"].clone()
    hW["fc.weight"].zero_()
    hW["fc.weight"][:, :H] = torch.eye(H, dtype=hW["fc.weight"].dtype, device=hW["fc.weight"].device)
    if "fc.bias" in hW:
        hW["fc.bias"].zero_()
    hW["layers.0.self_attn.o_proj.weight"].zero_()
    hW["layers.0.mlp.down_proj.weight"].zero_()
    return hW


@torch.no_grad()
def make_copy_head_eagle3_(hW: Dict[str, torch.Tensor], tW: Dict[str, torch.Tensor], hcfg: dict, sharp: float = 6.0,
                           corrupt_frac: float = 0.0, seed: int = 4321):
    """EAGLE-3 "copy head" (needs an MHA head config: num_key_value_heads == num_attention_heads):
    fc = 0 (residual stream 0), q = k = sharp * norm(emb) slice per head (self position wins the
    softmax because RoPE cancels at relative distance 0), v = norm(emb), o = I, down_proj = 0, and the
    draft lm_head = the target lm_head rows of the draft vocabulary.  Output feature = norm(emb(tok_{j+1}))."""
    H = hcfg["hidden_size"]
    assert hcfg["num_key_value_heads"] == hcfg["num_attention_heads"], "copy head needs MHA"
    dt, dev = hW["fc.weight"].dtype, hW["fc.weight"].device
    hW["embed_tokens.weight"] = tW["model.embed_tokens.weight"].clone()
    hW["fc.weight"].zero_()
    eye = torch.eye(H, dtype=dt, device=dev)
    for nm, s in (("q_proj", sharp), ("k_proj", sharp), ("v_proj", 1.0)):
        w = hW[f"midlayer.self_attn.{nm}.weight"]
        w.zero_()
        w[:, :H] = eye * s  # acts on the norm(emb) half of cat(norm(emb), norm(hidden))
    # v also carries -norm(hidden): inside the level loop the head feeds on its own (unit-RMS) output, and
    # residual + (norm(emb) - norm(hidden)) cancels it, leaving norm(emb(tok)) at every depth.
    hW["midlayer.self_attn.v_proj.weight"][:, H:] = -eye
    hW["midlayer.self_attn.o_proj.weight"].copy_(eye)
    hW["midlayer.mlp.down_proj.weight"].zero_()
    if "d2t" in hW:
        rows = torch.arange(hW["d2t"].numel(), device=hW["d2t"].device) + hW["d2t"]
        hW["lm_head.weight"] = tW["lm_head.weight"][rows].clone()
    else:
        hW["lm_head.weight"] = tW["lm_head.weight"].clone()
    if corrupt_frac > 0:
        # make the draft WRONG for a fraction of vocabulary rows (rows rotated among a random subset), so accept
        # lengths vary from cycle to cycle while both models keep large margins
        g = torch.Generator()
        g.manual_seed(seed)
        n = hW["lm_head.weight"].shape[0]
        idx = torch.randperm(n, generator=g)[: max(2, int(n * corrupt_frac))].to(hW["lm_head.weight"].device)
        hW["lm_head.weight"][idx] = hW["lm_head.weight"][idx.roll(1)]
    return hW


def correlated_llama3_eagle3(num_layers: int, dtype: torch.dtype, device, draft_vocab_size: int = 32000, corrupt_frac: float = 0.25,
                             seed: int = 20):
    """Llama-3-8B-shaped (H=4096, I=14336, 32 query / 8 kv heads, V=128256) correlated pair at `num_layers` target layers: a
    permutation-bigram target closed over the draft vocabulary + an EAGLE-3 copy head (32 MHA heads, d2t with 32000 rows) whose
    lm_head is wrong on `corrupt_frac` of its rows, so accept lengths vary (tau > 1) while both models keep arg-max margins of
    ~100 bf16 ulps.  Used by the full-shape parity test (tests/test_fullshape_gpu.py) and `bench.py --fixture correlated`.
    Returns (tcfg, tW, hcfg, hW); prompts must be drawn from the draft vocabulary (`draft_vocab_ids`)."""
    tcfg = target_config("llama3-8b")
    tcfg["num_hidden_layers"] = num_layers
    hcfg = head_config("llama3-8b", True, draft_vocab_size=draft_vocab_size, num_key_value_heads=tcfg["num_attention_heads"])
    tW = make_target_weights(tcfg, seed, dtype, device=device)
    used = draft_vocab_ids(tcfg["vocab_size"], draft_vocab_size)
    make_bigram_target_(tW, tcfg, residual_eps=0.5, closed_set=used)
    hW = make_head_weights(hcfg, tW, True, seed + 1, dtype, device=device)
    make_copy_head_eagle3_(hW, tW, hcfg, corrupt_frac=corrupt_frac)
    return tcfg, tW, hcfg, hW


def correlated_llama2_eagle1(name: str, num_layers: int, dtype: torch.dtype, device, head_scale: Optional[float] = None,
                             corrupt_frac: float = 0.25, seed: int = 30):
    """An EAGLE-1 pair at the width of a named Llama-2 shape ("vicuna-7b", "llama2-13b": MHA, rope theta 1e4, V = 32000) with
    `num_layers` target layers: a permutation-bigram target + an EAGLE-1 copy head (fc over 2H with bias; the draft reads the
    target lm_head) whose own embed_tokens has `corrupt_frac` of its rows rotated among themselves, so the draft is wrong after
    those tokens and accept lengths vary.  head_scale (make_bigram_target_'s, default 0.05, a sharp target): a few tens over H
    gives a soft one.  The bigram logit is head_scale * <emb(t), final hidden>, below head_scale * H at model width because the
    random layers add about as much to the residual stream as the embedding carries.  Load the head with load_emb_from_target=False (as from_pretrained
    does), or the engine embeds with the target's table.  Returns (tcfg, tW, hcfg, hW)."""
    tcfg = target_config(name)
    tcfg["num_hidden_layers"] = num_layers
    hcfg = head_config(name, False)
    tW = make_target_weights(tcfg, seed, dtype, device=device)
    make_bigram_target_(tW, tcfg, residual_eps=0.5, **({} if head_scale is None else dict(head_scale=head_scale)))
    hW = make_copy_head_eagle1_(make_head_weights(hcfg, tW, False, seed + 1, dtype, device=device), tW)
    if corrupt_frac > 0:
        E = hW["embed_tokens.weight"]
        g = torch.Generator()
        g.manual_seed(seed + 2)
        idx = torch.randperm(E.shape[0], generator=g)[: max(2, int(E.shape[0] * corrupt_frac))].to(E.device)
        E[idx] = E[idx.roll(1)]
    return tcfg, tW, hcfg, hW


def draft_vocab_ids(vocab_size: int, draft_vocab_size: int) -> torch.Tensor:
    """Target-vocabulary ids reachable through make_d2t's strided map."""
    return torch.arange(draft_vocab_size, dtype=torch.long) * (vocab_size // draft_vocab_size)


# --------------------------------------------------------------------------------------
# named tiny fixtures shared by the golden generator (oracle/make_golden.py runs the unmodified reference on them),
# the parity tests and bench.py's tp_parity check
# --------------------------------------------------------------------------------------
# a named fixture's weights under another draft-tree geometry: name -> (weights of, tree kwargs)
GEOMETRY_FIXTURES = {
    "e3_corr_bf16_D7": ("e3_corr_bf16", dict(total_token=60, depth=7, top_k=10)),      # EaModel.from_pretrained's default: 70 draft columns
    "e3_corr_bf16_D8K16": ("e3_corr_bf16", dict(total_token=64, depth=8, top_k=16)),   # 128 draft columns, 64 verify rows
}


def fixture_models(name: str):
    """(tcfg, tW, hcfg, hW, eagle3, dtype, tree kwargs) for a named fixture; shared with tests."""
    if name in GEOMETRY_FIXTURES:
        base, tree = GEOMETRY_FIXTURES[name]
        return fixture_models(base)[:6] + (dict(tree),)
    if name == "e3_rand_bf16":
        dtype, eagle3 = torch.bfloat16, True
        tcfg = target_config("tiny")
        tW = make_target_weights(tcfg, 0, dtype)
        hcfg = head_config("tiny", True, draft_vocab_size=512)
        hW = make_head_weights(hcfg, tW, True, 1, dtype)
        tree = dict(total_token=60, depth=6, top_k=10)
    elif name == "e3_corr_bf16":
        dtype, eagle3 = torch.bfloat16, True
        tcfg = target_config("tiny")
        tW = make_bigram_target_(make_target_weights(tcfg, 2, dtype), tcfg, residual_eps=0.5)
        hcfg = head_config("tiny", True, draft_vocab_size=1024, num_key_value_heads=2)
        hW = make_copy_head_eagle3_(make_head_weights(hcfg, tW, True, 3, dtype), tW, hcfg, corrupt_frac=0.25)
        tree = dict(total_token=60, depth=6, top_k=10)
    elif name == "e3_gqa_bf16":
        dtype, eagle3 = torch.bfloat16, True
        tcfg = target_config("tiny-gqa4")
        tW = make_bigram_target_(make_target_weights(tcfg, 8, dtype), tcfg, residual_eps=0.5)
        hcfg = head_config("tiny-gqa4", True, draft_vocab_size=1024, num_key_value_heads=4)
        hW = make_copy_head_eagle3_(make_head_weights(hcfg, tW, True, 9, dtype), tW, hcfg, corrupt_frac=0.3)
        tree = dict(total_token=48, depth=5, top_k=8)
    elif name == "e1_corr_fp16":
        dtype, eagle3 = torch.float16, False
        tcfg = target_config("tiny-mha")
        tW = make_bigram_target_(make_target_weights(tcfg, 4, dtype), tcfg, residual_eps=0.5)
        hcfg = head_config("tiny-mha", False)
        hW = make_copy_head_eagle1_(make_head_weights(hcfg, tW, False, 5, dtype), tW)
        tree = dict(total_token=60, depth=5, top_k=10)
    elif name == "e1_rand_bf16":
        dtype, eagle3 = torch.bfloat16, False
        tcfg = target_config("tiny-mha")
        tW = make_target_weights(tcfg, 6, dtype)
        hcfg = head_config("tiny-mha", False)
        hW = make_head_weights(hcfg, tW, False, 7, dtype)
        tree = dict(total_token=40, depth=4, top_k=8)
    elif name == "e3_tp8_bf16":
        # 8 query / 8 kv heads, I = 2048: the target shards 2-, 4- and 8-way (bench.py's tp_parity run at every N)
        dtype, eagle3 = torch.bfloat16, True
        tcfg = target_config("tiny-h8")
        tW = make_bigram_target_(make_target_weights(tcfg, 21, dtype), tcfg, residual_eps=0.5)
        hcfg = head_config("tiny-h8", True, draft_vocab_size=1024, num_key_value_heads=8)
        hW = make_copy_head_eagle3_(make_head_weights(hcfg, tW, True, 22, dtype), tW, hcfg, corrupt_frac=0.25)
        tree = dict(total_token=60, depth=6, top_k=10)
    else:
        raise KeyError(name)
    return tcfg, tW, hcfg, hW, eagle3, dtype, tree


FIXTURES = {
    # name: (prompt_len, prompt_seed, gen kwargs, sampling seed)
    "e3_rand_bf16": (37, 10, dict(temperature=0.0, max_new_tokens=24, max_length=512), None),
    "e3_corr_bf16": (29, 11, dict(temperature=0.0, max_new_tokens=48, max_length=512), None),
    "e1_corr_fp16": (33, 12, dict(temperature=0.0, max_new_tokens=48, max_length=512), None),
    "e3_gqa_bf16": (70, 14, dict(temperature=0.0, max_new_tokens=40, max_length=512), None),
    "e1_rand_bf16": (21, 13, dict(temperature=0.0, max_new_tokens=16, max_length=512), None),
    "e3_tp8_bf16": (45, 15, dict(temperature=0.0, max_new_tokens=40, max_length=512), None),
    "e3_corr_bf16_D7": (29, 11, dict(temperature=0.0, max_new_tokens=48, max_length=512), None),
    "e3_corr_bf16_D8K16": (29, 11, dict(temperature=0.0, max_new_tokens=48, max_length=512), None),
    "e3_corr_bf16_T1": (29, 11, dict(temperature=1.0, max_new_tokens=32, max_length=512), 1234),
    # the HF warpers of utils.py:38-54 in action: temperature -> top-p -> top-k
    "e3_corr_bf16_T07": (29, 11, dict(temperature=0.7, top_p=0.9, top_k=20, max_new_tokens=32, max_length=512), 4321),
    # near-uniform target (random weights): here every warper changes what gets sampled, so the run discriminates them
    "e3_rand_bf16_T05": (37, 10, dict(temperature=0.5, top_p=0.6, top_k=8, max_new_tokens=24, max_length=512), 99),
    "e3_rand_bf16_TP": (37, 10, dict(temperature=0.8, top_p=0.02, top_k=0, max_new_tokens=24, max_length=512), 98),   # top-p binding
}



def base_fixture(fx: str) -> str:
    for suffix in ("_T1", "_T07", "_T05", "_TP", "_EOS", "_EOT", "_MAXLEN"):
        if fx.endswith(suffix):
            return fx[: -len(suffix)]
    return fx


def make_prompt(vocab: int, n: int, seed: int):
    g = torch.Generator()
    g.manual_seed(seed)
    return torch.randint(0, vocab - 200, (1, n), generator=g)

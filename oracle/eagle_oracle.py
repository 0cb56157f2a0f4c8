"""Torch-CPU restatement of the reference's draft -> verify -> accept hot path.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Every function cites the reference
file:line (under eagle/model/ of the reference) whose arithmetic it restates.  The
restatement keeps the reference's *rounding points* (which intermediate is rounded to
the model dtype, which is kept in fp32) because those decide the bf16/fp16 results:

* RMSNorm: variance and scaling in fp32, cast to the input dtype, THEN times weight
  (cnets.py:379-384, modeling_llama_kv.py:128-132).
* attention: QK^T rounded to model dtype, divided by sqrt(d) in model dtype, fp32 mask
  added, softmax in fp32, probabilities cast back, PV in model dtype
  (modeling_llama_kv.py:722-743, cnets.py:295-312).
* RoPE: cos/sin tables built in fp32 and cast to the model dtype on use
  (modeling_llama_kv.py:160-205, cnets.py:117-143); q*cos, rot(q)*sin and their sum are
  three separate model-dtype roundings (modeling_llama_kv.py:423-445).
* draft log-softmax / top-k / cumulative scores run in the model dtype
  (cnets.py:697-757).

Parity status: pinned by tests/test_oracle_golden.py against vectors produced by the
unmodified reference (oracle/make_golden.py).
"""
from __future__ import annotations

import math
import random
import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# configuration
# --------------------------------------------------------------------------------------
@dataclass
class ModelCfg:
    """Llama-family shape description (HF LlamaConfig / EConfig fields we need)."""

    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    num_key_value_heads: int
    rms_norm_eps: float = 1e-6
    rope_theta: float = 10000.0
    max_position_embeddings: int = 2048
    # draft-head only (configs.py:77-124 + free-form extras read by cnets.py:486-534)
    draft_vocab_size: Optional[int] = None
    target_hidden_size: Optional[int] = None
    bias: bool = True  # EAGLE-1 fc bias (ea_model.py:49-54)

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def n_rep(self) -> int:
        return self.num_attention_heads // self.num_key_value_heads


Weights = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------------------
# elementary ops
# --------------------------------------------------------------------------------------
def rms_norm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """cnets.py:379-384 / modeling_llama_kv.py:128-132."""
    dt = x.dtype
    h = x.to(torch.float32)
    var = h.pow(2).mean(-1, keepdim=True)
    h = h * torch.rsqrt(var + eps)
    return w * h.to(dt)


def rope_table(dim: int, n_pos: int, base: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos/sin tables [n_pos, dim] (modeling_llama_kv.py:148-186, cnets.py:110-133)."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim))
    t = torch.arange(n_pos, dtype=inv_freq.dtype)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos(), emb.sin()


def _rotate_half(x: torch.Tensor) -> torch.Tensor:
    d = x.shape[-1] // 2
    return torch.cat((-x[..., d:], x[..., :d]), dim=-1)


def apply_rope(q, k, cos, sin, position_ids):
    """modeling_llama_kv.py:423-445 / cnets.py:98-107.  cos/sin: [n_pos, dim] in q.dtype."""
    c = cos[position_ids].unsqueeze(1)
    s = sin[position_ids].unsqueeze(1)
    return (q * c) + (_rotate_half(q) * s), (k * c) + (_rotate_half(k) * s)


def _repeat_kv(x: torch.Tensor, n_rep: int) -> torch.Tensor:
    """modeling_llama_kv.py:540-560 / cnets.py:78-88."""
    if n_rep == 1:
        return x
    b, h, s, d = x.shape
    return x[:, :, None, :, :].expand(b, h, n_rep, s, d).reshape(b, h * n_rep, s, d)


def eager_attention(q, k, v, mask, n_rep: int) -> torch.Tensor:
    """matmul -> /sqrt(d) -> +mask -> softmax(fp32) -> matmul (modeling_llama_kv.py:719-743)."""
    k = _repeat_kv(k, n_rep)
    v = _repeat_kv(v, n_rep)
    w = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(q.shape[-1])
    if mask is not None:
        w = w + mask
    w = F.softmax(w, dim=-1, dtype=torch.float32).to(q.dtype)
    return torch.matmul(w, v)


def _causal_mask(n: int, past: int) -> torch.Tensor:
    """_make_causal_mask with dtype forced to fp32 (modeling_llama_kv.py:52-84, :1020-1027)."""
    m = torch.full((n, n), torch.finfo(torch.float32).min)
    idx = torch.arange(n)
    m.masked_fill_(idx < (idx + 1).view(n, 1), 0)
    if past > 0:
        m = torch.cat([torch.zeros(n, past, dtype=torch.float32), m], dim=-1)
    return m[None, None]


def swiglu_mlp(x, wg, wu, wd):
    """modeling_llama_kv.py:501-535 / cnets.py:347-367 (pretraining_tp == 1)."""
    return F.linear(F.silu(F.linear(x, wg)) * F.linear(x, wu), wd)


# --------------------------------------------------------------------------------------
# target model with preallocated KV (modeling_llama_kv.py + kv_cache.py)
# --------------------------------------------------------------------------------------
class TargetKV:
    """Preallocated K/V planes + per-plane lengths (kv_cache.py:4-66, :69-157)."""

    def __init__(self, cfg: ModelCfg, max_length: int, dtype: torch.dtype):
        L, kvh, d = cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.head_dim
        self.data = torch.zeros(2 * L, 1, kvh, max_length, d, dtype=dtype)
        self.length = 0  # all 2L planes always share one length (kv_cache.py:126-130)

    def reset(self):
        self.length = 0

    def append(self, plane: int, x: torch.Tensor) -> torch.Tensor:
        """KVCache.cat (kv_cache.py:52-66) without advancing the shared length."""
        n = x.shape[2]
        self.data[plane, :, :, self.length:self.length + n].copy_(x)
        return self.data[plane, :, :, : self.length + n]

    def compact(self, select_indices: torch.Tensor, prev_len: int):
        """update_inference_inputs' gather-compaction (utils.py:444-452)."""
        tgt = self.data[..., select_indices, :]
        self.data[..., prev_len:prev_len + tgt.shape[-2], :].copy_(tgt)
        self.length = prev_len + tgt.shape[-2]


class TargetModel:
    """LlamaForCausalLM restated as pure functions over an HF-named weight dict."""

    def __init__(self, cfg: ModelCfg, W: Weights):
        self.cfg, self.W = cfg, W
        self.dtype = W["model.embed_tokens.weight"].dtype
        n_pos = max(cfg.max_position_embeddings, 4096)
        cos, sin = rope_table(cfg.head_dim, n_pos, cfg.rope_theta)
        self.cos, self.sin = cos.to(self.dtype), sin.to(self.dtype)

    def _mask(self, n: int, past: int, tree_mask: Optional[torch.Tensor]):
        """_prepare_decoder_attention_mask (modeling_llama_kv.py:1010-1043)."""
        expanded = torch.zeros(1, 1, n, past + n, dtype=self.dtype)  # all-ones padding mask
        if n <= 1:
            return expanded
        m = _causal_mask(n, past) + expanded
        if tree_mask is not None:
            tl = tree_mask.size(-1)
            m[:, :, -tl:, -tl:][tree_mask == 0] = m.min()
        return m

    def _layer(self, i: int, x, mask, position_ids, kv: TargetKV):
        """LlamaDecoderLayer.forward (modeling_llama_kv.py:801-863) + LlamaAttention.forward (:643-773)."""
        cfg, W = self.cfg, self.W
        p = f"model.layers.{i}."
        b, n, _ = x.shape
        h = rms_norm(x, W[p + "input_layernorm.weight"], cfg.rms_norm_eps)
        q = F.linear(h, W[p + "self_attn.q_proj.weight"]).view(b, n, cfg.num_attention_heads, cfg.head_dim).transpose(1, 2)
        k = F.linear(h, W[p + "self_attn.k_proj.weight"]).view(b, n, cfg.num_key_value_heads, cfg.head_dim).transpose(1, 2)
        v = F.linear(h, W[p + "self_attn.v_proj.weight"]).view(b, n, cfg.num_key_value_heads, cfg.head_dim).transpose(1, 2)
        q, k = apply_rope(q, k, self.cos, self.sin, position_ids)
        k = kv.append(2 * i, k)
        v = kv.append(2 * i + 1, v)
        a = eager_attention(q, k, v, mask, cfg.n_rep)
        a = a.transpose(1, 2).contiguous().reshape(b, n, cfg.hidden_size)
        x = x + F.linear(a, W[p + "self_attn.o_proj.weight"])
        h = rms_norm(x, W[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
        return x + swiglu_mlp(h, W[p + "mlp.gate_proj.weight"], W[p + "mlp.up_proj.weight"], W[p + "mlp.down_proj.weight"])

    def forward(self, input_ids, kv: TargetKV, position_ids=None, tree_mask=None):
        """LlamaModel.forward (modeling_llama_kv.py:1046-1200): returns (normed hidden, 3 taps)."""
        cfg = self.cfg
        n = input_ids.shape[1]
        past = kv.length
        if position_ids is None:
            position_ids = torch.arange(past, past + n, dtype=torch.long)[None]
        else:
            position_ids = position_ids.view(-1, n).long()
        x = F.embedding(input_ids, self.W["model.embed_tokens.weight"])
        mask = self._mask(n, past, tree_mask)
        taps = []
        L = cfg.num_hidden_layers
        for i in range(L):
            if i == L - 3 or i == L // 2 or i == 2:  # modeling_llama_kv.py:1138-1139
                taps.append(x)
            x = self._layer(i, x, mask, position_ids, kv)
        kv.length = past + n
        return rms_norm(x, self.W["model.norm.weight"], cfg.rms_norm_eps), taps

    def lm_head(self, h):
        return F.linear(h, self.W["lm_head.weight"])


# --------------------------------------------------------------------------------------
# draft heads
# --------------------------------------------------------------------------------------
class DraftHead:
    """EAGLE-3 (cnets.py) or EAGLE-1/2 (cnets1.py) draft head + dynamic tree builder."""

    def __init__(self, cfg: ModelCfg, W: Weights, eagle3: bool, total_tokens=60, depth=7, top_k=10):
        self.cfg, self.W, self.eagle3 = cfg, W, eagle3
        self.total_tokens = total_tokens - 1  # cnets.py:522
        self.depth, self.top_k = depth, top_k
        self.dtype = W["embed_tokens.weight"].dtype
        # cnets.py:216-223 -- base = config.rope_theta when present, cache of max_position_embeddings rows
        n_pos = max(cfg.max_position_embeddings, 4096)
        cos, sin = rope_table(cfg.head_dim, n_pos, cfg.rope_theta)
        self.cos, self.sin = cos.to(self.dtype), sin.to(self.dtype)
        self.stable_kv = None
        self.trace = None  # optional dict filled by topk_generate for kernel-level tests

    def reset_kv(self):
        self.stable_kv = None

    # -- mask (cnets.py:554-584) ---------------------------------------------------------
    @staticmethod
    def _mask(n: int, past: int, tree_mask, single_row_tree_mask: bool = False):
        expanded = torch.zeros(1, 1, n, past + n, dtype=torch.float32)
        if n <= 1 and not (single_row_tree_mask and tree_mask is not None):
            return expanded
        # modeling_eagle.py:714-745 (static tree) always has an expanded all-ones mask to write the tree mask into, so a
        # one-row level is tree-masked there; cnets.py:554-584 only builds a mask for n > 1
        m = (_causal_mask(n, past) + expanded) if n > 1 else expanded
        if tree_mask is not None:
            s0, s1 = tree_mask.shape[-2:]
            m[:, :, -s0:, -s1:][tree_mask == 0] = torch.finfo(torch.float32).min
        return m

    def _attn(self, p: str, x, mask, position_ids, past_kv):
        """LlamaAttention.forward (cnets.py:241-333)."""
        cfg, W = self.cfg, self.W
        b, n, _ = x.shape
        q = F.linear(x, W[p + "q_proj.weight"]).view(b, n, cfg.num_attention_heads, cfg.head_dim).transpose(1, 2)
        k = F.linear(x, W[p + "k_proj.weight"]).view(b, n, cfg.num_key_value_heads, cfg.head_dim).transpose(1, 2)
        v = F.linear(x, W[p + "v_proj.weight"]).view(b, n, cfg.num_key_value_heads, cfg.head_dim).transpose(1, 2)
        q, k = apply_rope(q, k, self.cos, self.sin, position_ids)
        if past_kv is not None:
            k = torch.cat([past_kv[0], k], dim=2)
            v = torch.cat([past_kv[1], v], dim=2)
        a = eager_attention(q, k, v, mask, cfg.n_rep)
        a = a.transpose(1, 2).contiguous().reshape(b, n, cfg.hidden_size)
        return F.linear(a, W[p + "o_proj.weight"]), (k, v)

    def forward(self, hidden, input_ids, past_kv=None, position_ids=None, tree_mask=None, single_row_tree_mask=False):
        """Model.forward: cnets.py:586-664 (EAGLE-3) / cnets1.py:570-667 (EAGLE-1/2).

        Returns (out_hidden [1,n,H], new_kv) where new_kv is a tuple with one (k, v) per layer.
        """
        cfg, W = self.cfg, self.W
        n = hidden.shape[1]
        emb = F.embedding(input_ids, W["embed_tokens.weight"])
        past = 0 if past_kv is None else past_kv[0][0].shape[2]
        if position_ids is None:
            position_ids = torch.arange(past, past + n, dtype=torch.long)[None]
        else:
            position_ids = position_ids.view(-1, n).long()
        mask = self._mask(n, past, tree_mask, single_row_tree_mask)
        emb = emb.to(hidden.dtype)
        if self.eagle3:
            if hidden.shape[-1] != emb.shape[-1]:
                hidden = F.linear(hidden, W["fc.weight"])  # cnets.py:639-640
            residual = hidden
            hn = rms_norm(hidden, W["midlayer.hidden_norm.weight"], cfg.rms_norm_eps)
            en = rms_norm(emb, W["midlayer.input_layernorm.weight"], cfg.rms_norm_eps)
            x = torch.cat((en, hn), dim=-1)  # cnets.py:427-430
            a, kv = self._attn("midlayer.self_attn.", x, mask, position_ids, None if past_kv is None else past_kv[0])
            h = residual + a
            hh = rms_norm(h, W["midlayer.post_attention_layernorm.weight"], cfg.rms_norm_eps)
            h = h + swiglu_mlp(hh, W["midlayer.mlp.gate_proj.weight"], W["midlayer.mlp.up_proj.weight"],
                               W["midlayer.mlp.down_proj.weight"])
            return h, (kv,)
        # EAGLE-1/2: fc(cat(emb, hidden)) then N layers, layer 0 without input norm (cnets1.py:623, :428-429)
        h = F.linear(torch.cat((emb, hidden), dim=-1), W["fc.weight"], W.get("fc.bias"))
        new_kv = []
        for i in range(cfg.num_hidden_layers):
            p = f"layers.{i}."
            x = h if i == 0 else rms_norm(h, W[p + "input_layernorm.weight"], cfg.rms_norm_eps)
            a, kv = self._attn(p + "self_attn.", x, mask, position_ids, None if past_kv is None else past_kv[i])
            h = h + a
            hh = rms_norm(h, W[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
            h = h + swiglu_mlp(hh, W[p + "mlp.gate_proj.weight"], W[p + "mlp.up_proj.weight"], W[p + "mlp.down_proj.weight"])
            new_kv.append(kv)
        return h, tuple(new_kv)

    def _head_logits(self, h, target_lm_head):
        if self.eagle3:  # cnets.py:700, :734
            return F.linear(rms_norm(h, self.W["norm.weight"], self.cfg.rms_norm_eps), self.W["lm_head.weight"])
        return F.linear(h, target_lm_head)  # cnets1.py:702, :732

    def _to_target_vocab(self, idx):
        if self.eagle3 and self.cfg.draft_vocab_size is not None and self.cfg.draft_vocab_size != self.cfg.vocab_size:
            return idx + self.W["d2t"][idx]  # cnets.py:712-713, :751-755
        return idx

    # -- dynamic tree growth (cnets.py:669-827; identical logic cnets1.py:672-822) --------------
    @torch.no_grad()
    def topk_generate(self, hidden_states, input_ids, target_lm_head, sampling: bool):
        k, depth, total = self.top_k, self.depth, self.total_tokens
        sample_token = input_ids[:, -1]
        input_ids = input_ids[:, 1:]
        len_posi = input_ids.shape[1]
        if self.stable_kv is not None:
            kv_len = self.stable_kv[0][0].shape[2]
            out_hidden, past = self.forward(hidden_states, input_ids[:, kv_len:], past_kv=self.stable_kv)
        else:
            out_hidden, past = self.forward(hidden_states, input_ids)
        self.stable_kv = past
        last_hidden = out_hidden[:, -1]
        stable_out = out_hidden

        raw = self._head_logits(last_hidden, target_lm_head)
        last_p = F.log_softmax(raw, dim=-1)
        level_logits = [last_p]
        level_raw = [raw]
        top = torch.topk(last_p, k, dim=-1)
        topk_index, topk_p = top.indices, top.values
        scores = topk_p[0]
        scores_list = [scores[None]]
        parents_list = [torch.zeros(1, dtype=torch.long)]
        ss_token = [self._to_target_vocab(topk_index)]
        level_ids = self._to_target_vocab(topk_index)
        input_hidden = last_hidden[None].repeat(1, k, 1)
        tree_mask = torch.eye(k)[None, None]
        tree_mask_init = tree_mask
        topk_cs_index = torch.arange(k)
        level_hidden = []

        for i in range(depth):
            position_ids = len_posi + torch.zeros(k, dtype=torch.long)
            out_hidden, past = self.forward(input_hidden, level_ids, past_kv=past, position_ids=position_ids,
                                            tree_mask=tree_mask)
            level_hidden.append(out_hidden)
            len_posi += 1
            bias = 1 + k ** 2 * max(0, i - 1) + (k if i > 0 else 0)
            parents_list.append(topk_cs_index + bias)

            raw = self._head_logits(out_hidden[0], target_lm_head)
            last_p = F.log_softmax(raw, dim=-1)
            level_logits.append(last_p)
            level_raw.append(raw)
            top = torch.topk(last_p, k, dim=-1)
            topk_index, topk_p = top.indices, top.values
            cu_scores = topk_p + scores[:, None]
            topk_cs = torch.topk(cu_scores.view(-1), k, dim=-1)
            topk_cs_index, scores = topk_cs.indices, topk_cs.values
            out_ids = topk_cs_index // k
            input_hidden = out_hidden[:, out_ids]
            level_ids = self._to_target_vocab(topk_index.view(-1)[topk_cs_index][None])
            ss_token.append(self._to_target_vocab(topk_index))
            scores_list.append(cu_scores)
            tree_mask = torch.cat((tree_mask[:, :, out_ids], tree_mask_init), dim=3)

        scores_flat = torch.cat(scores_list, dim=0).view(-1)
        tokens_flat = torch.cat(ss_token, dim=0).view(-1)
        parents_flat = torch.cat(parents_list, dim=0)
        out = finalize_tree(scores_flat, tokens_flat, parents_flat, sample_token, k, total, sampling)
        if self.trace is not None:
            self.trace.update(scores_flat=scores_flat, tokens_flat=tokens_flat, parents_flat=parents_flat,
                              stable_out=stable_out, level_hidden=level_hidden, level_logp=level_logits, level_raw=level_raw)
        return out


def finalize_tree(scores_flat, tokens_flat, parents_flat, sample_token, k: int, total: int, sampling: bool):
    """Global rerank + tree buffers (cnets.py:760-827).

    scores_flat [k + depth*k*k], tokens_flat same, parents_flat [1 + depth*k].
    Returns draft_tokens [1,T], retrieve_indices [n_leaf, max_depth] (long), tree_mask [1,1,T,T] fp32,
    tree_position_ids [T].
    """
    top_idx = torch.topk(scores_flat, total, dim=-1).indices
    top_idx = torch.sort(top_idx).values
    draft_tokens = torch.cat((sample_token, tokens_flat[top_idx]), dim=0)
    draft_parents = parents_flat[top_idx // k].long()
    mask_index = torch.searchsorted(top_idx, draft_parents - 1, right=False)
    mask_index[draft_parents == 0] = -1
    mask_index = mask_index + 1
    mi = mask_index.tolist()
    tree_mask = torch.eye(total + 1).bool()
    tree_mask[:, 0] = True
    for i in range(total):
        tree_mask[i + 1].add_(tree_mask[mi[i]])
    tree_position_ids = torch.sum(tree_mask, dim=1) - 1
    tree_mask_f = tree_mask.float()[None, None]
    max_depth = int(torch.max(tree_position_ids)) + 1
    noleaf = torch.unique(mask_index).tolist()
    leaf_num = total - (len(noleaf) - 1)
    retrieve = [[-1] * max_depth for _ in range(leaf_num)]
    pos = tree_position_ids.tolist()
    rid = 0
    for i in range(total + 1):
        if i not in noleaf:
            cid = i
            for j in reversed(range(pos[i] + 1)):
                retrieve[rid][j] = cid
                cid = mi[cid - 1]
            rid += 1
    if sampling:  # cnets.py:811-821: lexicographic row sort with -1 -> large
        big = total + 5
        retrieve = sorted(retrieve, key=lambda r: [x if x >= 0 else big for x in r])
    return draft_tokens[None], torch.tensor(retrieve, dtype=torch.long), tree_mask_f, tree_position_ids


# --------------------------------------------------------------------------------------
# posterior + commit (utils.py)
# --------------------------------------------------------------------------------------
def evaluate_posterior_greedy(logits, candidates):
    """utils.py:360-373."""
    posterior_mask = (candidates[:, 1:] == torch.argmax(logits[:, :-1], dim=-1)).int()
    cand_accept = torch.cumprod(posterior_mask, dim=1).sum(dim=1)
    accept_length = cand_accept.max()
    if accept_length == 0:
        best = torch.tensor(0, dtype=torch.long)
    else:
        best = torch.argmax(cand_accept).to(torch.long)
    return best, accept_length, logits[best, accept_length]


def warp_logits(logits, temperature: float, top_p: float, top_k: int):
    """prepare_logits_processor's list applied in order (utils.py:38-54): temperature, top-p, top-k.

    Restates HF TemperatureLogitsWarper / TopPLogitsWarper / TopKLogitsWarper
    (transformers.generation.logits_process, pinned >=4.53.1 by requirements.txt:2; not vendored).
    logits: [1, V]."""
    if temperature >= 1e-5 and temperature != 1.0:
        logits = logits / temperature
    if 1e-8 <= top_p < 1.0:
        sorted_logits, sorted_idx = torch.sort(logits, descending=False)
        cum = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
        remove = cum <= (1 - top_p)
        remove[..., -1:] = 0
        remove = remove.scatter(1, sorted_idx, remove)
        logits = logits.masked_fill(remove, -float("inf"))
    if top_k > 0:
        kk = min(int(top_k), logits.size(-1))
        remove = logits < torch.topk(logits, kk)[0][..., -1, None]
        logits = logits.masked_fill(remove, -float("inf"))
    return logits


def evaluate_posterior_sampling(logits, candidates, warp, rand=random.random):
    """utils.py:375-415: sequential multi-candidate speculative sampling with q(x) == 1."""
    accept_length = 1
    accept_cand = candidates[0][:1]
    best_candidate = 0
    adjustflag = False
    gtp = None
    for i in range(1, candidates.shape[1]):
        if i != accept_length:
            break
        adjustflag = False
        is_eq = (candidates[:, :accept_length] == accept_cand).all(dim=1)
        fi = torch.nonzero(is_eq, as_tuple=True)[0][0]
        gtp = torch.softmax(warp(logits[fi, i - 1][None])[0], dim=0)
        seen = []
        for j in range(candidates.shape[0]):
            if is_eq[j]:
                xi = candidates[j, i].item()
                if xi in seen or xi == -1:
                    continue
                seen.append(xi)
                r = rand()
                if r <= gtp[xi] / 1.0:
                    accept_cand = torch.cat((accept_cand, candidates[j, i][None]), dim=0)
                    accept_length += 1
                    best_candidate = j
                    break
                gtp[xi] = 0
                gtp = gtp / gtp.sum()
                adjustflag = True
    if adjustflag and accept_length != candidates.shape[1]:
        sample_p = gtp
    else:
        sample_p = torch.softmax(warp(logits[best_candidate, accept_length - 1][None])[0], dim=0)
    return torch.tensor(best_candidate), accept_length - 1, sample_p


class OracleEaModel:
    """EaModel.eagenerate / naivegenerate restated (ea_model.py:198-380) over the pieces above."""

    def __init__(self, tcfg: ModelCfg, tW: Weights, hcfg: ModelCfg, hW: Weights, eagle3: bool,
                 total_token=60, depth=7, top_k=10, eos_token_id: int = -1, eot_token_id: int = -1, tree_choices=None):
        self.target = TargetModel(tcfg, tW)
        # tree_choices: fixed draft tree (oracle/static_tree.py, SURVEY.md 8 row a11) instead of the dynamic one;
        # total_token / depth then follow from the choice list
        self.tree_choices = tree_choices
        if tree_choices is not None:
            total_token = len(tree_choices) + 1
            depth = max(len(c) for c in tree_choices) - 1
        self.head = DraftHead(hcfg, hW, eagle3, total_token, depth, top_k)
        self.eagle3 = eagle3
        self.eos_token_id, self.eot_token_id = eos_token_id, eot_token_id
        self.kv: Optional[TargetKV] = None
        self.cycle_log: Optional[List[dict]] = None  # per-cycle record for tests
        self.time_log: Optional[List[float]] = None  # wall-clock stamps: start, after initialize_tree, after each cycle

    def _kv(self, max_length):
        if self.kv is None:
            self.kv = TargetKV(self.target.cfg, max_length, self.target.dtype)
        self.kv.reset()
        return self.kv

    def _tree(self, feats, ids, sampling):
        if self.tree_choices is not None:
            from . import static_tree
            return static_tree.static_tree(self.head, feats, ids, self.target.W["lm_head.weight"], self.tree_choices,
                                           self.head.top_k)
        return self.head.topk_generate(feats, ids, self.target.W["lm_head.weight"], sampling)

    def _features(self, hidden, taps):
        return torch.cat(taps, dim=-1) if self.eagle3 else hidden  # utils.py:248-252, :324-328

    @torch.no_grad()
    def eagenerate(self, input_ids, temperature=0.0, top_p=0.0, top_k=0.0, max_new_tokens=512,
                   max_length=2048, log=False, is_llama3=False, rand=random.random):
        sampling = temperature > 1e-5
        warp = (lambda lg: warp_logits(lg, temperature, top_p, int(top_k))) if sampling else None
        input_ids = input_ids.clone()
        self.head.reset_kv()
        kv = self._kv(max_length)
        input_len = input_ids.shape[1]
        if self.time_log is not None:
            self.time_log.append(time.time())
        # ---- initialize_tree (utils.py:232-254): prefill + first token + first draft tree
        hidden, taps = self.target.forward(input_ids, kv)
        orig = self.target.lm_head(hidden)
        if sampling:
            probs = torch.softmax(warp(orig[:, -1]), dim=1)
            token = torch.multinomial(probs, 1)
        else:
            token = torch.argmax(orig[:, -1])[None, None]
        feats = self._features(hidden, taps)
        draft_tokens, retrieve, tree_mask, tree_pos = self._tree(feats, torch.cat((input_ids, token), dim=1), sampling)
        new_token = 0
        limit = max_length - self.head.total_tokens - 10
        idx = 0
        if self.time_log is not None:
            self.time_log.append(time.time())
        for idx in range(limit):
            # ---- tree_decoding (utils.py:306-331)
            position_ids = tree_pos + input_ids.shape[1]
            hidden, taps = self.target.forward(draft_tokens, kv, position_ids=position_ids[None], tree_mask=tree_mask)
            tree_logits = self.target.lm_head(hidden)
            feats_new = self._features(hidden, taps)
            logits = tree_logits[0, retrieve]
            cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
            # ---- evaluate_posterior (utils.py:337-415)
            if sampling:
                best, accept_length, sample_p = evaluate_posterior_sampling(logits, cands, warp, rand)
            else:
                best, accept_length, sample_p = evaluate_posterior_greedy(logits, cands)
            # ---- update_inference_inputs (utils.py:418-473)
            prev_len = input_ids.shape[1]
            a = int(accept_length)
            select = retrieve[best, : a + 1] + prev_len
            input_ids = torch.cat([input_ids, cands[None, best, : a + 1]], dim=-1)
            kv.compact(select, prev_len)
            accept_feats = feats_new[:, retrieve][:, best, : a + 1]
            if sampling:
                token = torch.multinomial(sample_p, 1)[None]
            else:
                token = torch.argmax(sample_p)[None, None]
            if self.cycle_log is not None:
                self.cycle_log.append(dict(draft_tokens=draft_tokens.clone(), retrieve=retrieve.clone(),
                                           tree_mask=tree_mask.clone(), tree_pos=tree_pos.clone(),
                                           node_argmax=torch.argmax(tree_logits[0], dim=-1),
                                           best=int(best), accept_length=a, bonus=int(token)))
            draft_tokens, retrieve, tree_mask, tree_pos = self._tree(accept_feats, torch.cat((input_ids, token), dim=1),
                                                                     sampling)
            new_token += a + 1
            if self.time_log is not None:
                self.time_log.append(time.time())
            new_ids = input_ids[0, input_len:].tolist()
            if is_llama3 and self.eot_token_id in new_ids:
                break
            if self.eos_token_id in new_ids:
                break
            if new_token > max_new_tokens:
                break
            if input_ids.shape[1] > limit:
                break
        return (input_ids, new_token, idx) if log else input_ids

    @torch.no_grad()
    def naivegenerate(self, input_ids, max_new_tokens=512, max_length=2048, log=False):
        """Greedy vanilla decoding through the same preallocated KV (ea_model.py:305-380, greedy branch)."""
        input_ids = input_ids.clone()
        kv = self._kv(max_length)
        input_len = input_ids.shape[1]
        hidden, _ = self.target.forward(input_ids, kv)
        new_token = 0
        limit = max_length - self.head.total_tokens - 10
        idx = 0
        for idx in range(limit):
            nxt = torch.argmax(self.target.lm_head(hidden)[:, -1])[None, None]
            hidden, _ = self.target.forward(nxt, kv)
            input_ids = torch.cat([input_ids, nxt], dim=-1)
            new_token += 1
            if self.eos_token_id in input_ids[0, input_len:].tolist():
                break
            if new_token > max_new_tokens:
                break
            if input_ids.shape[1] > limit:
                break
        return (input_ids, new_token, idx) if log else input_ids

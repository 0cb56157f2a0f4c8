"""`EaModel`: the reference's public API (eagle/model/ea_model.py:25-558) over the H100 engine.

Same constructor arguments, method names, argument meanings, return conventions and
checkpoint format as the reference, so callers (`gen_ea_answer_*.py`, `webui.py`) switch by
changing one import.  Everything between the arguments and the returned ids -- prefill, draft
tree growth, tree-masked verification, posterior acceptance, KV compaction -- runs inside
libeagle_b200.so (hand-written sm_90a CUDA); torch is used here only to hold the caller's
tensors and to read checkpoints.  There is no PyTorch / CPU fallback path.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import warnings
from types import SimpleNamespace
from typing import Dict, Iterator, Optional

import torch

from . import _lib
from .quant import is_target_projection, quantize_4bit, quantize_fp8_block, quantize_int8_rowwise

_TORCH2ENGINE = {torch.bfloat16: _lib.DT_BF16, torch.float16: _lib.DT_FP16, torch.float32: _lib.DT_FP32,
                 torch.int64: _lib.DT_INT64, torch.bool: _lib.DT_BOOL, torch.int8: _lib.DT_INT8,
                 torch.uint8: _lib.DT_UINT8, torch.float8_e4m3fn: _lib.DT_FP8_E4M3}


def _llama3_inv_freq(inv_freq: torch.Tensor, rs: dict, max_position_embeddings: int) -> torch.Tensor:
    """Llama-3.1 frequency transform: what LlamaRotaryEmbedding_L31 gets from ROPE_INIT_FUNCTIONS["llama3"]
    (modeling_llama_kv.py:208-292 -> transformers.modeling_rope_utils._compute_llama3_parameters), fp32 like there."""
    factor = float(rs["factor"])
    low, high = float(rs["low_freq_factor"]), float(rs["high_freq_factor"])
    old = float(rs.get("original_max_position_embeddings", max_position_embeddings))
    low_freq_wavelen, high_freq_wavelen = old / low, old / high
    wavelen = 2 * math.pi / inv_freq
    out = torch.where(wavelen > low_freq_wavelen, inv_freq / factor, inv_freq)
    smooth = (old / wavelen - low) / (high - low)
    smoothed = (1 - smooth) * out / factor + smooth * out
    medium = ~(wavelen < high_freq_wavelen) * ~(wavelen > low_freq_wavelen)
    return torch.where(medium, smoothed, out)


def _rope_table(dim: int, n_pos: int, base: float, dtype: torch.dtype, rope_scaling: Optional[dict] = None,
                max_position_embeddings: Optional[int] = None, is_head: bool = False):
    """cos/sin caches exactly as the reference's rotary classes build them: fp32 math, cast to the model dtype on use; only the
    first dim/2 columns are distinct (emb = cat(freqs, freqs)).
      target (LlamaAttention._init_rope, modeling_llama_kv.py:607-634): no rope_scaling -> LlamaRotaryEmbedding(base=rope_theta);
        {"type": "linear"|"dynamic", "factor"} -> the scaled classes (:295-420, base=rope_theta); anything else (a Llama-3.1
        config has "rope_type": "llama3" and no "type") falls through to LlamaRotaryEmbedding_L31 (:208-292);
      head (cnets.py:215-236, cnets1.py:220-241): the linear / dynamic classes are built WITHOUT base (10000), any other
        rope_scaling raises."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2).float() / dim))
    t = torch.arange(n_pos, dtype=inv_freq.dtype)
    if rope_scaling:
        typ = rope_scaling.get("type")
        if typ in ("linear", "dynamic") and "factor" in rope_scaling:
            factor = float(rope_scaling["factor"])
            if is_head:
                inv_freq = 1.0 / (10000.0 ** (torch.arange(0, dim, 2).float() / dim))
            if typ == "linear":
                t = t / factor
            elif max_position_embeddings is not None and n_pos > max_position_embeddings:
                # LlamaDynamicNTKScalingRotaryEmbedding rebuilds its cache with a length-dependent base once the sequence outgrows
                # max_position_embeddings (:400-420); inside it the table is the unscaled one
                raise NotImplementedError(f"dynamic NTK rope scaling beyond max_position_embeddings={max_position_embeddings} "
                                          f"(engine KV capacity needs {n_pos} positions)")
        elif is_head:
            raise ValueError(f"Unknown RoPE scaling type {typ}")  # cnets.py:236
        else:
            rope_type = rope_scaling.get("rope_type", typ)
            if rope_type == "llama3":
                inv_freq = _llama3_inv_freq(inv_freq, rope_scaling, max_position_embeddings or n_pos)
            elif rope_type not in (None, "default"):
                raise NotImplementedError(f"rope_scaling type {rope_type!r} is not implemented (supported: linear, dynamic, llama3)")
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    return freqs.cos().to(dtype).contiguous(), freqs.sin().to(dtype).contiguous()


def _flatten_choices(choices):
    flat = [int(v) for c in choices for v in c]
    lens = [len(c) for c in choices]
    return (C.c_int32 * max(1, len(flat)))(*flat), (C.c_int32 * max(1, len(lens)))(*lens)


def static_tree_buffers(choices, top_k: int = 10) -> dict:
    """The integer tables of a fixed tree in the reference's formats, computed by the library's host code (no GPU):
    generate_tree_buffers (utils.py:89-207) -> tree_attn_mask [1,1,T,T], tree_indices [T], tree_position_ids [T],
    retrieve_indices [n_leaf, width]; generate_tree_buffers_for_eagle (modeling_eagle.py:625-692) -> per draft level
    attn_mask [1,1,count,cum], tree_indices [count], repeat_nums."""
    lib = _lib.load()
    n = len(choices)
    if n < 1:
        raise _lib.EngineError("static tree: empty choice list")
    flat, lens = _flatten_choices(choices)
    T = n + 1
    ti, tp = (C.c_int32 * T)(), (C.c_int32 * T)()
    tm, ri = (C.c_float * (T * T))(), (C.c_int32 * (T * T))()
    lc, ls, lr = (C.c_int32 * n)(), (C.c_int32 * n)(), (C.c_int32 * n)()
    lm = (C.c_float * (n * n))()
    n_leaf, width, n_levels, n_inner = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    _lib.check(lib.eb200_static_tree_buffers(flat, lens, n, int(top_k), ti, tp, tm, ri, C.byref(n_leaf), C.byref(width),
                                             C.byref(n_levels), lc, ls, lr, lm, C.byref(n_inner)))
    ni = n_inner.value
    full = torch.tensor(list(lm)[: ni * ni], dtype=torch.float32).view(ni, ni)
    out = {
        "tree_attn_mask": torch.tensor(list(tm), dtype=torch.float32).view(1, 1, T, T),
        "tree_indices": torch.tensor(list(ti), dtype=torch.long),
        "tree_position_ids": torch.tensor(list(tp), dtype=torch.long),
        "retrieve_indices": torch.tensor(list(ri)[: n_leaf.value * width.value], dtype=torch.long).view(n_leaf.value, width.value),
        "draft": {"attn_mask": [], "tree_indices": [], "repeat_nums": []},
    }
    start = 0
    for l in range(n_levels.value):
        cnt = lc[l]
        out["draft"]["attn_mask"].append(full[start:start + cnt, : start + cnt].clone()[None, None])
        out["draft"]["tree_indices"].append(torch.tensor(list(ls)[start:start + cnt], dtype=torch.long))
        runs = []
        for r in list(lr)[start:start + cnt]:
            if r == len(runs):
                runs.append(0)
            runs[r] += 1
        out["draft"]["repeat_nums"].append(runs)
        start += cnt
    return out


class EaModel(torch.nn.Module):
    """Drop-in for eagle.model.ea_model.EaModel (inference surface).  An nn.Module like the reference's (no parameters of its
    own: the weights live in the engine), so `.eval()`, `.training`, `.to()` callers keep working."""

    def __init__(self, target_config: dict, head_config: dict, use_eagle3: bool = True, total_token: int = 60,
                 depth: int = 7, top_k: int = 10, threshold: float = 1.0, torch_dtype: torch.dtype = torch.bfloat16,
                 device: int = 0, max_length: int = 2048, tokenizer=None, flags: int = 0, tp_rank: int = 0,
                 tp_size: int = 1, tree_choices=None, load_in_8bit: bool = False, quantization_config=None):
        super().__init__()
        self.training = False
        self.lib = _lib.load()
        # tree_choices: a fixed draft tree (e.g. eagle_b200.static_trees.mc_sim_7b_63) instead of the dynamic re-ranked one
        # (the reference's static variant: utils.py:89-207, modeling_eagle.py:863-957); fixes total_token and depth
        self.tree_choices = [list(c) for c in tree_choices] if tree_choices is not None else None
        if self.tree_choices is not None:
            total_token = len(self.tree_choices) + 1
            depth = max(len(c) for c in self.tree_choices) - 1
        self._tune_total_token = total_token == -1
        if total_token == -1:
            total_token = 60  # capacity; finalize() then self-tunes among {40,48,50,56,60} like ea_model.py:148-168
        tc, hc = target_config, head_config
        self.config = SimpleNamespace(**tc)
        self.use_eagle3 = bool(use_eagle3)
        self.hidden_size, self.vocab_size = tc["hidden_size"], tc["vocab_size"]
        self.dtype = torch_dtype
        self.device = int(device)
        self.tokenizer = tokenizer
        self.threshold = threshold  # stored and never read, like the reference (cnets.py:524)
        self.max_length = int(max_length)
        # int8 target projections (eagle_b200.quant): bitsandbytes' weight format, exact W8A16 arithmetic
        self.load_in_8bit = bool(load_in_8bit)
        # quantization_config (a transformers BitsAndBytesConfig / FineGrainedFP8Config or its dict): load_in_4bit gives 4-bit
        # target projections in bitsandbytes' nf4 / fp4 format with exact W4A16 arithmetic (eagle_b200.quant), load_in_8bit the
        # int8 ones, quant_method "fp8" transformers' fine-grained FP8 ones (128 x 128 block scales, exact W8A16 arithmetic)
        from .checkpoint import quantization_config_dict, target_weights_4bit, target_weights_fp8
        qc = quantization_config_dict(quantization_config)
        self.quant_4bit = target_weights_4bit(qc, torch_dtype)
        self.quant_fp8 = target_weights_fp8(qc, target_config.get("num_hidden_layers", 1))
        if qc and not self.quant_4bit and not self.quant_fp8:
            if not qc.get("load_in_8bit"):
                raise ValueError("quantization_config: supported are bitsandbytes load_in_4bit (nf4 / fp4) and load_in_8bit, "
                                 "and FineGrainedFP8Config (quant_method 'fp8')")
            self.load_in_8bit = True
        if self.quant_4bit and self.load_in_8bit:
            raise ValueError("load_in_8bit and a 4-bit quantization_config exclude each other")
        if self.quant_fp8 and self.load_in_8bit:
            raise ValueError("load_in_8bit and an FP8 quantization_config exclude each other")
        if self.load_in_8bit:
            flags |= _lib.FLAG_TARGET_INT8
        if self.quant_4bit:
            flags |= _lib.FLAG_TARGET_NF4 if self.quant_4bit == "nf4" else _lib.FLAG_TARGET_FP4
        if self.quant_fp8:
            flags |= _lib.FLAG_TARGET_FP8
        # attributes callers touch (ea_model.py:168; evaluation scripts)
        self.ea_layer = SimpleNamespace(total_tokens=total_token - 1, depth=depth, top_k=top_k)
        self.base_model = SimpleNamespace(config=self.config, dtype=torch_dtype, device=torch.device("cuda", int(device)))
        cfg = _lib.Config()
        cfg.abi_version = _lib.ABI_VERSION
        cfg.dtype = _lib.BF16 if torch_dtype == torch.bfloat16 else _lib.FP16
        if torch_dtype not in (torch.bfloat16, torch.float16):
            raise ValueError("eagle_b200 runs the model in bf16 or fp16 (the dtypes the reference is run in)")
        cfg.vocab_size, cfg.hidden_size = tc["vocab_size"], tc["hidden_size"]
        cfg.intermediate_size, cfg.num_layers = tc["intermediate_size"], tc["num_hidden_layers"]
        cfg.num_heads, cfg.num_kv_heads = tc["num_attention_heads"], tc.get("num_key_value_heads", tc["num_attention_heads"])
        cfg.rms_norm_eps = tc.get("rms_norm_eps", 1e-6)
        cfg.eagle3 = 1 if use_eagle3 else 0
        cfg.head_hidden_size, cfg.head_intermediate_size = hc["hidden_size"], hc["intermediate_size"]
        cfg.head_num_layers = 1 if use_eagle3 else hc.get("num_hidden_layers", 1)
        cfg.head_num_heads = hc["num_attention_heads"]
        cfg.head_num_kv_heads = hc.get("num_key_value_heads", hc["num_attention_heads"])
        cfg.draft_vocab_size = hc.get("draft_vocab_size", hc["vocab_size"]) if use_eagle3 else hc["vocab_size"]
        cfg.head_fc_bias = 0 if use_eagle3 else (1 if hc.get("bias", True) else 0)  # ea_model.py:49-54
        cfg.head_rms_norm_eps = hc.get("rms_norm_eps", 1e-6)
        cfg.total_token, cfg.depth, cfg.top_k = total_token, depth, top_k
        cfg.max_length = self.max_length
        cfg.max_rope_positions = self.max_length + 256
        cfg.tp_rank, cfg.tp_size, cfg.device, cfg.flags = tp_rank, tp_size, self.device, flags
        self._cfg = cfg
        self._h = C.c_void_p()
        _lib.check(self.lib.eb200_create(C.byref(cfg), C.byref(self._h)))
        n_pos = cfg.max_rope_positions
        head_dim = tc.get("head_dim") or tc["hidden_size"] // tc["num_attention_heads"]
        if head_dim != 128:
            raise ValueError(f"eagle_b200 kernels are written for head_dim 128 (got {head_dim})")
        tcos, tsin = _rope_table(head_dim, n_pos, float(tc.get("rope_theta", 10000.0)), torch_dtype, tc.get("rope_scaling"),
                                 tc.get("max_position_embeddings"))
        _lib.check(self.lib.eb200_set_rope_table(self._h, 0, tcos.data_ptr(), tsin.data_ptr(), n_pos))
        # cnets.py:216-223: the head uses config.rope_theta when present, else 10000
        hcos, hsin = _rope_table(128, n_pos, float(hc.get("rope_theta", 10000.0)), torch_dtype, hc.get("rope_scaling"),
                                 hc.get("max_position_embeddings"), is_head=True)
        _lib.check(self.lib.eb200_set_rope_table(self._h, 1, hcos.data_ptr(), hsin.data_ptr(), n_pos))
        if self.tree_choices is not None:
            flat, lens = _flatten_choices(self.tree_choices)
            _lib.check(self.lib.eb200_set_static_tree(self._h, flat, lens, len(self.tree_choices)))
        self._finalized = False
        self._out = torch.empty(self.max_length + 256, dtype=torch.int64).pin_memory() if torch.cuda.is_available() \
            else torch.empty(self.max_length + 256, dtype=torch.int64)

    # ---------------------------------------------------------------------------------------------
    # weights
    # ---------------------------------------------------------------------------------------------
    def _load(self, name: str, t: torch.Tensor):
        if t.dtype.is_floating_point and t.dtype != self.dtype and t.dtype != torch.float8_e4m3fn and \
                not name.endswith((".SCB", ".absmax", ".weight_scale_inv")):
            t = t.to(self.dtype)  # `.to(base_model.dtype)` (ea_model.py:77)
        t = t.contiguous()
        if t.is_cuda:
            # the engine copies on its own (non-blocking) stream: the producer stream must have finished writing `t`
            torch.cuda.current_stream(t.device).synchronize()
        shape = (C.c_int64 * t.dim())(*t.shape)
        _lib.check(self.lib.eb200_load_tensor(self._h, name.encode(), t.data_ptr(), shape, t.dim(), _TORCH2ENGINE[t.dtype]))

    def _load_target(self, name: str, t: torch.Tensor):
        """One target tensor; with load_in_8bit (4-bit, FP8) a model-dtype projection weight is quantized here (eagle_b200.quant),
        one tensor at a time, on the tensor's device, and goes in as its int8 weight + SCB pair (uint8 codes + `.weight.absmax`;
        float8_e4m3fn weight + `.weight_scale_inv`)."""
        if self.load_in_8bit and t.dtype.is_floating_point and name.endswith(".weight") and is_target_projection(name):
            q, scb = quantize_int8_rowwise(t.to(self.dtype))
            self._load(name, q)
            self._load(name[: -len("weight")] + "SCB", scb)
        elif self.quant_4bit and t.dtype.is_floating_point and name.endswith(".weight") and is_target_projection(name):
            packed, absmax = quantize_4bit(t.to(self.dtype), self.quant_4bit)
            self._load(name, packed)
            self._load(name + ".absmax", absmax)
        elif self.quant_fp8 and t.dtype.is_floating_point and t.dtype != torch.float8_e4m3fn and name.endswith(".weight") and \
                is_target_projection(name):
            q, scale_inv = quantize_fp8_block(t.to(self.dtype))
            self._load(name, q)
            self._load(name[: -len("weight")] + "weight_scale_inv", scale_inv)
        else:
            self._load(name, t)

    def load_target_state_dict(self, sd: Dict[str, torch.Tensor]):
        """HF target keys.  With load_in_8bit the projections may be model-dtype weights (quantized while loading) or int8
        `weight` + fp32 `SCB` pairs (bitsandbytes' serialization); `weight_format` entries are ignored."""
        for k, v in sd.items():
            if "rotary_emb" in k or k.endswith(".weight_format"):
                continue
            self._load_target(k, v)

    def load_head_state_dict(self, sd: Dict[str, torch.Tensor], load_emb_from_target: bool = True):
        """Draft checkpoint keys as saved by the reference's trainers (strict=False like ea_model.py:76).
        The head first embeds with the target's table (load_emb=True, cnets.py:488-519); with load_emb_from_target=False an
        `embed_tokens.weight` in the checkpoint then overwrites it, which is what the reference's load_state_dict does
        (from_pretrained passes False; synthetic fixtures that share the table pass True and save the copy)."""
        for k, v in sd.items():
            if k == "embed_tokens.weight" and load_emb_from_target is True:
                continue
            if k == "t2d" or "rotary_emb" in k:
                continue
            self._load("head." + k, v)

    def init_tp(self, group=None):
        """Tensor parallel: join the NCCL communicator (call after construction, before finalize())."""
        from .tp import init_engine_tp
        init_engine_tp(self, group)
        return self

    def finalize(self):
        _lib.check(self.lib.eb200_finalize(self._h))
        self._finalized = True
        if self._tune_total_token:
            self.tune_total_token()
        return self

    def tune_total_token(self, candidates=(40, 48, 50, 56, 60), weights=(1, 1.05, 1.07, 1.1, 1.13), iters: int = 20) -> int:
        """total_token=-1 (ea_model.py:148-168): time the target forward over `length` rows for each candidate, divide by the
        reference's expected-gain weights and keep the cheapest.  Timed on the device (CUDA events inside the library)."""
        times = []
        for length, x in zip(candidates, weights):
            ms = C.c_double()
            _lib.check(self.lib.eb200_time_target_forward(self._h, int(length), int(iters), C.byref(ms)))
            times.append(ms.value / x)
        total_token = int(candidates[times.index(min(times))])
        _lib.check(self.lib.eb200_set_total_token(self._h, total_token))
        self._cfg.total_token = total_token
        self.ea_layer.total_tokens = total_token - 1
        self.tuned_times_ms = times
        return total_token

    @classmethod
    def from_state_dicts(cls, target_config: dict, target_sd, head_config: dict, head_sd, use_eagle3=True, **kw):
        m = cls(target_config, head_config, use_eagle3=use_eagle3, **kw)
        if kw.get("tp_size", 1) > 1:
            m.init_tp()
        m.load_target_state_dict(target_sd)
        m.load_head_state_dict(head_sd)
        return m.finalize()

    @classmethod
    def from_pretrained(cls, use_eagle3=True, base_model_path=None, ea_model_path=None, total_token=60, depth=7,
                        top_k=10, threshold=1.0, **kwargs):
        """Same signature as the reference (ea_model.py:88-170).  Reads an HF Llama checkpoint directory
        (config.json + safetensors / .bin shards) and a draft-head directory (config.json + pytorch_model.bin or
        model.safetensors).  kwargs honoured: torch_dtype, max_length, device, tree_choices, load_in_8bit (int8 target projections,
        eagle_b200.quant; a checkpoint saved in transformers' bitsandbytes 8-bit format loads its int8 values as stored),
        quantization_config (a BitsAndBytesConfig or its dict: load_in_4bit with nf4 / fp4 gives 4-bit target projections; a
        checkpoint saved in transformers' bitsandbytes 4-bit format loads its codes as stored; a FineGrainedFP8Config or its dict
        gives FP8 target projections, and a checkpoint saved in transformers' fine-grained FP8 format loads its FP8 weights as
        stored); HF placement knobs (`device_map`, `low_cpu_mem_usage`) are accepted with a warning, a bare load_in_4bit and
        anything else raise."""
        from .checkpoint import (check_4bit_checkpoint, iter_4bit_triples, iter_checkpoint_tensors, iter_fp8_pairs, iter_int8_pairs,
                                 quantization_config_dict, read_json, target_weights_4bit, target_weights_fp8, target_weights_int8)
        honoured = {"torch_dtype", "max_length", "device", "tree_choices", "load_in_8bit", "load_in_4bit", "quantization_config"}
        placement = {"device_map", "low_cpu_mem_usage"}  # HF / accelerate loading knobs
        unknown = set(kwargs) - honoured - placement
        if unknown:
            raise TypeError(f"EaModel.from_pretrained: unsupported arguments {sorted(unknown)}")
        ignored = sorted(k for k in kwargs if k in placement and kwargs[k] not in (None, False))
        if kwargs.get("load_in_4bit"):
            # a bare load_in_4bit meant transformers 4.x's implicit defaults (fp4, fp32 compute) and is gone from transformers 5
            raise ValueError("a bare load_in_4bit=True is not supported: name the 4-bit format, "
                             "quantization_config=BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type='nf4' or 'fp4')")
        if ignored:
            warnings.warn(f"eagle_b200 places the whole model on one GPU (`device`); ignoring {ignored}", stacklevel=2)
        tc = read_json(os.path.join(base_model_path, "config.json"))
        if tc.get("architectures", ["LlamaForCausalLM"])[0] != "LlamaForCausalLM":
            raise ValueError("eagle_b200 supports Llama-family targets (the configs named in BASELINE.json)")
        dtype = kwargs.get("torch_dtype", torch.float16)
        # 4-bit first (target_weights_int8 refuses every 4-bit request): codes stored by transformers' bitsandbytes 4-bit
        # serialization, else a 4-bit quantization_config argument
        qc_arg = quantization_config_dict(kwargs.get("quantization_config"))
        stored_4bit = target_weights_4bit(tc.get("quantization_config"), dtype, pre_quantized=True)
        asked_4bit = target_weights_4bit(qc_arg, dtype, pre_quantized=bool(stored_4bit))
        asked_8bit = bool(kwargs.get("load_in_8bit")) or bool(qc_arg.get("load_in_8bit"))
        if asked_4bit and asked_8bit:
            raise ValueError("load_in_8bit and a 4-bit quantization_config exclude each other")
        if stored_4bit:
            # the stored format decides; a request for another one is refused rather than ignored
            if asked_8bit or (asked_4bit and asked_4bit != stored_4bit):
                raise ValueError(f"{base_model_path} holds bitsandbytes {stored_4bit} weights; the request for "
                                 f"{'load_in_8bit' if asked_8bit else asked_4bit} conflicts with them")
            check_4bit_checkpoint(base_model_path, stored_4bit, dtype)
        elif asked_4bit and tc.get("quantization_config"):
            raise ValueError(f"{base_model_path} is already quantized (quantization_config {tc['quantization_config']}); a 4-bit "
                             f"quantization_config applies to bf16 / fp16 checkpoints only")
        quant_4bit = stored_4bit or asked_4bit
        # FP8: a stored FP8 checkpoint is recognised only when no int8 request is made (load_in_8bit on it is refused by
        # target_weights_int8, as before FP8 loaded); an FP8 quantization_config applies to bf16 / fp16 checkpoints or to a
        # checkpoint already in that format
        n_layers = tc.get("num_hidden_layers", 1)
        asked_fp8 = target_weights_fp8(qc_arg, n_layers)
        if asked_fp8 and asked_8bit:
            raise ValueError("load_in_8bit and an FP8 quantization_config exclude each other")
        stored_fp8 = not (quant_4bit or asked_8bit) and target_weights_fp8(tc.get("quantization_config"), n_layers)
        if asked_fp8 and tc.get("quantization_config") and not stored_fp8:
            raise ValueError(f"{base_model_path} is already quantized (quantization_config {tc['quantization_config']}); an FP8 "
                             f"quantization_config applies to bf16 / fp16 checkpoints only")
        fp8 = stored_fp8 or asked_fp8
        int8 = False if (quant_4bit or fp8) else target_weights_int8(tc, kwargs.get("load_in_8bit", False) or bool(qc_arg.get("load_in_8bit")))
        hc = read_json(os.path.join(ea_model_path, "config.json"))
        tok = None
        try:
            from transformers import AutoTokenizer
            tok = AutoTokenizer.from_pretrained(base_model_path, use_fast=False)
        except Exception:
            tok = None
        m = cls(tc, hc, use_eagle3=use_eagle3, total_token=total_token, depth=depth, top_k=top_k, threshold=threshold,
                torch_dtype=dtype, device=kwargs.get("device", 0), max_length=kwargs.get("max_length", 2048), tokenizer=tok,
                tree_choices=kwargs.get("tree_choices"), load_in_8bit=int8,
                quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": quant_4bit} if quant_4bit else
                                    {"quant_method": "fp8"} if fp8 else None)
        triples = iter_4bit_triples(base_model_path, stored_4bit, dtype) if stored_4bit else \
            iter_fp8_pairs(base_model_path) if stored_fp8 else iter_int8_pairs(base_model_path)
        for k, v, aux in triples:
            if "rotary_emb" in k:
                continue
            if aux is not None:  # stored bitsandbytes int8 / 4-bit / FP8: loaded as is, not requantized
                m._load(k, v)
                m._load(k + ".absmax" if stored_4bit else k[: -len("weight")] + ("weight_scale_inv" if stored_fp8 else "SCB"), aux)
            else:
                m._load_target(k, v)
        head_sd = dict(iter_checkpoint_tensors(ea_model_path, prefer_bin=True))
        m.load_head_state_dict(head_sd, load_emb_from_target=False)  # a checkpoint embed_tokens wins (ea_model.py:76)
        return m.finalize()

    def get_tokenizer(self):
        return self.tokenizer

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.eb200_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---------------------------------------------------------------------------------------------
    # generation
    # ---------------------------------------------------------------------------------------------
    def _gen_params(self, temperature, top_p, top_k, max_new_tokens, max_length, is_llama3):
        gp = _lib.GenParams()
        gp.temperature, gp.top_p, gp.top_k = float(temperature), float(top_p), int(top_k)
        gp.max_new_tokens, gp.max_length = int(max_new_tokens), int(max_length)
        eos = getattr(self.tokenizer, "eos_token_id", None) if self.tokenizer is not None else None
        gp.eos_token_id = -1 if eos is None else int(eos)
        gp.stop_token_id = -1
        if is_llama3 and self.tokenizer is not None:
            gp.stop_token_id = int(self.tokenizer.convert_tokens_to_ids("<|eot_id|>"))
        # The reference draws from the global RNGs (random.random, torch.multinomial), so consecutive calls continue one stream.
        # Here each sampling call takes a fresh 63-bit seed from torch's default generator: reproducible under
        # torch.manual_seed, different from call to call.  Greedy calls leave the generator untouched, like the reference.
        gp.seed = int(torch.randint(0, 2 ** 63 - 1, (1,)).item()) if float(temperature) > 1e-5 else 0
        return gp

    def _check_call(self, input_ids, max_length):
        if not self._finalized:
            raise RuntimeError("weights not loaded: call finalize() / use from_pretrained")
        if input_ids.dim() != 2 or input_ids.shape[0] != 1:
            raise ValueError("Only support batch size 1 for now!!")  # the reference's commented assert (ea_model.py:219)
        if max_length > self.max_length:
            raise ValueError(f"max_length {max_length} exceeds the KV capacity {self.max_length} allocated at load time")
        ids = input_ids.to(torch.int64).contiguous()
        if ids.is_cuda:
            torch.cuda.current_stream(ids.device).synchronize()  # engine stream is not ordered after torch's
        return ids

    def _run(self, fn, input_ids, temperature, top_p, top_k, max_new_tokens, max_length, log, is_llama3):
        ids = self._check_call(input_ids, max_length)
        gp = self._gen_params(temperature, top_p, top_k, max_new_tokens, max_length, is_llama3)
        n, new_token, steps = C.c_int32(), C.c_int32(), C.c_int32()
        _lib.check(fn(self._h, ids.data_ptr(), ids.shape[1], C.byref(gp), self._out.data_ptr(), self._out.numel(),
                      C.byref(n), C.byref(new_token), C.byref(steps)))
        out = self._out[: n.value].clone()[None].to(input_ids.device)
        return (out, new_token.value, steps.value) if log else out

    @torch.no_grad()
    def eagenerate(self, input_ids, temperature=0.0, top_p=0.0, top_k=0.0, max_new_tokens=512, max_length=2048,
                   log=False, is_llama3=False):
        """ea_model.py:198-303.  Returns ids [1, P+n] (or (ids, new_token, idx) with log=True)."""
        return self._run(self.lib.eb200_generate, input_ids, temperature, top_p, top_k, max_new_tokens, max_length, log, is_llama3)

    @torch.no_grad()
    def naivegenerate(self, input_ids, temperature=0.0, top_p=0.0, top_k=0.0, max_new_tokens=512, max_length=2048,
                      log=False, is_llama3=False):
        """ea_model.py:305-380: vanilla autoregressive decoding through the same engine and KV."""
        return self._run(self.lib.eb200_naive_generate, input_ids, temperature, top_p, top_k, max_new_tokens, max_length, log,
                         is_llama3)

    @torch.no_grad()
    def ea_generate(self, input_ids, temperature=0.0, top_p=0.0, top_k=0.0, max_new_tokens=512, max_length=2048,
                    log=False, is_llama3=False) -> Iterator[torch.Tensor]:
        """ea_model.py:382-483: generator yielding the full ids after every cycle."""
        ids = self._check_call(input_ids, max_length)
        gp = self._gen_params(temperature, top_p, top_k, max_new_tokens, max_length, is_llama3)
        first = C.c_int64()
        _lib.check(self.lib.eb200_prefill(self._h, ids.data_ptr(), ids.shape[1], C.byref(gp), C.byref(first)))
        cur = ids.cpu()
        limit = max_length - self.ea_layer.total_tokens - 10
        toks = (C.c_int64 * 16)()
        n, nxt = C.c_int32(), C.c_int64()
        new_token = 0
        for _ in range(limit):
            _lib.check(self.lib.eb200_step(self._h, toks, C.byref(n), C.byref(nxt)))
            new = torch.tensor([toks[j] for j in range(n.value)], dtype=torch.int64)[None]
            cur = torch.cat((cur, new), dim=1)
            new_token += n.value
            yield cur.to(input_ids.device)
            new_list = cur[0, ids.shape[1]:].tolist()
            if gp.stop_token_id >= 0 and gp.stop_token_id in new_list:
                break
            if gp.eos_token_id >= 0 and gp.eos_token_id in new_list:
                break
            if new_token > max_new_tokens:
                break
            if cur.shape[1] > limit:
                break

    @torch.no_grad()
    def naive_generate(self, input_ids, temperature=0.0, top_p=0.0, top_k=0.0, max_new_tokens=512, max_length=2048,
                       log=False, is_llama3=False) -> Iterator[torch.Tensor]:
        """ea_model.py:485-558: generator form of naivegenerate; yields the ids after EVERY decoded token."""
        ids = self._check_call(input_ids, max_length)
        gp = self._gen_params(temperature, top_p, top_k, max_new_tokens, max_length, is_llama3)
        first = C.c_int64()
        _lib.check(self.lib.eb200_naive_begin(self._h, ids.data_ptr(), ids.shape[1], C.byref(gp), C.byref(first)))
        cur = ids.cpu()
        limit = max_length - self.ea_layer.total_tokens - 10
        fed, nxt = C.c_int64(), C.c_int64()
        new_token = 0
        for _ in range(limit):
            _lib.check(self.lib.eb200_naive_step(self._h, C.byref(fed), C.byref(nxt)))
            cur = torch.cat((cur, torch.tensor([[fed.value]], dtype=torch.int64)), dim=1)
            new_token += 1
            yield cur.to(input_ids.device)
            if gp.stop_token_id >= 0 and fed.value == gp.stop_token_id:
                break
            if gp.eos_token_id >= 0 and fed.value == gp.eos_token_id:
                break
            if new_token > max_new_tokens:
                break
            if cur.shape[1] > limit:
                break

    # ---------------------------------------------------------------------------------------------
    # inspection helpers used by the parity tests
    # ---------------------------------------------------------------------------------------------
    def prefill(self, input_ids):
        ids = self._check_call(input_ids, self.max_length)
        gp = self._gen_params(0.0, 0.0, 0, 0, self.max_length, False)
        first = C.c_int64()
        _lib.check(self.lib.eb200_prefill(self._h, ids.data_ptr(), ids.shape[1], C.byref(gp), C.byref(first)))
        return int(first.value)

    def step(self):
        toks = (C.c_int64 * 16)()
        n, nxt = C.c_int32(), C.c_int64()
        _lib.check(self.lib.eb200_step(self._h, toks, C.byref(n), C.byref(nxt)))
        return [int(toks[j]) for j in range(n.value)], int(nxt.value)

    def get_tree(self):
        """(draft_tokens [1,T], retrieve_indices [n_leaf, max_depth], tree_mask [1,1,T,T], tree_position_ids [T])
        in the formats topK_genrate returns (cnets.py:823-827)."""
        T = self._cfg.total_token
        dt = torch.empty(T, dtype=torch.int64)
        tm = torch.empty(T * T, dtype=torch.float32)
        tp = torch.empty(T, dtype=torch.int64)
        ri = torch.full((T * 16,), -1, dtype=torch.int64)
        nl, md = C.c_int32(), C.c_int32()
        _lib.check(self.lib.eb200_get_tree(self._h, dt.data_ptr(), tm.data_ptr(), tp.data_ptr(), ri.data_ptr(), C.byref(nl), C.byref(md)))
        return dt[None], ri[: nl.value * md.value].view(nl.value, md.value), tm.view(1, 1, T, T), tp

    def get_verify(self):
        T = self._cfg.total_token
        am = torch.empty(T, dtype=torch.int64)
        best, acc, n = C.c_int32(), C.c_int32(), C.c_int32()
        _lib.check(self.lib.eb200_get_verify(self._h, am.data_ptr(), C.byref(best), C.byref(acc), C.byref(n)))
        return am, best.value, acc.value, n.value

    def debug_read(self, what: str) -> torch.Tensor:
        r, c = C.c_int32(), C.c_int32()
        _lib.check(self.lib.eb200_debug_read(self._h, what.encode(), None, 0, C.byref(r), C.byref(c)))
        out = torch.empty(r.value, c.value, dtype=torch.float32)
        _lib.check(self.lib.eb200_debug_read(self._h, what.encode(), out.data_ptr(), out.numel(), C.byref(r), C.byref(c)))
        return out

    def cuda_stream(self):
        """The engine's stream as a torch ExternalStream (to bracket calls with CUDA events)."""
        return torch.cuda.ExternalStream(int(self.lib.eb200_get_stream(self._h)), device=self.device)

    def set_uniforms(self, values):
        """Sampling path only: uniforms the posterior consumes in order before its seeded RNG (tests replay a stream)."""
        t = torch.tensor(list(values), dtype=torch.float32)
        _lib.check(self.lib.eb200_set_uniforms(self._h, t.data_ptr() if t.numel() else None, t.numel()))

    def set_profiling(self, on: bool):
        _lib.check(self.lib.eb200_set_profiling(self._h, 1 if on else 0))

    def stats(self) -> dict:
        s = _lib.Stats()
        _lib.check(self.lib.eb200_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in _lib.Stats._fields_}

    def reset_stats(self):
        _lib.check(self.lib.eb200_reset_stats(self._h))

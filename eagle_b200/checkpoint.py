"""Checkpoint readers: HF Llama directories and EAGLE draft-head directories (SURVEY.md 5).

The formats are the reference's: a target directory with `config.json` and
`model.safetensors[.index.json]` / `pytorch_model[-*].bin` shards (read by HF `from_pretrained`,
ea_model.py:101-118), and a head directory with `config.json` plus `pytorch_model.bin` (preferred,
ea_model.py:124-129) or `model.safetensors` (:130-135).  Tensors are streamed one at a time so a
16 GB checkpoint never needs a second host copy.
"""
from __future__ import annotations

import glob
import json
import os
import re
from typing import Iterator, Optional, Tuple

import torch


def read_json(path: str) -> dict:
    with open(path, "r") as f:
        return json.load(f)


def _iter_safetensors(path: str) -> Iterator[Tuple[str, torch.Tensor]]:
    from safetensors import safe_open
    with safe_open(path, framework="pt", device="cpu") as f:
        for k in f.keys():
            yield k, f.get_tensor(k)


def iter_checkpoint_tensors(directory: str, prefer_bin: bool = False) -> Iterator[Tuple[str, torch.Tensor]]:
    st = sorted(glob.glob(os.path.join(directory, "*.safetensors")))
    bins = sorted(glob.glob(os.path.join(directory, "pytorch_model*.bin")))
    if prefer_bin and bins:
        st = []
    if st:
        for p in st:
            yield from _iter_safetensors(p)
        return
    if bins:
        for p in bins:
            sd = torch.load(p, map_location="cpu", weights_only=True)
            for k, v in sd.items():
                yield k, v
        return
    raise FileNotFoundError(f"no *.safetensors or pytorch_model*.bin under {directory}")


def target_weights_int8(config: dict, load_in_8bit=False, load_in_4bit=False) -> bool:
    """Whether the target's decoder projections load as int8 (EaModel `load_in_8bit`).  True for `load_in_8bit=True` on a
    bf16 / fp16 checkpoint and for a checkpoint transformers saved in bitsandbytes 8-bit format (`quantization_config` with
    `load_in_8bit: true`), whose stored int8 values are used as they are.  Raises ValueError, before anything is loaded, for
    what is not supported: 4-bit loading and any other quantization_config (4-bit, fp8, gptq, ...)."""
    supported = ("supported: load_in_8bit=True (int8 target projections in bitsandbytes' weight format, W8A16 arithmetic) "
                 "on bf16 / fp16 Llama checkpoints or on transformers' bitsandbytes 8-bit checkpoints")
    if load_in_4bit:
        raise ValueError(f"eagle_b200 does not load 4-bit weights (load_in_4bit); {supported}")
    qc = config.get("quantization_config")
    if qc:
        method = qc.get("quant_method", "bitsandbytes")
        if method == "bitsandbytes" and qc.get("load_in_8bit") and not qc.get("load_in_4bit"):
            return True
        raise ValueError(f"unsupported quantization_config (quant_method={method!r}, load_in_4bit={qc.get('load_in_4bit')}); "
                         f"{supported}")
    return bool(load_in_8bit)


def iter_int8_pairs(directory: str) -> Iterator[Tuple[str, torch.Tensor, Optional[torch.Tensor]]]:
    """Tensors of a target checkpoint as (name, tensor, SCB): an int8 projection `weight` comes with its fp32 `SCB` row
    scales, every other tensor with None.  `weight_format` entries (older bitsandbytes serializations) are skipped.  Tensors
    are streamed; a weight waits only for its own SCB (adjacent in sorted safetensors key order)."""
    from .quant import is_target_projection
    weights, scales = {}, {}
    for k, v in iter_checkpoint_tensors(directory):
        if k.endswith(".weight_format"):
            continue
        if k.endswith(".SCB"):
            base = k[: -len("SCB")]
            if base in weights:
                yield base + "weight", weights.pop(base), v
            else:
                scales[base] = v
        elif k.endswith(".weight") and v.dtype == torch.int8:
            if not is_target_projection(k):
                raise ValueError(f"{k}: int8 weights are supported for the target decoder projections only")
            base = k[: -len("weight")]
            if base in scales:
                yield k, v, scales.pop(base)
            else:
                weights[base] = v
        else:
            yield k, v, None
    if weights or scales:
        raise ValueError(f"int8 checkpoint {directory}: unpaired weight / SCB entries "
                         f"{sorted(list(weights) + list(scales))[:4]}")


_DTYPE_NAMES = {torch.bfloat16: "bfloat16", torch.float16: "float16", torch.float32: "float32"}


def quantization_config_dict(quantization_config) -> dict:
    """A transformers BitsAndBytesConfig (anything with to_dict()) or its dict."""
    if quantization_config is None:
        return {}
    if hasattr(quantization_config, "to_dict"):
        return quantization_config.to_dict()
    return dict(quantization_config)


def _dtype_name(v) -> Optional[str]:
    if v is None:
        return None
    if isinstance(v, torch.dtype):
        return _DTYPE_NAMES.get(v, str(v))
    return str(v).replace("torch.", "")


def target_weights_4bit(quantization_config, torch_dtype: torch.dtype, pre_quantized: bool = False) -> Optional[str]:
    """The 4-bit code table ("nf4" / "fp4") a quantization_config asks for, or None when it does not ask for 4-bit loading.

    Honoured: `load_in_4bit` with `bnb_4bit_quant_type` nf4 or fp4 (transformers' default fp4 when unset), `bnb_4bit_quant_storage`
    uint8 or unset, and `bnb_4bit_compute_dtype` unset, float32 or the model dtype -- an fp32 matmul on upcast model-dtype inputs
    with one output rounding is the engine's arithmetic, while e.g. fp16 compute on a bf16 model first rounds the activations to
    fp16.  `bnb_4bit_use_double_quant` is refused when quantizing at load (bitsandbytes' 8-bit dynamic-map quantizer of the absmax
    is not restated); a pre-quantized checkpoint's nested absmax is decompressed exactly instead.  Raises ValueError otherwise."""
    qc = quantization_config_dict(quantization_config)
    if not qc.get("load_in_4bit"):
        return None
    method = qc.get("quant_method", "bitsandbytes")
    if method != "bitsandbytes":
        raise ValueError(f"4-bit loading supports bitsandbytes quantization only (quant_method={method!r})")
    quant_type = qc.get("bnb_4bit_quant_type") or "fp4"
    if quant_type not in ("nf4", "fp4"):
        raise ValueError(f"bnb_4bit_quant_type={quant_type!r} is not supported (nf4 or fp4)")
    storage = _dtype_name(qc.get("bnb_4bit_quant_storage"))
    if storage not in (None, "uint8"):
        raise ValueError(f"bnb_4bit_quant_storage={storage!r} is not supported (uint8)")
    compute = _dtype_name(qc.get("bnb_4bit_compute_dtype"))
    if compute not in (None, "float32", _DTYPE_NAMES.get(torch_dtype)):
        raise ValueError(f"bnb_4bit_compute_dtype={compute!r} is not supported for a {_DTYPE_NAMES.get(torch_dtype)} model: the engine "
                         f"computes W' x in fp32 with one rounding to the model dtype (leave it unset, float32 or the model dtype)")
    if qc.get("bnb_4bit_use_double_quant") and not pre_quantized:
        raise ValueError("bnb_4bit_use_double_quant=True is not supported when quantizing at load (bitsandbytes' 8-bit absmax "
                         "quantizer is not restated); double-quantized checkpoints load")
    return quant_type


_QS_PREFIX = ".weight.quant_state.bitsandbytes__"


def _check_4bit_state(name: str, st: dict, quant_map: torch.Tensor, quant_type: str, torch_dtype: torch.dtype):
    from . import quant
    if st.get("quant_type") != quant_type:
        raise ValueError(f"{name}: quant_type {st.get('quant_type')!r} differs from the config's {quant_type!r}")
    if int(st.get("blocksize", -1)) != quant.BLOCKSIZE_4BIT:
        raise ValueError(f"{name}: blocksize {st.get('blocksize')} is not supported (64, the blocksize transformers uses)")
    if str(st.get("dtype", "")).replace("torch.", "") != _DTYPE_NAMES.get(torch_dtype):
        raise ValueError(f"{name}: stored dtype {st.get('dtype')!r} differs from torch_dtype {torch_dtype}")
    if not torch.equal(quant_map.float(), quant.code_table(quant_type)):
        raise ValueError(f"{name}: quant_map differs from the engine's {quant_type} table")
    if int(st["shape"][1]) % quant.BLOCKSIZE_4BIT:
        raise ValueError(f"{name}: in-features {st['shape'][1]} are not a multiple of 64, so 64-element blocks would straddle rows")


def _decode_state(v: torch.Tensor) -> dict:
    return json.loads(bytes(v.to(torch.uint8).tolist()).decode())


def check_4bit_checkpoint(directory: str, quant_type: str, torch_dtype: torch.dtype):
    """The refusals of iter_4bit_triples, from the quant states and quant maps alone (safetensors: only those entries are read), so
    that a checkpoint the engine cannot load is refused before an engine is created."""
    st_files = sorted(glob.glob(os.path.join(directory, "*.safetensors")))
    states, maps = {}, {}
    if st_files:
        from safetensors import safe_open

        def entries():
            for p in st_files:
                with safe_open(p, framework="pt", device="cpu") as f:
                    for k in f.keys():
                        if _QS_PREFIX in k or k.endswith(".weight.quant_map"):
                            yield k, f.get_tensor(k)
    else:
        entries = lambda: iter_checkpoint_tensors(directory)  # noqa: E731
    for k, v in entries():
        if _QS_PREFIX in k:
            states[k[: k.index(_QS_PREFIX)]] = _decode_state(v)
        elif k.endswith(".weight.quant_map"):
            maps[k[: -len(".weight.quant_map")]] = v
    for base, st in sorted(states.items()):
        if base not in maps:
            raise ValueError(f"4-bit checkpoint {directory}: {base}.weight has no quant_map")
        _check_4bit_state(base + ".weight", st, maps[base], quant_type, torch_dtype)


def iter_4bit_triples(directory: str, quant_type: str, torch_dtype: torch.dtype) -> Iterator[Tuple[str, torch.Tensor, Optional[torch.Tensor]]]:
    """Tensors of a target checkpoint saved by transformers in bitsandbytes 4-bit format, as (name, tensor, absmax): a 4-bit
    projection's `weight` comes back as uint8 [out, in/2] with its fp32 absmax [out, in/64] (a double-quantized absmax is
    decompressed exactly, quant.decompress_nested_absmax), every other tensor with None.  Refused with ValueError: a blocksize
    other than 64, a quant_map other than the engine's table, a stored dtype other than `torch_dtype`, in-features not a multiple
    of 64, a quant_type other than the config's.  Written from transformers' list of keys (quantizer_bnb_4bit.py); no checkpoint
    saved by bitsandbytes itself was available to compare against."""
    from . import quant
    parts = {}
    suffixes = ("absmax", "quant_map", "nested_absmax", "nested_quant_map")

    def complete(base):
        d = parts[base]
        if "weight" not in d or "absmax" not in d or "quant_map" not in d or "state" not in d:
            return None
        st = d["state"]
        if st.get("nested_blocksize") is not None or "nested_absmax" in st:
            if "nested_absmax" not in d or "nested_quant_map" not in d:
                return None
        return d

    def finish(base, d):
        st = d["state"]
        name = base + "weight"
        _check_4bit_state(name, st, d["quant_map"], quant_type, torch_dtype)
        n, k = (int(v) for v in st["shape"])
        nb = n * k // quant.BLOCKSIZE_4BIT
        if d["weight"].numel() != n * k // 2:
            raise ValueError(f"{name}: {d['weight'].numel()} packed bytes, the quant_state shape [{n}, {k}] needs {n * k // 2}")
        if d["absmax"].numel() != nb:
            raise ValueError(f"{name}: {d['absmax'].numel()} absmax values, the quant_state shape [{n}, {k}] needs {nb}")
        absmax = d["absmax"]
        if "nested_absmax" in d:
            absmax = quant.decompress_nested_absmax(absmax, d["nested_absmax"], d["nested_quant_map"], int(st["nested_blocksize"]),
                                                    float(st["nested_offset"]))
        packed = d["weight"].reshape(n, k // 2)
        return name, packed, absmax.float().reshape(n, k // quant.BLOCKSIZE_4BIT)

    for k, v in iter_checkpoint_tensors(directory):
        base = None
        if _QS_PREFIX in k:
            base = k[: k.index(_QS_PREFIX) + 1]
            parts.setdefault(base, {})["state"] = _decode_state(v)
        elif any(k.endswith(".weight." + s) for s in suffixes):
            base, suf = k.rsplit(".weight.", 1)
            base += "."
            parts.setdefault(base, {})[suf] = v
        elif k.endswith(".weight") and v.dtype == torch.uint8:
            base = k[: -len("weight")]
            parts.setdefault(base, {})["weight"] = v
        else:
            yield k, v, None
            continue
        d = complete(base)
        if d is not None:
            yield finish(base, parts.pop(base))
    if parts:
        raise ValueError(f"4-bit checkpoint {directory}: incomplete entries for {sorted(parts)[:4]}")


def bnb_4bit_entries(name: str, w: torch.Tensor, quant_type: str, double_quant: bool = False) -> dict:
    """The keys transformers writes for one bitsandbytes 4-bit `name` ("...weight") quantized from `w` (quant.quantize_4bit).
    With double_quant the absmax is stored as uint8 codes of a 256-entry map over 256-value blocks around their mean; the map and
    rounding are this function's own (bitsandbytes' dynamic map is not restated), and the decompressed absmax is what the
    checkpoint holds."""
    from . import quant
    packed, absmax = quant.quantize_4bit(w, quant_type)
    n, k = w.shape
    state = {"quant_type": quant_type, "blocksize": quant.BLOCKSIZE_4BIT, "dtype": _DTYPE_NAMES[w.dtype], "shape": [n, k]}
    out = {name: packed.reshape(-1, 1), name + ".quant_map": quant.code_table(quant_type)}
    flat = absmax.reshape(-1)
    if double_quant:
        nbs = 256
        offset = float(flat.mean())
        centred = flat - offset
        pad = (-centred.numel()) % nbs
        nested_absmax = torch.nn.functional.pad(centred, (0, pad)).reshape(-1, nbs).abs().amax(dim=1)
        nested_map = torch.linspace(-1.0, 1.0, 256, dtype=torch.float32)
        scale = torch.where(nested_absmax > 0, nested_absmax, torch.ones_like(nested_absmax)).repeat_interleave(nbs)[: flat.numel()]
        codes = torch.bucketize(centred / scale, (nested_map[1:] + nested_map[:-1]) / 2).to(torch.uint8)
        out[name + ".absmax"] = codes
        out[name + ".nested_absmax"] = nested_absmax
        out[name + ".nested_quant_map"] = nested_map
        state.update({"nested_blocksize": nbs, "nested_offset": offset, "nested_dtype": "float32"})
    else:
        out[name + ".absmax"] = flat
    out[name + ".quant_state.bitsandbytes__" + quant_type] = torch.tensor(list(json.dumps(state).encode()), dtype=torch.uint8)
    return out


def target_weights_fp8(quantization_config, num_layers: int = 1) -> bool:
    """Whether a quantization_config (transformers' FineGrainedFP8Config or its dict, or a checkpoint's `quantization_config`)
    asks for FP8 target projections.  Honoured: `quant_method` "fp8" with `weight_block_size` [128, 128] (transformers' default
    when absent) and `activation_scheme` "dynamic": the engine multiplies by the dequantized W' in the model dtype, so only the
    weight format matters.  Raises ValueError for what it cannot honour: a static activation scheme (its checkpoints carry
    `activation_scale` tensors the model-dtype arithmetic would ignore), any other block size or a per-tensor scale
    (`weight_block_size: null`), `dequantize: true`, and a `modules_to_not_convert` that names a decoder projection of one of
    the `num_layers` layers (transformers' should_convert_module rule)."""
    qc = quantization_config_dict(quantization_config)
    method = qc.get("quant_method")
    if getattr(method, "value", method) != "fp8":
        return False
    scheme = str(qc.get("activation_scheme") or "dynamic").lower()
    if scheme != "dynamic":
        raise ValueError(f"FP8 activation_scheme={scheme!r} is not supported: static schemes carry activation_scale tensors; "
                         f"the engine loads dynamic-scheme FP8 weights and multiplies by them in the model dtype")
    block = qc.get("weight_block_size", (128, 128))
    if block is None or [int(v) for v in block] != [128, 128]:
        raise ValueError(f"FP8 weight_block_size={block!r} is not supported: the engine reads one scale per 128 x 128 block "
                         f"(FineGrainedFP8Config's default)")
    if qc.get("dequantize"):
        raise ValueError("FP8 dequantize=True is not supported: load the dequantized bf16 / fp16 checkpoint instead")
    from .quant import PROJECTIONS
    for key in qc.get("modules_to_not_convert") or ():
        for i in range(max(1, int(num_layers))):
            for proj in PROJECTIONS:
                name = f"model.layers.{i}.{proj}"
                if re.match(f"{key}\\.", name) or re.match(f"{key}", name) or name.endswith(key):
                    raise ValueError(f"FP8 modules_to_not_convert entry {key!r} keeps the decoder projection {name} unquantized; the "
                                     f"engine stores every decoder projection in FP8 or none")
    return True


def fp8_config_dict() -> dict:
    """The quantization_config transformers writes for FineGrainedFP8Config() (lm_head stays in the model dtype)."""
    return {"quant_method": "fp8", "activation_scheme": "dynamic", "weight_block_size": [128, 128], "dequantize": False,
            "modules_to_not_convert": ["lm_head"]}


def iter_fp8_pairs(directory: str) -> Iterator[Tuple[str, torch.Tensor, Optional[torch.Tensor]]]:
    """Tensors of a target checkpoint saved in transformers' fine-grained FP8 format as (name, tensor, weight_scale_inv): an FP8
    projection's float8_e4m3fn `weight` comes with its fp32 [out / 128, in / 128] `weight_scale_inv`, every other tensor with None.
    Streamed like iter_int8_pairs.  Refused with ValueError: FP8 weights outside the decoder projections, `activation_scale`
    tensors (static activation schemes), a scale whose shape does not tile its weight in 128 x 128 blocks, unpaired entries."""
    from .quant import FP8_BLOCK, is_target_projection
    weights, scales = {}, {}

    def pair(name, q, s):
        n, k = q.shape
        if n % FP8_BLOCK or k % FP8_BLOCK or tuple(s.shape) != (n // FP8_BLOCK, k // FP8_BLOCK):
            raise ValueError(f"{name}: weight [{n}, {k}] and weight_scale_inv {list(s.shape)} are not one scale per 128 x 128 block")
        return name, q, s

    for k, v in iter_checkpoint_tensors(directory):
        if k.endswith(".activation_scale"):
            raise ValueError(f"{k}: static FP8 activation scales are not supported (activation_scheme 'dynamic' only)")
        if k.endswith(".weight_scale_inv"):
            base = k[: -len("weight_scale_inv")]
            if base in weights:
                yield pair(base + "weight", weights.pop(base), v)
            else:
                scales[base] = v
        elif v.dtype == torch.float8_e4m3fn:
            if not (k.endswith(".weight") and is_target_projection(k)):
                raise ValueError(f"{k}: FP8 weights are supported for the target decoder projections only")
            base = k[: -len("weight")]
            if base in scales:
                yield pair(k, v, scales.pop(base))
            else:
                weights[base] = v
        else:
            yield k, v, None
    if weights or scales:
        raise ValueError(f"FP8 checkpoint {directory}: unpaired weight / weight_scale_inv entries {sorted(list(weights) + list(scales))[:4]}")


def save_head_checkpoint(directory: str, head_config: dict, head_sd: dict, as_bin: bool = False):
    """Write a draft-head directory in the reference's format (config.json + weights)."""
    os.makedirs(directory, exist_ok=True)
    with open(os.path.join(directory, "config.json"), "w") as f:
        json.dump({"architectures": ["LlamaForCausalLM"], "model_type": "llama", **head_config}, f, indent=1)
    sd = {k: v.contiguous().cpu() for k, v in head_sd.items()}
    if as_bin:
        torch.save(sd, os.path.join(directory, "pytorch_model.bin"))
    else:
        from safetensors.torch import save_file
        save_file(sd, os.path.join(directory, "model.safetensors"))


def save_target_checkpoint(directory: str, target_config: dict, target_sd: dict, load_in_4bit: Optional[str] = None,
                           double_quant: bool = False, fp8: bool = False):
    """HF Llama directory (config.json + model.safetensors).  A state dict holding int8 `weight` + `SCB` pairs is saved the
    way transformers saves a bitsandbytes 8-bit model: add `quantization_config` with `load_in_8bit: true` to the config.
    load_in_4bit="nf4" | "fp4" saves the model-dtype decoder projections of `target_sd` in bitsandbytes' 4-bit format instead
    (bnb_4bit_entries, double-quantized absmax with double_quant) and adds the matching `quantization_config`.  fp8=True saves
    them in transformers' fine-grained FP8 format (quant.quantize_fp8_block: float8_e4m3fn `weight` + fp32 `weight_scale_inv`)
    with FineGrainedFP8Config's `quantization_config`."""
    os.makedirs(directory, exist_ok=True)
    if fp8:
        from .quant import is_target_projection, quantize_fp8_block
        sd = {}
        for k, v in target_sd.items():
            if k.endswith(".weight") and v.dtype.is_floating_point and is_target_projection(k):
                sd[k], sd[k[: -len("weight")] + "weight_scale_inv"] = quantize_fp8_block(v)
            else:
                sd[k] = v
        target_sd = sd
        target_config = {**target_config, "quantization_config": fp8_config_dict()}
    if load_in_4bit:
        from .quant import is_target_projection
        sd = {}
        for k, v in target_sd.items():
            if k.endswith(".weight") and v.dtype.is_floating_point and is_target_projection(k):
                sd.update(bnb_4bit_entries(k, v, load_in_4bit, double_quant))
            else:
                sd[k] = v
        target_sd = sd
        target_config = {**target_config, "quantization_config": {
            "quant_method": "bitsandbytes", "load_in_4bit": True, "load_in_8bit": False, "bnb_4bit_quant_type": load_in_4bit,
            "bnb_4bit_use_double_quant": bool(double_quant), "bnb_4bit_quant_storage": "uint8",
            "bnb_4bit_compute_dtype": target_config.get("torch_dtype", "float32")}}
    with open(os.path.join(directory, "config.json"), "w") as f:
        json.dump({"architectures": ["LlamaForCausalLM"], "model_type": "llama", **target_config}, f, indent=1)
    from safetensors.torch import save_file
    save_file({k: v.contiguous().cpu() for k, v in target_sd.items()}, os.path.join(directory, "model.safetensors"))

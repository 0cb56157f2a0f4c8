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


def save_target_checkpoint(directory: str, target_config: dict, target_sd: dict):
    """HF Llama directory (config.json + model.safetensors).  A state dict holding int8 `weight` + `SCB` pairs is saved the
    way transformers saves a bitsandbytes 8-bit model: add `quantization_config` with `load_in_8bit: true` to the config."""
    os.makedirs(directory, exist_ok=True)
    with open(os.path.join(directory, "config.json"), "w") as f:
        json.dump({"architectures": ["LlamaForCausalLM"], "model_type": "llama", **target_config}, f, indent=1)
    from safetensors.torch import save_file
    save_file({k: v.contiguous().cpu() for k, v in target_sd.items()}, os.path.join(directory, "model.safetensors"))

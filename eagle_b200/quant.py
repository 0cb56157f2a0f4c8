"""8-bit target weights (`load_in_8bit=True`): bitsandbytes' weight format with an exact W8A16 product.

A quantized projection weight W [out, in] is stored as `weight` int8 plus `SCB` fp32 [out], the row absmax -- the keys
transformers serializes bitsandbytes 8-bit models with.  The engine multiplies the model-dtype activations by

    W' = dequantize_int8_rowwise(q, SCB, dtype) = dtype((q.float() * SCB[:, None]) * 7.874015718698502e-3)

which is transformers' own dequantization (integrations/bitsandbytes.py), so an int8 engine computes bit for bit what a
bf16 / fp16 engine loaded with W' computes.  bitsandbytes' LLM.int8 matmul (int8 activations, outlier columns above 6.0 in
fp16) is not reproduced: the tokens of an int8 engine are those of W' in the model dtype.
"""
from __future__ import annotations

from typing import Tuple

import torch

# the int8 target projections of a Llama decoder layer (the modules transformers converts; lm_head and embeddings stay)
PROJECTIONS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
               "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj")


def is_target_projection(name: str) -> bool:
    """`model.layers.{i}.<projection>.weight` (or `.SCB`) of the target model."""
    if not name.startswith("model.layers."):
        return False
    rest = name[len("model.layers."):].split(".", 1)
    if len(rest) != 2 or not rest[0].isdigit():
        return False
    return any(rest[1] in (p + ".weight", p + ".SCB") for p in PROJECTIONS)


def quantize_int8_rowwise(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Row-wise absmax quantization of a [out, in] weight: SCB = max|W_row| in fp32,
    q = round_half_even(W.float() * (127 / SCB)) saturated to [-127, 127]; an all-zero row gives SCB = 0 and q = 0.

    This restates bitsandbytes' row-wise rule (`int8_vectorwise_quant`) from its description; bitsandbytes is not a
    dependency, so the two have not been compared value for value.  Runs on w's device."""
    if w.dim() != 2 or not w.dtype.is_floating_point:
        raise ValueError("quantize_int8_rowwise expects a floating-point [out, in] weight")
    wf = w.float()
    scb = wf.abs().amax(dim=1)
    inv = torch.where(scb > 0, 127.0 / torch.where(scb > 0, scb, torch.ones_like(scb)), torch.zeros_like(scb))
    q = torch.round(wf * inv[:, None]).clamp_(-127, 127).to(torch.int8)
    return q.contiguous(), scb.contiguous()


def dequantize_int8_rowwise(q: torch.Tensor, scb: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """W' = dtype((q.float() * SCB[:, None]) * 7.874015718698502e-3): two fp32 roundings in that order, then one cast --
    transformers' `weight.data * state.SCB.view(-1, 1) * 7.874015718698502e-3`.  The values the int8 engine multiplies by."""
    return ((q.float() * scb.float().view(-1, 1)) * 7.874015718698502e-3).to(dtype)

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


# ---------------------------------------------------------------------------------------------------------------------------
# 4-bit target weights (`quantization_config=BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type="nf4" | "fp4")`)
#
# bitsandbytes stores a [out, in] weight blockwise over the flattened tensor, blocksize 64: one fp32 absmax per 64 consecutive
# elements and two 4-bit codes per byte, element 2j in the HIGH nibble of byte j.  The engine multiplies by
#
#     W' = dequantize_4bit(packed, absmax) = dtype(code[q] * absmax)      (one fp32 product, one round-to-nearest cast)
#
# which is what transformers' Linear4bit multiplies by for more than one row (dequantize_4bit, then a model-dtype matmul), so a
# 4-bit engine computes bit for bit what a bf16 / fp16 engine loaded with W' computes.  bitsandbytes' single-row `gemv_4bit`
# kernel has other arithmetic and is not reproduced: a 4-bit engine's tokens are those of W'.
# ---------------------------------------------------------------------------------------------------------------------------
BLOCKSIZE_4BIT = 64
# The code tables, transcribed from the constants of bitsandbytes' CUDA dequantizers (csrc/kernels.cu: dDequantizeNF4 and
# dDequantizeFP4Tree).  FP4 codes 8..15 are the negated values of codes 0..7; bitsandbytes computes them as (c * absmax) * -1,
# so code 8 dequantizes to -0.0, which the signed zero in the table reproduces.  tests/test_w4_cpu.py pins the fp32 bit patterns.
NF4_CODE = (-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635, -0.18477343022823334,
            -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141458511, 0.24611230194568634, 0.33791524171829224,
            0.44070982933044434, 0.5626170039176941, 0.7229568362236023, 1.0)
_FP4_POS = (0.0, 0.0052083333, 0.66666667, 1.0, 0.33333333, 0.5, 0.16666667, 0.25)
FP4_CODE = _FP4_POS + tuple(-v for v in _FP4_POS)
QUANT_TYPES_4BIT = ("nf4", "fp4")


def code_table(quant_type: str) -> torch.Tensor:
    """The 16 fp32 code values of `nf4` or `fp4`."""
    if quant_type not in QUANT_TYPES_4BIT:
        raise ValueError(f"4-bit quant_type must be one of {QUANT_TYPES_4BIT}, got {quant_type!r}")
    return torch.tensor(NF4_CODE if quant_type == "nf4" else FP4_CODE, dtype=torch.float32)


def _nearest_code(x: torch.Tensor, values: torch.Tensor) -> torch.Tensor:
    """Index into `values` of the entry nearest to x; at an exact midpoint the smaller entry (x must exceed a midpoint to move up)."""
    order = torch.argsort(values)
    v = values[order].double()
    mids = (v[1:] + v[:-1]) / 2  # exact in float64 for fp32 entries
    return order[torch.searchsorted(mids, x.double().contiguous(), right=False)]


def quantize_4bit(w: torch.Tensor, quant_type: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """Blockwise 4-bit quantization of a [out, in] weight (in % 64 == 0) -> (packed uint8 [out, in/2], absmax fp32 [out, in/64]).

    absmax is the block max of |fp32(w)|; each value is normalised as fp32(x) * fp32(1 / absmax) and coded as the nearest table
    entry, an exact midpoint going to the smaller entry.  FP4 codes |x| over codes 0..7 and sets the sign bit (code + 8) for
    x < 0.  An all-zero block has absmax 0 and dequantizes to zeros.

    This restates bitsandbytes' rule (`quantize_4bit`, blocksize 64) from its description; bitsandbytes is not a dependency, so
    the two have not been compared value for value.  Runs on w's device."""
    if w.dim() != 2 or not w.dtype.is_floating_point:
        raise ValueError("quantize_4bit expects a floating-point [out, in] weight")
    if w.shape[1] % BLOCKSIZE_4BIT:
        raise ValueError(f"quantize_4bit: in-features {w.shape[1]} are not a multiple of the blocksize {BLOCKSIZE_4BIT}")
    table = code_table(quant_type).to(w.device)
    n, k = w.shape
    blocks = w.float().reshape(-1, BLOCKSIZE_4BIT)
    absmax = blocks.abs().amax(dim=1)
    safe = torch.where(absmax > 0, absmax, torch.ones_like(absmax))
    inv = torch.where(absmax > 0, 1.0 / safe, torch.zeros_like(absmax))
    x = blocks * inv[:, None]
    if quant_type == "nf4":
        codes = _nearest_code(x, table)
    else:
        codes = _nearest_code(x.abs(), table[:8]) + torch.where(x < 0, 8, 0)
    codes = codes.reshape(n, k).to(torch.uint8)
    packed = (codes[:, 0::2] << 4) | codes[:, 1::2]
    return packed.contiguous(), absmax.reshape(n, k // BLOCKSIZE_4BIT).contiguous()


def unpack_4bit(packed: torch.Tensor) -> torch.Tensor:
    """[out, in/2] uint8 -> [out, in] codes (int64): element 2j from the high nibble of byte j, 2j + 1 from the low one."""
    p = packed.to(torch.int64)
    return torch.stack((p >> 4, p & 15), dim=2).reshape(p.shape[0], -1)


def dequantize_4bit(packed: torch.Tensor, absmax: torch.Tensor, quant_type: str, dtype: torch.dtype) -> torch.Tensor:
    """W' = dtype(code[q] * absmax): one fp32 product per element, then one round-to-nearest cast.  The values the 4-bit engine
    multiplies by."""
    table = code_table(quant_type).to(packed.device)
    vals = table[unpack_4bit(packed)]
    return (vals * absmax.float().repeat_interleave(BLOCKSIZE_4BIT, dim=1)).to(dtype)


def decompress_nested_absmax(absmax_u8: torch.Tensor, nested_absmax: torch.Tensor, nested_quant_map: torch.Tensor,
                             nested_blocksize: int, nested_offset: float) -> torch.Tensor:
    """Double-quantized absmax (bnb_4bit_use_double_quant) -> fp32: fp32(nested_quant_map[a] * nested_absmax[i // nested_blocksize])
    + nested_offset, two fp32 roundings, as bitsandbytes' dequantize_blockwise followed by `absmax += offset`."""
    a = absmax_u8.reshape(-1).to(torch.int64)
    scale = nested_absmax.float().repeat_interleave(int(nested_blocksize))[: a.numel()]
    out = nested_quant_map.float()[a] * scale
    return out + torch.tensor(float(nested_offset), dtype=torch.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# FP8 target weights (`quantization_config=FineGrainedFP8Config()`, or a checkpoint with `quant_method: "fp8"`)
#
# transformers' fine-grained FP8 stores a [out, in] weight as `weight` float8_e4m3fn plus `weight_scale_inv` fp32
# [out / 128, in / 128], one scale per 128 x 128 block.  The engine multiplies by
#
#     W' = dequantize_fp8_block(q, scale_inv, dtype) = dtype(fp32(q) * scale_inv[n // 128, k // 128])   (one product, one cast)
#
# which is transformers' own dequantization (Fp8Dequantize: `quantized.to(scales.dtype) * scales`, then the model-dtype cast),
# so an FP8 engine computes bit for bit what a bf16 / fp16 engine loaded with W' computes.  FP8Linear's W8A8 arithmetic
# (activations quantized per token group at run time, Triton / DeepGEMM kernels) is not reproduced: an FP8 engine's tokens are
# those of W' in the model dtype.
# ---------------------------------------------------------------------------------------------------------------------------
FP8_BLOCK = 128
FP8_MAX = 448.0  # torch.finfo(torch.float8_e4m3fn).max


def quantize_fp8_block(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Blockwise FP8 quantization of a [out, in] weight (both multiples of 128) -> (q float8_e4m3fn [out, in], scale_inv fp32
    [out / 128, in / 128]), restating transformers' Fp8Quantize.convert: per 128 x 128 block amax = max|fp32(w)|,
    scale = 448 / amax (1 for an all-zero block), q = fp8(clamp(fp32(w) * scale, +-448)), scale_inv = fp32(1 / scale).
    Runs on w's device."""
    if w.dim() != 2 or not w.dtype.is_floating_point:
        raise ValueError("quantize_fp8_block expects a floating-point [out, in] weight")
    n, k = w.shape
    if n % FP8_BLOCK or k % FP8_BLOCK:
        raise ValueError(f"quantize_fp8_block: shape [{n}, {k}] is not a multiple of the {FP8_BLOCK} x {FP8_BLOCK} block")
    q = torch.empty(n, k, dtype=torch.float8_e4m3fn, device=w.device)
    scale_inv = torch.empty(n // FP8_BLOCK, k // FP8_BLOCK, dtype=torch.float32, device=w.device)
    step = 8 * FP8_BLOCK  # rows per pass: the blocks are independent, and the fp32 temporaries of a 70B projection stay small
    for r in range(0, n, step):
        blocks = w[r: r + step].float().reshape(-1, FP8_BLOCK, k // FP8_BLOCK, FP8_BLOCK)
        amax = blocks.abs().amax(dim=(1, 3))
        scale = torch.where(amax > 0, FP8_MAX / torch.where(amax > 0, amax, torch.ones_like(amax)), torch.ones_like(amax))
        q[r: r + step] = torch.clamp(blocks * scale[:, None, :, None], min=-FP8_MAX, max=FP8_MAX).to(torch.float8_e4m3fn).reshape(-1, k)
        scale_inv[r // FP8_BLOCK: (r + step) // FP8_BLOCK] = (1.0 / scale).to(torch.float32)
    return q, scale_inv


def dequantize_fp8_block(q: torch.Tensor, scale_inv: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """W' = dtype(fp32(q) * scale_inv[n // 128, k // 128]): one fp32 product per element, then one round-to-nearest cast.  The
    values the FP8 engine multiplies by."""
    n, k = q.shape
    s = scale_inv.float().repeat_interleave(FP8_BLOCK, dim=0).repeat_interleave(FP8_BLOCK, dim=1)
    if s.shape != (n, k):
        raise ValueError(f"dequantize_fp8_block: scale_inv {tuple(scale_inv.shape)} does not tile [{n}, {k}] in {FP8_BLOCK} x {FP8_BLOCK} blocks")
    return (q.float() * s).to(dtype)

"""Float64 reference of the tree attention kernel (eagle_b200/csrc/attention.cu) and a per-element bound on how far the
kernel may legitimately differ from it.

The kernel computes, with the reference's rounding points (T = round to the model dtype, to nearest even):

    S1 = T(q . k)                       fp32 tensor-core accumulation over head_dim = 128
    S2 = T(fp32(S1) / fp32(sqrt(128)))  bit-identical to the IEEE fp32 division (tools/check_div.py)
    P  = T(softmax(S2))                 over the visible columns: the prefix [0, n_ctx) plus the tree columns whose ancestor
                                        bit is set; exp as ex2.approx, one row sum, __frcp_rn
    O  = T(P . V)                       fp32 tensor-core accumulation, then the fp32 sum of the cluster ranks' partials

This module evaluates the same chain in float64 with an explicit round-to-nearest-even (`rne`; torch's float64 -> bf16 /
fp16 casts round twice, via float32, and get exactly the ties wrong).  Where the kernel's fp32 arithmetic may land on the
other side of a rounding boundary, the reference carries both candidates:

* S1: the float64 dot product is within `qk_err * sum|q_i k_i|` of the kernel's fp32 sum.  If that window contains a
  rounding boundary of the model dtype, S1 (and so S2) may take either neighbouring value.
* P: softmax(S2) is bounded exactly over the S2 candidates (lower: own S2 low, every other S2 high; upper: the converse).
  The kernel's exponentials and row sum add a relative error `p_err` (below); P may take any dtype value that rounds from
  inside the widened interval.
* O: the interval of sum P_j V_j over the P candidates, plus `pv_err * sum P_j |V_j|` of fp32 accumulation.

The bound of an output element is then 1 ulp of O (the final rounding, plus slack for the accumulation that is not
spelled out above) + how far the P candidates move sum P V + the accumulation term.  Elements whose row has no ambiguous
S or P entry are held to 1 ulp.

Error constants (u = 2^-24, the fp32 unit roundoff):

* Tensor-core accumulation (mma.sync m16n8k16, fp32 accumulate): products of two bf16/fp16 values are exact; each MMA adds
  16 products and the accumulator with at most 2u of relative error per step on the magnitudes summed so far (the adder
  aligns to the largest addend and may truncate rather than round: 2u = one full fp32 ulp).  An addend passes through one
  MMA per 16 columns of the reduction after its own, hence err <= 2u * steps * sum|addends|:
    - QK: 128 / 16 = 8 steps                                -> qk_err = 16u
    - PV: 4 steps per 64-row KV tile a CTA sweeps (tiles_per) plus the kvs - 1 fp32 additions of the rank combine
                                                            -> pv_err = (8 * tiles_per + kvs) u
* exp: ex2.approx.ftz.f32 is within 2 ulp (2^-22 relative) of 2^x.  Its argument x = fma(s, log2e_f, -fp32(m * log2e_f))
  carries the rounding of log2e_f (<= u relative), of m * log2e_f (<= u) and of the fma (<= u |x|), so
  |dx| <= u (|s| log2e + 2 |m| log2e + |s - m| log2e), a relative error of ln2 |dx| <= u (|s| + 2|m| + |s - m|) in 2^x:
  e_exp(s) = 4u + u (2|s| + 3 M) with M = max |S2| of the row (|s - m| <= |s| + M).  The product e * inv adds u.
* Row sum: each lane adds 8 columns per 16-byte vector of the strip, at most ceil(tiles_per / 4) vectors, then a 5-level
  warp tree and the kvs partial sums: depth d = 8 ceil(tiles_per / 4) + 5 + kvs fp32 additions of positive terms, d u of
  relative error.  With a KV split every partial sum is rescaled by ex2((m_s - m) log2e): 4u + 3u * 2M, times u for the
  product.  __frcp_rn adds u.  The sum's error is common to the whole row: sum_err = max e_exp + rescale + (d + 1) u.
* p_err(s) = 1.05 (e_exp(s) + u + sum_err): 5 % covers the second-order terms of the first-order sum above.
* ftz: a probability below 2^-100 may come out as 0 (ex2.approx.ftz flushes subnormal results).
* The float64 reference itself: 2^-44 sum|q k| on S1, 2^-40 sum P|V| on O (float64 matmul, any device, any order).
"""
from __future__ import annotations

import ctypes as C
import math

import torch

U = 2.0 ** -24
# significand bits with the implicit one, smallest normal exponent, largest finite value
_FMT = {torch.bfloat16: (8, -126, float.fromhex("0x1.fep127")), torch.float16: (11, -14, 65504.0)}
_SQRT_D_F32 = float(torch.tensor(math.sqrt(128.0), dtype=torch.float32))  # fp32(sqrt(128)), as the kernel's constant


def ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of `dtype` values at |x| (float64; the spacing above x when x is a power of two)."""
    p, emin, _ = _FMT[dtype]
    x = x.to(torch.float64)
    _, e = torch.frexp(x)  # |x| in [2^(e-1), 2^e)
    q = torch.clamp(e - p, min=emin - p + 1)
    return torch.ldexp(torch.ones_like(x), q)


def rne(x: torch.Tensor, dtype) -> torch.Tensor:
    """float64 -> the nearest `dtype` value, ties to even, as float64.  One rounding (x / ulp is exact, torch.round rounds
    halves to even); overflow gives +-inf like an IEEE conversion."""
    _, _, fmax = _FMT[dtype]
    x = x.to(torch.float64)
    s = ulp(x, dtype)
    r = torch.round(x / s) * s
    return torch.where(r.abs() > fmax, torch.copysign(torch.full_like(r, math.inf), r), r)


def visible_mask(rows: int, n_ctx: int, n_tree: int, kv_len: int, masks, device=None) -> torch.Tensor:
    """[rows, kv_len] bool, the kernel's visible(): column c < n_ctx always, tree column j = c - n_ctx iff bit j of the row's
    128-bit ancestor mask (masks[r] = (word0, word1) as Python ints; None = causal, row r sees tree columns 0..r)."""
    vis = torch.zeros(rows, kv_len, dtype=torch.bool)
    vis[:, : min(n_ctx, kv_len)] = True
    for r in range(rows):
        if masks is None:
            bits = (1 << (r + 1)) - 1
        else:
            lo, hi = masks[r]
            bits = (int(lo) & (2 ** 64 - 1)) | ((int(hi) & (2 ** 64 - 1)) << 64)
        for j in range(min(n_tree, 128, kv_len - n_ctx)):
            if (bits >> j) & 1:
                vis[r, n_ctx + j] = True
    return vis.to(device) if device is not None else vis


def kernel_error_model(kv_len: int, kvs: int = 1, tiles_per: int | None = None) -> dict:
    """Accumulation-depth constants of the kernel's launch geometry (module docstring).  Default: one CTA sweeps every tile,
    the deepest chain any geometry has."""
    if tiles_per is None:
        tiles_per = max(1, -(-kv_len // 64))
    return dict(qk_err=16 * U, pv_err=(8 * tiles_per + kvs) * U, sum_depth=8 * (-(-tiles_per // 4)) + 5 + kvs, kvs=kvs)


def tree_attention_ref(q, kc, vc, n_ctx: int, n_tree: int, masks, dtype, kv_len: int | None = None, model: dict | None = None):
    """q [rows, nh, 128], kc / vc [nkv, >= kv_len, 128] (model dtype, any device).  Returns (o, bound, stats):
    o [rows, nh, 128] float64, the unrounded sum T(softmax(S2)) V; bound [rows, nh, 128] float64 on |kernel - o|; stats
    counts the ambiguous S1 / P entries (visible (row, head, column) triples), the output elements no ambiguous entry reaches
    (`clean`) and the median bound in ulps of O."""
    rows, nh, d = q.shape
    nkv = kc.shape[0]
    n_rep = nh // nkv
    kv_len = n_ctx + n_tree if kv_len is None else kv_len
    model = model or kernel_error_model(kv_len)
    dev = q.device
    vis = visible_mask(rows, n_ctx, n_tree, kv_len, masks, dev)  # [rows, kv]
    any_vis = vis.any(-1)
    o_all = torch.zeros(nh, rows, d, dtype=torch.float64, device=dev)
    b_all = torch.zeros_like(o_all)
    n_amb_s = n_amb_p = 0
    clean = torch.zeros(nh, rows, d, dtype=torch.bool, device=dev)
    for g in range(nkv):
        k64 = kc[g, :kv_len].to(torch.float64)
        v64 = vc[g, :kv_len].to(torch.float64)
        q64 = q[:, g * n_rep:(g + 1) * n_rep].to(torch.float64).transpose(0, 1)  # [n_rep, rows, d]
        s1x = q64 @ k64.T
        a = q64.abs() @ k64.abs().T
        w1 = model["qk_err"] * a + 2.0 ** -44 * a
        s1 = rne(s1x, dtype)
        s1lo, s1hi = rne(s1x - w1, dtype), rne(s1x + w1, dtype)

        def scale(x):
            return rne((x / _SQRT_D_F32).to(torch.float32).to(torch.float64), dtype)

        s2, s2lo, s2hi = scale(s1), scale(s1lo), scale(s1hi)
        n_amb_s += int(((s1lo != s1hi) & vis).sum())
        neg = torch.tensor(-math.inf, dtype=torch.float64, device=dev)
        s2m, lom, him = (torch.where(vis, x, neg) for x in (s2, s2lo, s2hi))
        m = him.amax(-1, keepdim=True)
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        e, elo, ehi = torch.exp(s2m - m), torch.exp(lom - m), torch.exp(him - m)
        z, zlo, zhi = e.sum(-1, keepdim=True), elo.sum(-1, keepdim=True), ehi.sum(-1, keepdim=True)
        one = torch.ones_like(z)
        z, zlo, zhi = (torch.where(x > 0, x, one) for x in (z, zlo, zhi))
        p = e / z
        plo = elo / (zhi - ehi + elo).clamp(min=1e-300)
        phi = ehi / (zlo - elo + ehi).clamp(min=1e-300)
        # kernel exponentials, row sum, reciprocal (module docstring)
        sabs = torch.where(vis, torch.maximum(s2lo.abs(), s2hi.abs()), torch.zeros_like(s2))
        big_m = sabs.amax(-1, keepdim=True)
        e_exp = 4 * U + U * (2 * sabs + 3 * big_m)
        sum_err = e_exp.amax(-1, keepdim=True) + (model["sum_depth"] + 1) * U
        if model["kvs"] > 1:
            sum_err = sum_err + 4 * U + 6 * U * big_m + U
        p_err = 1.05 * (e_exp + U + sum_err)
        lo_pre, hi_pre = plo * (1 - p_err), phi * (1 + p_err)
        p_t = rne(p, dtype)
        p_lo = torch.where(lo_pre < 2.0 ** -100, torch.zeros_like(lo_pre), rne(lo_pre, dtype))
        p_hi = rne(hi_pre, dtype)
        p_t, p_lo, p_hi = (torch.where(vis, x, torch.zeros_like(x)) for x in (p_t, p_lo, p_hi))
        n_amb_p += int((p_lo != p_hi).sum())
        vpos, vneg = v64.clamp(min=0), v64.clamp(max=0)
        o = p_t @ v64
        o_lo = p_lo @ vpos + p_hi @ vneg
        o_hi = p_hi @ vpos + p_lo @ vneg
        absw = p_hi @ v64.abs()
        acc = (model["pv_err"] + 2.0 ** -40) * absw
        spread = torch.maximum(o_hi - o, o - o_lo).clamp(min=0)
        bound = ulp(o.abs() + spread + acc, dtype) + spread + acc
        o_all[g * n_rep:(g + 1) * n_rep] = o
        b_all[g * n_rep:(g + 1) * n_rep] = bound
        clean[g * n_rep:(g + 1) * n_rep] = spread == 0
    o_all = o_all.transpose(0, 1).contiguous()
    b_all = b_all.transpose(0, 1).contiguous()
    # a row that sees no column: the kernel writes zeros (inverse row sum 0)
    b_all[~any_vis] = 0.0
    ulps = (b_all / ulp(o_all.abs(), dtype))[any_vis]
    stats = dict(amb_s=n_amb_s, amb_p=n_amb_p, clean=int(clean.transpose(0, 1)[any_vis].sum()), n=o_all.numel(),
                 median_ulps=float(ulps.median()) if ulps.numel() else 0.0)
    return o_all, b_all, stats


def check_against(got: torch.Tensor, o: torch.Tensor, bound: torch.Tensor, what: str = "") -> None:
    """Assert |got - o| <= bound elementwise (got: the kernel's [rows, nh, 128] in the model dtype)."""
    g = got.to(torch.float64).to(o.device)
    err = (g - o).abs()
    bad = ~(err <= bound)  # NaN counts as bad
    if bool(bad.any()):
        idx = bad.nonzero()
        i = tuple(idx[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())}/{bad.numel()} elements outside the rounding-aware bound; first at "
                             f"(row, head, dim) {idx[:6].tolist()}: got {float(g[i])!r} want {float(o[i])!r} "
                             f"bound {float(bound[i]):.3g}; worst err/bound {float((err / bound.clamp(min=1e-300)).max()):.3g}")


def attention_plan(lib, max_kv: int, n_heads: int, n_kv_heads: int, hpc_cap: int = 0, kvs_cap: int = 0):
    """eb200_k_attention_plan: ((hpc, kvs, kv_stride, smem), None), or (None, the library's message)."""
    hpc, kvs, stride, smem = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    rc = lib.eb200_k_attention_plan(max_kv, n_heads, n_kv_heads, hpc_cap, kvs_cap, C.byref(hpc), C.byref(kvs), C.byref(stride),
                                    C.byref(smem))
    if rc:
        return None, lib.eb200_last_error().decode()
    return (hpc.value, kvs.value, stride.value, smem.value), None

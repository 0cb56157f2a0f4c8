"""Parity of the persistent per-layer chain kernel (eagle_b200/csrc/mega.cu) on the H100, through the C ABI.

The kernel replaces, per decoder layer, modeling_llama_kv.py:801-863 (o_proj + residual, post-attention RMSNorm, SwiGLU MLP,
down_proj + residual, the next block's input RMSNorm and qkv projection with RoPE + KV append) and, after the last layer,
ea_model.py:190 + utils.py:362 (lm_head + arg-max).  Every stage is compared with the oracle's arithmetic (fp32 math, the
reference's rounding points) COMPUTED FROM THE KERNEL'S OWN PREVIOUS-STAGE OUTPUT, so each stage is held to the single-op
tolerance (1 ulp of the model dtype + 1e-3; integer outputs exact) instead of a compounded one.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import eagle_oracle as orc
from tests.test_kernels_gpu import DT, ULP, check, close, interleave64, lib, ptr  # noqa: F401  (lib is a fixture)

pytestmark = pytest.mark.gpu


def dev_randn(shape, g, scale, dtype):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


# ----------------------------------------------------------------------------------------------
# single GEMM through the chain kernel: stream-K partials + finish store, direct store, fused arg-max
# ----------------------------------------------------------------------------------------------
CHAIN_GEMM_CASES = [
    # M, N, K   (tiny problems leave most CTAs without a unit; odd tile counts; the benchmark's projection shapes)
    (1, 256, 256), (10, 512, 256), (60, 256, 2048), (64, 1024, 512), (7, 384, 768), (33, 200, 320),
    (60, 4096, 4096), (60, 6144, 4096), (60, 4096, 14336), (10, 32000, 4096), (10, 4096, 12288),
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", CHAIN_GEMM_CASES)
def test_chain_gemm_store(lib, M, N, K, dtype, mode):
    g = torch.Generator(device="cuda").manual_seed(M * 131 + N * 7 + K)
    X = dev_randn((64, K), g, 0.5, dtype)
    W = dev_randn((N, K), g, 0.05, dtype)
    bias = dev_randn((N,), g, 0.1, dtype)
    want = (X[:M].float() @ W.float().t() + bias.float()).to(dtype)
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    # three launches back to back: the phase counters reset themselves between launches
    check(lib, lib.eb200_k_chain_gemm(DT[dtype], mode, ptr(W), ptr(X), ptr(out), ptr(bias), None, M, N, K, 3, None))
    close(out[:M], want, dtype, f"chain gemm M={M} N={N} K={K} mode={mode}")
    if M < 64:
        assert float(out[M:].abs().max()) == 0.0  # rows beyond M are never written


@pytest.mark.parametrize("M,V,K", [(60, 128256, 4096), (1, 128256, 4096), (10, 1024, 256), (60, 32000, 4096)])
def test_chain_gemm_argmax_planted_winner_and_first_index_ties(lib, M, V, K):
    """Fused lm_head arg-max: every row has a planted clear winner; two rows have the winning weight row duplicated (once
    inside the same 128-row tile, once in a far-away tile): torch.argmax's first-index rule must hold across tiles and CTAs."""
    dtype = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(V + K + M)
    X = dev_randn((64, K), g, 0.5, dtype)
    W = dev_randn((V, K), g, 0.02, dtype)
    win = torch.randint(130, V - 130, (M,), generator=torch.Generator().manual_seed(5))
    win = torch.unique(win)[:M]
    while win.numel() < M:
        win = torch.unique(torch.cat([win, torch.randint(130, V - 130, (M,))]))[:M]
    win = win[torch.randperm(M, generator=torch.Generator().manual_seed(6))]
    for r in range(M):  # logit(r, win[r]) ~ 8 * |x_r|^2 / |x_r|^2-scaled: far above the N(0, ~0.6) background
        W[win[r]] = (X[r].float() * (6.0 / float(X[r].float().pow(2).sum()))).to(dtype)
    want = win.clone()
    if M >= 2:
        dup_same = int(win[0]) + 1 if (int(win[0]) % 128) < 127 else int(win[0]) - 1
        if dup_same not in win.tolist():
            W[dup_same] = W[win[0]]
            want[0] = min(int(win[0]), dup_same)
        far = (int(win[1]) + V // 2) % V
        if far not in win.tolist() and far != dup_same:
            W[far] = W[win[1]]
            want[1] = min(int(win[1]), far)
    out = torch.full((64,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    check(lib, lib.eb200_k_chain_gemm(DT[dtype], 2, ptr(W), ptr(X), None, None, ptr(out), M, V, K, 2, None))
    assert out[:M].cpu().tolist() == want.tolist()
    # and it agrees with arg-max over the materialised model-dtype logits wherever the top-2 margin exceeds one ulp
    logits = (X[:M].float() @ W.float().t()).to(dtype)
    assert torch.equal(logits.float().argmax(-1).cpu(), want)


# ----------------------------------------------------------------------------------------------
# the four-phase layer segment
# ----------------------------------------------------------------------------------------------
def rms_ref(x, w, eps):
    xf = x.float()
    return (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype).float()).to(x.dtype)


LAYER_CASES = [
    # M, H, I, heads, kv heads
    (10, 256, 512, 2, 1), (60, 256, 512, 2, 2), (60, 512, 1024, 4, 2), (7, 512, 1408, 4, 4),
    (60, 4096, 14336, 32, 8), (10, 4096, 14336, 32, 8), (60, 5120, 13824, 40, 40),
]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,H,I,nh,nkv", LAYER_CASES)
def test_chain_layer_segment_stage_by_stage(lib, M, H, I, nh, nkv, dtype):
    if dtype == torch.float16 and H > 512:
        pytest.skip("full-size shapes are checked in bf16 (the benchmark dtype); fp16 on the small ones")
    eps = 1e-5
    A = nh * 128
    g = torch.Generator(device="cuda").manual_seed(H + I + M)
    attn = dev_randn((64, A), g, 0.5, dtype)
    x0 = dev_randn((64, H), g, 1.0, dtype)
    Wo = dev_randn((H, A), g, 0.02, dtype)
    Wg = dev_randn((I, H), g, 0.03, dtype)
    Wu = dev_randn((I, H), g, 0.03, dtype)
    Wd = dev_randn((H, I), g, 0.02, dtype)
    Wqkv = dev_randn(((nh + 2 * nkv) * 128, H), g, 0.03, dtype)
    ln2 = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(dtype)
    ln1n = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(dtype)
    Wgu = interleave64(Wg, Wu)
    cap, kv_base = 256, 37
    pos = torch.randint(0, 200, (64,), generator=torch.Generator().manual_seed(1), dtype=torch.int32).cuda()
    cos, sin = orc.rope_table(128, 256, 500000.0)
    cosT, sinT = cos.to(dtype), sin.to(dtype)
    cos64, sin64 = cosT[:, :64].contiguous().cuda(), sinT[:, :64].contiguous().cuda()

    def run(n_phases):
        x = x0.clone()
        xn = torch.zeros(64, H, dtype=dtype, device="cuda")
        act = torch.zeros(64, I, dtype=dtype, device="cuda")
        tap = torch.zeros(64, H, dtype=dtype, device="cuda")
        q = torch.zeros(64, A, dtype=dtype, device="cuda")
        kc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
        vc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
        torch.cuda.synchronize()
        check(lib, lib.eb200_k_chain_layer(DT[dtype], M, H, I, nh, nkv, n_phases, ptr(Wo), ptr(Wgu), ptr(Wd), ptr(Wqkv), ptr(ln2), ptr(ln1n),
                                           ptr(attn), ptr(x), ptr(xn), ptr(act), ptr(tap), ptr(q), ptr(kc), ptr(vc), cap, ptr(cos64), ptr(sin64),
                                           ptr(pos), kv_base, eps, None))
        return x, xn, act, tap, q, kc, vc

    def norm_close(got, want, what):
        # w * T(x * rstd): rstd carries the fp32 summation order of sum(x^2), so T(x * rstd) may sit one ulp off before the second
        # rounding -> two ulps of the model dtype on a handful of elements
        got, want = got.float().cpu(), want.float().cpu()
        bad = (got - want).abs() > 1e-3 + 2 * ULP[dtype] * want.abs()
        one = (got - want).abs() > 1e-3 + ULP[dtype] * want.abs()
        assert not bool(bad.any()) and float(one.float().mean()) < 1e-3, f"{what}: {int(bad.sum())} beyond 2 ulp, {int(one.sum())} beyond 1 ulp of {bad.numel()}"

    # ---- phase 0: x1 = T(T(attn Wo^T) + x0), xn1 = ln2 * T(x1 * rstd)
    x1, xn1, _, _, _, _, _ = run(1)
    proj = F.linear(attn[:M].float(), Wo.float()).to(dtype)
    want = x0[:M] + proj
    err = (x1[:M].float() - want.float()).abs()
    tol = 1e-3 + ULP[dtype] * (proj.float().abs() + want.float().abs())
    assert bool((err <= tol).all()), f"o_proj+residual: {int((err > tol).sum())} bad, max err {float(err.max())}"
    assert torch.equal(x1[M:], x0[M:])
    norm_close(xn1[:M], rms_ref(x1[:M], ln2, eps), "post-attention RMSNorm of the kernel's own x")
    # ---- phase 1: act = T(T(silu(T(gate))) * T(up)) from the kernel's xn1
    _, xn1b, act, _, _, _, _ = run(2)
    assert torch.equal(xn1b, xn1), "the chain must be deterministic"
    gate = F.linear(xn1[:M].float(), Wg.float()).to(dtype)
    up = F.linear(xn1[:M].float(), Wu.float()).to(dtype)
    want = F.silu(gate) * up
    err = (act[:M].float() - want.float()).abs()
    tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
    assert bool((err <= tol).all()), f"swiglu: {int((err > tol).sum())} bad, max err {float(err.max())}"
    # ---- phase 2: x2 = T(T(act Wd^T) + x1), tap copy, xn2 = ln1' * norm(x2)
    x2, xn2, act_b, tap, _, _, _ = run(3)
    assert torch.equal(act_b, act)
    proj = F.linear(act[:M].float(), Wd.float()).to(dtype)
    want = x1[:M] + proj
    err = (x2[:M].float() - want.float()).abs()
    tol = 1e-3 + ULP[dtype] * (proj.float().abs() + want.float().abs())
    assert bool((err <= tol).all()), f"down_proj+residual: {int((err > tol).sum())} bad, max err {float(err.max())}"
    assert torch.equal(tap[:M], x2[:M]) and float(tap[M:].abs().max()) == 0.0
    norm_close(xn2[:M], rms_ref(x2[:M], ln1n, eps), "next input RMSNorm of the kernel's own x")
    # ---- phase 3: q / K / V rows from the kernel's xn2
    x2b, xn2b, _, _, q, kc, vc = run(4)
    assert torch.equal(x2b, x2) and torch.equal(xn2b, xn2)
    Wq, Wk, Wv = Wqkv[: nh * 128], Wqkv[nh * 128: (nh + nkv) * 128], Wqkv[(nh + nkv) * 128:]
    qf = F.linear(xn2[:M].float(), Wq.float()).to(dtype).view(1, M, nh, 128).transpose(1, 2).cpu()
    kf = F.linear(xn2[:M].float(), Wk.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2).cpu()
    vf = F.linear(xn2[:M].float(), Wv.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2).cpu()
    qr, kr = orc.apply_rope(qf, kf, cosT, sinT, pos[:M].cpu().long()[None])
    # RoPE combines two projections that may each sit one ulp off the fp32-order-of-summation reference before the rotation
    # (K = 4096 here): T(T(x cos) + T(rot sin)) is held to one ulp of each input pair member plus one ulp of the result
    def rope_close(got, want, pre, what):
        got, want, pre = got.float().cpu(), want.float().cpu(), pre.float().cpu()
        partner = torch.cat((pre[..., 64:], pre[..., :64]), dim=-1)
        tol = 1e-3 + ULP[dtype] * (pre.abs() + partner.abs() + want.abs())
        bad = (got - want).abs() > tol
        assert not bool(bad.any()), f"{what}: {int(bad.sum())}/{bad.numel()} beyond tolerance, max err {float((got - want).abs().max()):.4g}"

    rope_close(q[:M].view(M, nh, 128).transpose(0, 1), qr[0], qf[0], "q rope")
    rope_close(kc[:, kv_base:kv_base + M], kr[0], kf[0], "k rope/cache")
    close(vc[:, kv_base:kv_base + M], vf[0], dtype, "v cache")
    assert float(kc[:, :kv_base].abs().max()) == 0 and float(kc[:, kv_base + M:].abs().max()) == 0

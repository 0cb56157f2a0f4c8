"""Per-kernel parity on the H100: every CUDA kernel is called in isolation through the C ABI
(eb200_k_* entry points) and compared with the CPU oracle's arithmetic on the same seeded inputs.

Tolerances (written here, per the north star): integer/index outputs are bit-exact; floating-point
outputs are compared after the model-dtype rounding the reference also performs, allowing 1 ulp of the
model dtype (bf16: 2^-7 relative, fp16: 2^-10) plus 1e-3 absolute -- the kernels accumulate in fp32
like the reference, so what differs is summation order only.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import eagle_oracle as orc

pytestmark = pytest.mark.gpu

DT = {torch.bfloat16: 0, torch.float16: 1}
ULP = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}  # spacing of the model dtype relative to the binade


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def close(got, want, dtype, what=""):
    got, want = got.float().cpu(), want.float().cpu()
    tol = 1e-3 + ULP[dtype] * want.abs()
    bad = (got - want).abs() > tol
    if bad.any():
        idx = bad.nonzero()
        msg = (f"{what}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; max abs err "
               f"{float((got - want).abs().max()):.5g}; first bad {idx[:8].tolist()}; "
               f"got {got[bad][:8].tolist()} want {want[bad][:8].tolist()}")
        raise AssertionError(msg)


_KEEP = []


def ptr(t):
    """Raw pointer of a tensor; the tensor is kept alive (temporaries such as `x.cuda()` would otherwise be
    freed -- and their block reused by the next allocation -- before the kernel reads them)."""
    if t is None:
        return None
    _KEEP.append(t)
    if len(_KEEP) > 64:
        del _KEEP[:-64]
    return C.c_void_p(t.data_ptr())


# ----------------------------------------------------------------------------------------------
# skinny GEMM (wgmma + TMA) and its epilogues
# ----------------------------------------------------------------------------------------------
GEMM_CASES = [
    # M, N, K, splitk
    (1, 256, 256, 1), (10, 512, 256, 1), (16, 256, 512, 2), (60, 256, 256, 1), (64, 1024, 512, 1),
    (60, 512, 1024, 4), (7, 384, 768, 3), (60, 4096, 4096, 4), (33, 200, 320, 1), (10, 1000, 4096, 8),
]


# kernel selector of the eb200_k_gemm* test entry points: 0 = engine default (persistent stream-K), 1 = SIMT bring-up
# kernel, 2 = cluster split-K kernel
MODES = [0, 1, 2]


@pytest.mark.parametrize("simt", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,splitk", GEMM_CASES)
def test_gemm_store(lib, M, N, K, splitk, dtype, simt):
    if simt == 1 and N * K > 1 << 21:
        pytest.skip("SIMT bring-up kernel only on small shapes")
    g = torch.Generator().manual_seed(M * 131 + N * 7 + K)
    X = (torch.randn(64, K, generator=g) * 0.5).to(dtype)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
    bias = (torch.randn(N, generator=g) * 0.1).to(dtype)
    want = (X[:M].float() @ W.float().t() + bias.float()).to(dtype)
    Xd, Wd, bd = X.cuda(), W.cuda(), bias.cuda()
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_gemm(DT[dtype], simt, 0, ptr(Wd), None, ptr(Xd), ptr(out), None, ptr(bd), M, N, K, splitk, None))
    close(out[:M], want, dtype, f"gemm_store M={M} N={N} K={K} splitk={splitk} simt={simt}")
    if M < 64:
        assert float(out[M:].abs().max()) == 0.0  # rows beyond M are never written


@pytest.mark.parametrize("M,N,K,splitk,epi", [
    (60, 6144, 4096, 4, "qkv"), (60, 4096, 4096, 8, "res"), (60, 14336, 4096, 2, "swiglu"), (60, 4096, 14336, 8, "res"),
    (60, 128256, 4096, 1, "store"), (10, 32000, 4096, 1, "store"), (10, 6144, 8192, 4, "store"), (8, 4096, 12288, 8, "store"),
])
@pytest.mark.parametrize("mode", [0, 2])
def test_gemm_llama3_8b_shapes(lib, M, N, K, splitk, epi, mode):
    """The projections of the benchmark configuration (BASELINE.json configs[1..2]) at full size, checked against a
    float64 reference on sampled output columns (size-independent property: linearity in W rows)."""
    dtype = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(N + K)
    X = (torch.randn(64, K, generator=g, device="cuda") * 0.5).to(dtype)
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
    cols = torch.randint(0, N, (512,), generator=torch.Generator().manual_seed(3)).cuda()
    torch.cuda.synchronize()
    if epi == "swiglu":
        W2 = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
        torch.cuda.synchronize()
        out = torch.zeros(64, N, dtype=dtype, device="cuda")
        check(lib, lib.eb200_k_gemm(0, mode, 2, ptr(W), ptr(W2), ptr(X), ptr(out), None, None, M, N, K, splitk, None))
        gate = (X[:M].double() @ W[cols].double().t()).to(dtype)
        up = (X[:M].double() @ W2[cols].double().t()).to(dtype)
        want = F.silu(gate) * up
        err = (out[:M][:, cols].float() - want.float()).abs()
        tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
        assert bool((err <= tol).all()), f"max err {float(err.max())}"
        return
    res = torch.randn(64, N, generator=g, device="cuda").to(dtype) if epi == "res" else None
    torch.cuda.synchronize()
    out = res.clone() if res is not None else torch.zeros(64, N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    code = 1 if epi == "res" else 0
    check(lib, lib.eb200_k_gemm(0, mode, code, ptr(W), None, ptr(X), ptr(out), ptr(out) if res is not None else None, None, M, N, K, splitk, None))
    proj = (X[:M].double() @ W[cols].double().t()).to(dtype)
    want = (res[:M][:, cols] + proj) if res is not None else proj
    err = (out[:M][:, cols].float() - want.float()).abs()
    tol = 1e-3 + ULP[dtype] * (proj.float().abs() + want.float().abs())
    assert bool((err <= tol).all()), f"{epi}: {int((err > tol).sum())} bad, max err {float(err.max())}"


def interleave64(Wg, Wu):
    """The engine's gate/up layout (EPI_SWIGLU_IL): 128-row tiles of 64 gate rows followed by the 64 up rows of the same outputs."""
    N, K = Wg.shape
    assert N % 64 == 0
    return torch.stack((Wg.view(N // 64, 64, K), Wu.view(N // 64, 64, K)), dim=1).reshape(2 * N, K).contiguous()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,splitk", [(10, 512, 256, 1), (60, 1024, 256, 2), (60, 1408, 512, 1), (60, 1792, 4096, 4), (7, 64, 256, 1)])
def test_gemm_swiglu_interleaved(lib, M, N, K, splitk, dtype, mode):
    """Single-accumulator SwiGLU over interleaved gate/up rows: same rounding points as the two-matrix kernel, so the two
    must agree BIT FOR BIT (same fp32 accumulation order per element), and both sit within tolerance of the torch reference."""
    g = torch.Generator().manual_seed(12 + N)
    X = (torch.randn(64, K, generator=g)).to(dtype)
    Wg = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    Wu = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    gate = F.linear(X[:M].float(), Wg.float()).to(dtype)
    up = F.linear(X[:M].float(), Wu.float()).to(dtype)
    want = F.silu(gate) * up
    Wil = interleave64(Wg, Wu).cuda()
    Xd = X.cuda()
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    check(lib, lib.eb200_k_gemm(DT[dtype], mode, 5, ptr(Wil), None, ptr(Xd), ptr(out), None, None, M, N, K, splitk, None))
    err = (out[:M].float().cpu() - want.float()).abs()
    tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
    assert bool((err <= tol).all()), f"gemm_swiglu_il: {int((err > tol).sum())} bad, max err {float(err.max())}"
    if M < 64:
        assert float(out[M:].abs().max()) == 0.0
    if mode != 1 and N % 128 == 0:
        out2 = torch.zeros(64, N, dtype=dtype, device="cuda")
        Wgd, Wud = Wg.cuda(), Wu.cuda()
        torch.cuda.synchronize()
        check(lib, lib.eb200_k_gemm(DT[dtype], mode, 2, ptr(Wgd), ptr(Wud), ptr(Xd), ptr(out2), None, None, M, N, K, splitk, None))
        assert torch.equal(out, out2), "interleaved and two-matrix SwiGLU kernels disagree"


@pytest.mark.parametrize("mode", [0, 2])
def test_gemm_swiglu_interleaved_llama3_shape(lib, mode):
    """gate_up of Llama-3-8B at full size (N = 14336, K = 4096, 224 interleaved tiles), sampled columns vs float64."""
    dtype = torch.bfloat16
    M, N, K = 60, 14336, 4096
    g = torch.Generator(device="cuda").manual_seed(N + K + 1)
    X = (torch.randn(64, K, generator=g, device="cuda") * 0.5).to(dtype)
    Wg = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
    Wu = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
    Wil = interleave64(Wg, Wu)
    cols = torch.randint(0, N, (512,), generator=torch.Generator().manual_seed(3)).cuda()
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    check(lib, lib.eb200_k_gemm(0, mode, 5, ptr(Wil), None, ptr(X), ptr(out), None, None, M, N, K, 1, None))
    gate = (X[:M].double() @ Wg[cols].double().t()).to(dtype)
    up = (X[:M].double() @ Wu[cols].double().t()).to(dtype)
    want = F.silu(gate) * up
    err = (out[:M][:, cols].float() - want.float()).abs()
    tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
    assert bool((err <= tol).all()), f"max err {float(err.max())}"
    assert float(out[M:].abs().max()) == 0.0


@pytest.mark.parametrize("simt", MODES)
def test_gemm_onehot_layout(lib, simt):
    """X rows are one-hot: out[m, n] must equal W[n, k_m] exactly -- isolates descriptor / swizzle bugs."""
    dtype = torch.bfloat16
    M, N, K = 16, 256, 256
    W = torch.arange(N * K, dtype=torch.float32).reshape(N, K).remainder(251).sub(125).div(64).to(dtype)
    X = torch.zeros(64, K, dtype=dtype)
    ks = [(m * 37 + 5) % K for m in range(M)]
    for m, k in enumerate(ks):
        X[m, k] = 1.0
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_gemm(0, simt, 0, ptr(W.cuda()), None, ptr(X.cuda()), ptr(out), None, None, M, N, K, 1, None))
    want = torch.stack([W[:, k] for k in ks])
    got = out[:M].cpu()
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        raise AssertionError(f"layout mismatch at {bad[:10].tolist()} got {got[got != want][:10].tolist()} want {want[got != want][:10].tolist()}")


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,splitk", [(10, 256, 512, 1), (60, 512, 256, 2), (60, 4096, 1024, 4)])
def test_gemm_residual(lib, M, N, K, splitk, dtype, mode):
    g = torch.Generator().manual_seed(11)
    X = (torch.randn(64, K, generator=g) * 0.5).to(dtype)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
    res = torch.randn(64, N, generator=g).to(dtype)
    proj = F.linear(X[:M].float(), W.float()).to(dtype)
    want = res[:M] + proj  # x + o_proj(a): two roundings
    out = res.clone().cuda()
    check(lib, lib.eb200_k_gemm(DT[dtype], mode, 1, ptr(W.cuda()), None, ptr(X.cuda()), ptr(out), ptr(out), None, M, N, K, splitk, None))
    # 1 ulp of the projection (it may flip before the add) + 1 ulp of the sum
    err = (out[:M].float().cpu() - want.float()).abs()
    tol = 1e-3 + ULP[dtype] * (proj.float().abs() + want.float().abs())
    assert bool((err <= tol).all()), f"gemm_residual: {int((err > tol).sum())} bad, max err {float(err.max())}"
    assert torch.equal(out[M:].cpu(), res[M:])


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K,splitk", [(10, 512, 256, 1), (60, 1024, 256, 2), (60, 1408, 512, 1)])
def test_gemm_swiglu(lib, M, N, K, splitk, dtype, mode):
    g = torch.Generator().manual_seed(12)
    X = (torch.randn(64, K, generator=g)).to(dtype)
    Wg = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    Wu = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    gate = F.linear(X[:M].float(), Wg.float()).to(dtype)
    up = F.linear(X[:M].float(), Wu.float()).to(dtype)
    want = F.silu(gate) * up
    out = torch.zeros(64, N, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_gemm(DT[dtype], mode, 2, ptr(Wg.cuda()), ptr(Wu.cuda()), ptr(X.cuda()), ptr(out), None, None, M, N, K, splitk, None))
    # gate and up may each flip by 1 ulp before silu/mul (silu' <= 1.1), plus the final rounding: 3.2 ulp of the product
    err = (out[:M].float().cpu() - want.float()).abs()
    tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
    assert bool((err <= tol).all()), f"gemm_swiglu: {int((err > tol).sum())} bad, max err {float(err.max())}"


@pytest.mark.parametrize("simt", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,nh,nkv,K,splitk", [(10, 2, 1, 256, 1), (60, 4, 2, 512, 2), (7, 2, 2, 512, 1)])
def test_qkv_rope_kv_append(lib, M, nh, nkv, K, splitk, dtype, simt):
    g = torch.Generator().manual_seed(13)
    X = torch.randn(64, K, generator=g).to(dtype)
    Wq = (torch.randn(nh * 128, K, generator=g) * 0.06).to(dtype)
    Wk = (torch.randn(nkv * 128, K, generator=g) * 0.06).to(dtype)
    Wv = (torch.randn(nkv * 128, K, generator=g) * 0.06).to(dtype)
    cap, kv_base = 256, 37
    pos = torch.randint(0, 200, (64,), generator=g, dtype=torch.int32)
    cos, sin = orc.rope_table(128, 256, 500000.0)
    cosT, sinT = cos.to(dtype), sin.to(dtype)
    q = F.linear(X[:M].float(), Wq.float()).to(dtype).view(1, M, nh, 128).transpose(1, 2)
    k = F.linear(X[:M].float(), Wk.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2)
    v = F.linear(X[:M].float(), Wv.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2)
    qr, kr = orc.apply_rope(q, k, cosT, sinT, pos[:M].long()[None])
    Wqkv = torch.cat([Wq, Wk, Wv]).cuda()
    q_out = torch.zeros(64, nh * 128, dtype=dtype, device="cuda")
    kc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
    vc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_qkv_rope(DT[dtype], simt, ptr(Wqkv), ptr(X.cuda()), ptr(q_out), ptr(kc), ptr(vc),
                                    ptr(cosT[:, :64].contiguous().cuda()), ptr(sinT[:, :64].contiguous().cuda()),
                                    ptr(pos.cuda()), M, nh, nkv, K, cap, kv_base, splitk, None))
    close(q_out[:M].view(M, nh, 128).transpose(0, 1), qr[0], dtype, "q rope")
    close(kc[:, kv_base:kv_base + M], kr[0], dtype, "k rope/cache")
    close(vc[:, kv_base:kv_base + M], v[0], dtype, "v cache")
    assert float(kc[:, :kv_base].abs().max()) == 0 and float(kc[:, kv_base + M:].abs().max()) == 0


# ----------------------------------------------------------------------------------------------
# RMSNorm / argmax / log-softmax top-k
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("rows,H", [(1, 256), (60, 4096), (10, 8192)])
def test_rmsnorm(lib, rows, H, dtype):
    g = torch.Generator().manual_seed(14)
    x = (torch.randn(rows, H, generator=g) * 3).to(dtype)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype)
    want = orc.rms_norm(x, w, 1e-5)
    y = torch.zeros_like(x, device="cuda")
    check(lib, lib.eb200_k_rmsnorm(DT[dtype], ptr(x.cuda()), ptr(w.cuda()), ptr(y), rows, H, 1e-5, None))
    close(y, want, dtype, "rmsnorm")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("rows,V", [(1, 1024), (60, 128256), (5, 32000)])
def test_argmax_first_max(lib, rows, V, dtype):
    g = torch.Generator().manual_seed(15)
    x = torch.randn(rows, V, generator=g).to(dtype)
    x[0, 7] = x[0].max()  # force a tie: the first index must win
    x[0, 3] = x[0, 7]
    out = torch.zeros(rows, dtype=torch.int32, device="cuda")
    check(lib, lib.eb200_k_argmax(DT[dtype], ptr(x.cuda()), rows, V, ptr(out), None))
    assert out.cpu().tolist() == torch.argmax(x.float(), dim=-1).tolist()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("rows,V,k", [(1, 512, 10), (10, 32000, 10), (8, 1024, 8), (2, 128256, 10)])
def test_logsoftmax_topk(lib, rows, V, k, dtype):
    g = torch.Generator().manual_seed(16)
    x = (torch.randn(rows, V, generator=g) * 2).to(dtype)
    logp = F.log_softmax(x, dim=-1)  # model-dtype tensor in, model-dtype tensor out (cnets.py:702)
    tp = torch.zeros(rows, k, dtype=torch.float32, device="cuda")
    ti = torch.zeros(rows, k, dtype=torch.int32, device="cuda")
    check(lib, lib.eb200_k_logsoftmax_topk(DT[dtype], ptr(x.cuda()), rows, V, k, ptr(tp), ptr(ti), None))
    tp, ti = tp.cpu(), ti.cpu().long()
    # deterministic reference order: value desc, index asc (torch.topk leaves tie order unspecified)
    for r in range(rows):
        order = sorted(range(V), key=lambda i: (-float(logp[r, i]), i))[:k]
        want_v = logp[r, order].float()
        got_v = tp[r]
        # the selected values must be the k best values (1-ulp slack on the log-sum-exp rounding)
        close(got_v, want_v, dtype, f"topk values row {r}")
        # and the indices must carry exactly those values
        close(logp[r, ti[r]].float(), got_v, dtype, f"topk indices row {r}")
        assert len(set(ti[r].tolist())) == k


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
def _oracle_attention(q, kc, vc, n_ctx, n_tree, mask_bits, dtype):
    """q [rows, nh, 128]; kc/vc [nkv, cap, 128].  Dense fp32 mask like the reference, then eager attention."""
    rows, nh, _ = q.shape
    nkv = kc.shape[0]
    kv_len = n_ctx + n_tree
    m = torch.zeros(rows, kv_len)
    for r in range(rows):
        for j in range(n_tree):
            if not (mask_bits[r][j // 64] >> (j % 64)) & 1:
                m[r, n_ctx + j] = torch.finfo(torch.float32).min
    qq = q.transpose(0, 1)[None]
    out = orc.eager_attention(qq, kc[None, :, :kv_len], vc[None, :, :kv_len], m[None, None], nh // nkv)
    return out[0].transpose(0, 1)  # [rows, nh, 128]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("rows,nh,nkv,n_ctx,n_tree,causal", [
    (10, 2, 1, 37, 10, False), (60, 4, 2, 100, 60, False), (60, 8, 2, 700, 60, False), (64, 2, 2, 128, 64, True),
    (1, 2, 1, 50, 1, True), (10, 4, 4, 300, 60, False), (33, 2, 1, 0, 33, True), (10, 2, 1, 515, 70, False),
])
def test_tree_attention(lib, rows, nh, nkv, n_ctx, n_tree, causal, dtype):
    g = torch.Generator().manual_seed(rows * 7 + n_ctx)
    cap = n_ctx + n_tree + 5
    q = torch.randn(rows, nh, 128, generator=g).to(dtype)
    kc = torch.randn(nkv, cap, 128, generator=g).to(dtype)
    vc = torch.randn(nkv, cap, 128, generator=g).to(dtype)
    bits = []
    for r in range(rows):
        if causal:
            b = (1 << (r + 1)) - 1
        else:
            b = int(torch.randint(0, 2 ** 30, (1,), generator=g)) | (int(torch.randint(0, 2 ** 30, (1,), generator=g)) << 30) \
                | (int(torch.randint(0, 2 ** 10, (1,), generator=g)) << 60)
            b |= 1  # the root column is always visible (tree_mask[:, 0] = True, cnets.py:777)
            b &= (1 << n_tree) - 1
        bits.append((b & (2 ** 64 - 1), b >> 64))
    want = _oracle_attention(q, kc, vc, n_ctx, n_tree, bits, dtype)
    mask = None
    if not causal:
        flat = []
        for lo, hi in bits:
            flat += [lo - (1 << 64) if lo >= (1 << 63) else lo, hi]
        mask = torch.tensor(flat, dtype=torch.int64).cuda()
    out = torch.zeros(rows, nh * 128, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_attention(DT[dtype], ptr(q.reshape(rows, nh * 128).cuda()), ptr(kc.cuda()), ptr(vc.cuda()), ptr(out),
                                     rows, nh, nkv, cap, n_ctx, n_tree, ptr(mask), None))
    # P is rounded to the model dtype before PV: allow 2 ulp on the output
    got, w = out.view(rows, nh, 128).float().cpu(), want.float()
    tol = 2e-3 + 2 * ULP[dtype] * w.abs().clamp(min=0.1)
    bad = (got - w).abs() > tol
    assert not bad.any(), f"{int(bad.sum())}/{bad.numel()} bad; max err {float((got - w).abs().max())}; first {bad.nonzero()[:5].tolist()}"


# ----------------------------------------------------------------------------------------------
# integer kernels: tree build, greedy accept (bit-exact)
# ----------------------------------------------------------------------------------------------
def _random_pool(k, depth, seed, dtype):
    """A consistent candidate pool: level-major cumulative log-prob scores, tokens, parents (Appendix A)."""
    g = torch.Generator().manual_seed(seed)
    scores = [F.log_softmax(torch.randn(k, generator=g) * 2, -1).to(dtype)]
    front = scores[0].clone()
    parents = [torch.zeros(1, dtype=torch.long)]
    cs_index = torch.arange(k)
    for i in range(depth):
        bias = 1 + k * k * max(0, i - 1) + (k if i > 0 else 0)
        parents.append(cs_index + bias)
        p = F.log_softmax(torch.randn(k, k, generator=g) * 2, -1).to(dtype)
        cu = p + front[:, None]
        # perturb to avoid exact ties (tie policy is tested separately)
        scores.append(cu)
        top = torch.topk(cu.view(-1), k)
        cs_index, front = top.indices, top.values
    s = torch.cat([x.reshape(-1) for x in scores]).float()
    tokens = torch.randint(0, 32000, (s.numel(),), generator=g)
    return s, tokens, torch.cat(parents)


@pytest.mark.parametrize("k,depth,total,seed", [(10, 6, 60, 1), (10, 6, 60, 2), (10, 7, 60, 3), (8, 4, 40, 4), (10, 5, 26, 5),
                                                (4, 3, 30, 6), (10, 6, 64, 7), (16, 2, 60, 8)])
@pytest.mark.parametrize("sort_rows", [0, 1])
def test_tree_finalize_matches_oracle(lib, k, depth, total, seed, sort_rows):
    scores, tokens, parents = _random_pool(k, depth, seed, torch.float32)
    # make scores unique so torch.topk's unspecified tie order cannot matter
    scores = scores + torch.arange(scores.numel()) * 1e-7
    want = orc.finalize_tree(scores, tokens, parents, torch.tensor([777]), k, total - 1, bool(sort_rows))
    T = total
    dt = torch.zeros(T, dtype=torch.int64)
    tm = torch.zeros(T * T, dtype=torch.float32)
    tp = torch.zeros(T, dtype=torch.int64)
    ri = torch.full((T * 16,), -1, dtype=torch.int64)
    nl, md = C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_tree_finalize(0, ptr(scores.contiguous()), ptr(tokens.int().contiguous()), ptr(parents.int().contiguous()),
                                         k, depth, total, 777, sort_rows, ptr(dt), ptr(tm), ptr(tp), ptr(ri), C.byref(nl), C.byref(md)))
    w_tokens, w_retrieve, w_mask, w_pos = want
    assert torch.equal(dt[None], w_tokens)
    assert torch.equal(tm.view(1, 1, T, T), w_mask)
    assert torch.equal(tp, w_pos)
    assert (nl.value, md.value) == tuple(w_retrieve.shape)
    assert torch.equal(ri[: nl.value * md.value].view(nl.value, md.value), w_retrieve)


def test_tree_finalize_tie_policy(lib):
    """Equal scores: lowest flat index wins, so a parent is always kept before its equal-score child."""
    k, depth, total = 4, 2, 8
    n = k + depth * k * k
    scores = torch.full((n,), -5.0)
    scores[:k] = torch.tensor([-1.0, -1.0, -2.0, -2.0])
    scores[k:k + 4] = -1.0  # children of frontier slot 0 tie with their parent
    parents = torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 8], dtype=torch.int32)
    tokens = torch.arange(n, dtype=torch.int32)
    T = total
    dt = torch.zeros(T, dtype=torch.int64)
    tp = torch.zeros(T, dtype=torch.int64)
    nl, md = C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_tree_finalize(0, ptr(scores), ptr(tokens), ptr(parents), k, depth, total, 9, 0, ptr(dt), None, ptr(tp),
                                         None, C.byref(nl), C.byref(md)))
    # top-7 by (value desc, index asc): flat {0,1,4,5,6,7} at -1.0, then flat 2 at -2.0; tokens == flat indices
    assert dt.tolist() == [9, 0, 1, 2, 4, 5, 6, 7]
    assert tp.tolist() == [0, 1, 1, 1, 2, 2, 2, 2]


@pytest.mark.parametrize("seed", range(6))
def test_greedy_accept_matches_oracle(lib, seed):
    g = torch.Generator().manual_seed(100 + seed)
    k, depth, total = 10, 6, 60
    scores, tokens, parents = _random_pool(k, depth, seed, torch.float32)
    scores = scores + torch.arange(scores.numel()) * 1e-7
    tokens = torch.randint(0, 50, (scores.numel(),), generator=g)  # small vocab so matches happen
    draft_tokens, retrieve, _, _ = orc.finalize_tree(scores, tokens, parents, torch.tensor([3]), k, total - 1, False)
    V = 50
    logits_nodes = torch.randn(total, V, generator=g)
    # plant a partially correct path
    path = retrieve[seed % retrieve.shape[0]]
    for j in range(1, min(len(path), 2 + seed)):
        if path[j] >= 0:
            logits_nodes[path[j - 1], draft_tokens[0, path[j]]] = 50.0
    logits = logits_nodes[retrieve]
    cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
    w_best, w_acc, w_p = orc.evaluate_posterior_greedy(logits, cands)
    node_argmax = torch.argmax(logits_nodes, dim=-1).int()
    best, acc, bonus = C.c_int32(), C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_greedy_accept(ptr(node_argmax), ptr(draft_tokens[0].int().contiguous()), ptr(retrieve.int().contiguous()),
                                         total, retrieve.shape[0], retrieve.shape[1], C.byref(best), C.byref(acc), C.byref(bonus)))
    assert (best.value, acc.value) == (int(w_best), int(w_acc))
    assert bonus.value == int(torch.argmax(w_p))


# ----------------------------------------------------------------------------------------------
# sampling posterior (utils.py:375-415) with injected uniforms
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("temperature,top_p,top_k", [(1.0, 0.0, 0), (0.7, 0.0, 0), (1.0, 0.9, 0), (1.3, 0.0, 20), (0.8, 0.95, 50)])
def test_sample_posterior_matches_oracle(lib, seed, temperature, top_p, top_k):
    g = torch.Generator().manual_seed(200 + seed)
    k, depth, total, V = 10, 6, 60, 512
    scores, tokens, parents = _random_pool(k, depth, seed, torch.float32)
    scores = scores + torch.arange(scores.numel()) * 1e-7
    tokens = torch.randint(0, 40, (scores.numel(),), generator=g)  # small token range so candidates get real probability
    draft_tokens, retrieve, _, _ = orc.finalize_tree(scores, tokens, parents, torch.tensor([3]), k, total - 1, True)
    logits_nodes = (torch.randn(total, V, generator=g) * 1.5).to(torch.bfloat16)
    logits_nodes[:, :40] += 4.0  # the draft's token range is likely under the target too
    uniforms = torch.rand(64, generator=g)
    it = iter(uniforms.tolist())
    # oracle in fp32 on the same (model-dtype-valued) logits; the engine keeps probabilities in fp32 too
    warp = lambda lg: orc.warp_logits(lg, temperature, top_p, top_k)  # noqa: E731
    lg32 = logits_nodes.float()
    if temperature != 1.0:  # TemperatureLogitsWarper divides in the model dtype
        lg32 = (logits_nodes / temperature).float()
        warp = lambda lg: orc.warp_logits(lg, 1.0, top_p, top_k)  # noqa: E731
    cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
    w_best, w_acc, w_p = orc.evaluate_posterior_sampling(lg32[retrieve], cands, warp, rand=lambda: next(it))
    u_bonus = next(it)
    cdf = torch.cumsum(w_p.double(), 0)
    w_bonus = int(torch.searchsorted(cdf, torch.tensor(u_bonus * float(cdf[-1]), dtype=torch.float64)))
    best, acc, bonus, used = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_sample_posterior(0, ptr(logits_nodes.cuda()), V, ptr(draft_tokens[0].int().contiguous()),
                                            ptr(retrieve.int().contiguous()), total, retrieve.shape[0], retrieve.shape[1], temperature, top_p,
                                            top_k, ptr(uniforms.contiguous()), 64, C.byref(best), C.byref(acc), C.byref(bonus), C.byref(used)))
    assert (best.value, acc.value) == (int(w_best), int(w_acc))
    assert bonus.value == w_bonus or abs(float(cdf[bonus.value]) - u_bonus * float(cdf[-1])) < 1e-4

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


def close_rope(got, x, cos, sin, pos, want, dtype, what=""):
    """RoPE outputs T(T(x c) + T(rotate_half(x) s)) of the rounded projection x [heads, M, 128] at positions pos: 1e-3 plus one
    ulp of the output plus two of each product.  The kernel rounds the same products as the reference, but a one-ulp flip of x
    (or of its rotation partner) moves a product by an ulp of it, and where the two products cancel that is many ulps of the
    output (long K sums and large angles make such flips and cancellations common)."""
    c, s, x = cos[pos].float(), sin[pos].float(), x.float()
    terms = (x * c).abs() + (orc._rotate_half(x) * s).abs()
    got, want = got.float().cpu(), want.float().cpu()
    bad = (got - want).abs() > 1e-3 + ULP[dtype] * (want.abs() + 2 * terms)
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; first bad {bad.nonzero()[:8].tolist()}; "
                           f"got {got[bad][:8].tolist()} want {want[bad][:8].tolist()}")


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


# kernel selector of the eb200_k_gemm* test entry points: 0 and 2 = cluster split-K kernel (the engine's), 1 = SIMT
# bring-up kernel
MODES = [0, 1, 2]


def x_rows(M):
    """Rows of the activation buffer the test entry points read for M rows: 64, or 256 for the prompt prefill's launch."""
    return 256 if M > 64 else 64


# Above 64 rows the kernel runs the prompt prefill's 256-row instantiation (wgmma N = 256): 65 is its smallest launch; with
# splitk 3 each CTA reduces 86 rows, so a CTA's last 16-row chunk is partial; at M = 100 and splitk 8 ranks 4..7 own no valid row.
PREFILL_CASES = [  # M, N, K, splitk
    (65, 256, 512, 1), (70, 384, 768, 3), (128, 512, 512, 2), (129, 256, 1024, 8), (192, 640, 256, 4), (255, 384, 768, 3),
    (256, 1024, 512, 1), (256, 512, 1024, 8), (100, 256, 1024, 8),
]


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


LLAMA3_8B_KV, LLAMA2_7B_KV, LLAMA2_13B_KV = 8, 32, 40


@pytest.mark.parametrize("M,N,K,splitk,epi,nkv", [
    (60, 6144, 4096, 4, "qkv", LLAMA3_8B_KV), (60, 4096, 4096, 8, "res", None), (60, 14336, 4096, 2, "swiglu", None),
    (60, 4096, 14336, 8, "res", None), (60, 128256, 4096, 1, "store", None), (10, 32000, 4096, 1, "store", None),
    (10, 6144, 8192, 4, "store", None), (8, 4096, 12288, 8, "store", None),
    # a full 256-row prompt chunk: Llama-3-8B qkv / o / gate_up / down, Llama-3-70B o / down
    (256, 6144, 4096, 4, "qkv", LLAMA3_8B_KV), (256, 4096, 4096, 4, "res", None), (256, 14336, 4096, 1, "swiglu", None),
    (256, 4096, 14336, 4, "res", None), (256, 8192, 8192, 2, "res", None), (256, 8192, 28672, 2, "res", None),
    # Vicuna-7B / Llama-2-13B (MHA, I = 11008 / 13824) at the verify pass's 60 rows and a 256-row prompt chunk: qkv, o, gate_up,
    # down; and the EAGLE-1 head's fc over cat(emb, hidden) with its bias (the draft runs at most 64 rows, so 60 only)
    (60, 3 * 4096, 4096, 4, "qkv", LLAMA2_7B_KV), (60, 4096, 4096, 8, "res", None), (60, 11008, 4096, 2, "swiglu", None),
    (60, 4096, 11008, 4, "res", None), (60, 4096, 2 * 4096, 8, "fc", None),
    (256, 3 * 4096, 4096, 4, "qkv", LLAMA2_7B_KV), (256, 4096, 4096, 4, "res", None), (256, 11008, 4096, 1, "swiglu", None),
    (256, 4096, 11008, 4, "res", None),
    (60, 3 * 5120, 5120, 4, "qkv", LLAMA2_13B_KV), (60, 5120, 5120, 8, "res", None), (60, 13824, 5120, 2, "swiglu", None),
    (60, 5120, 13824, 8, "res", None), (60, 5120, 2 * 5120, 8, "fc", None),
    (256, 3 * 5120, 5120, 4, "qkv", LLAMA2_13B_KV), (256, 5120, 5120, 4, "res", None), (256, 13824, 5120, 1, "swiglu", None),
    (256, 5120, 13824, 4, "res", None),
])
@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_gemm_llama3_8b_shapes(lib, M, N, K, splitk, epi, nkv, mode, dtype):
    """The projections of the benchmark configurations (BASELINE.json: Llama-3-8B, Vicuna-7B, Llama-2-13B) at full size in both
    model dtypes, and those of a 256-row prompt chunk (Llama-3-70B's o / down too), checked against a float64 reference on
    sampled output columns (size-independent property: linearity in W rows).  At 256 rows the prefill's epilogues run: gate/up
    interleaved, and qkv through the QKV + RoPE epilogue with an identity rotation (cos 1, sin 0), which makes it a store into
    q and the K / V caches (the rotation itself is held to the reference by test_qkv_rope_kv_append)."""
    R = x_rows(M)
    g = torch.Generator(device="cuda").manual_seed(N + K)
    X = (torch.randn(R, K, generator=g, device="cuda") * 0.5).to(dtype)
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
    cols = torch.randint(0, N, (512,), generator=torch.Generator().manual_seed(3)).cuda()
    torch.cuda.synchronize()
    if epi == "swiglu":
        W2 = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(dtype)
        torch.cuda.synchronize()
        out = torch.zeros(R, N, dtype=dtype, device="cuda")
        if M > 64:
            Wil = interleave64(W, W2)
            torch.cuda.synchronize()
            check(lib, lib.eb200_k_gemm(DT[dtype], mode, 5, ptr(Wil), None, ptr(X), ptr(out), None, None, M, N, K, splitk, None))
        else:
            check(lib, lib.eb200_k_gemm(DT[dtype], mode, 2, ptr(W), ptr(W2), ptr(X), ptr(out), None, None, M, N, K, splitk, None))
        gate = (X[:M].double() @ W[cols].double().t()).to(dtype)
        up = (X[:M].double() @ W2[cols].double().t()).to(dtype)
        want = F.silu(gate) * up
        err = (out[:M][:, cols].float() - want.float()).abs()
        tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
        assert bool((err <= tol).all()), f"max err {float(err.max())}"
        return
    res = torch.randn(R, N, generator=g, device="cuda").to(dtype) if epi == "res" else None
    bias = (torch.randn(N, generator=g, device="cuda") * 0.1).to(dtype) if epi == "fc" else None
    torch.cuda.synchronize()
    out = res.clone() if res is not None else torch.zeros(R, N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    if epi == "qkv" and M > 64:
        nh = N // 128 - 2 * nkv
        cos = torch.ones(M, 64, dtype=dtype, device="cuda")
        kc = torch.zeros(nkv, M, 128, dtype=dtype, device="cuda")
        vc = torch.zeros(nkv, M, 128, dtype=dtype, device="cuda")
        q_out = torch.zeros(R, nh * 128, dtype=dtype, device="cuda")
        torch.cuda.synchronize()
        check(lib, lib.eb200_k_qkv_rope(DT[dtype], mode, ptr(W), ptr(X), ptr(q_out), ptr(kc), ptr(vc), ptr(cos), ptr(torch.zeros_like(cos)), None,
                                        M, nh, nkv, K, M, 0, splitk, None))
        out = torch.cat((q_out[:M], kc.transpose(0, 1).reshape(M, -1), vc.transpose(0, 1).reshape(M, -1)), dim=1)
    else:
        code = 1 if epi == "res" else 0
        check(lib, lib.eb200_k_gemm(DT[dtype], mode, code, ptr(W), None, ptr(X), ptr(out), ptr(out) if res is not None else None, ptr(bias),
                                    M, N, K, splitk, None))
    proj = (X[:M].double() @ W[cols].double().t() + (bias[cols].double() if bias is not None else 0)).to(dtype)
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
@pytest.mark.parametrize("M,N,K,splitk", [(10, 512, 256, 1), (60, 1024, 256, 2), (60, 1408, 512, 1), (60, 1792, 4096, 4), (7, 64, 256, 1)]
                         + [(M, 64 * (N // 128), K, sk) for M, N, K, sk in PREFILL_CASES])
def test_gemm_swiglu_interleaved(lib, M, N, K, splitk, dtype, mode):
    """Single-accumulator SwiGLU over interleaved gate/up rows: same rounding points as the two-matrix kernel, so the two
    must agree BIT FOR BIT (same fp32 accumulation order per element), and both sit within tolerance of the torch reference.
    Above 64 rows (the prefill's 256-row launch, which has no two-matrix form) only the reference bar applies."""
    if mode == 1 and M > 64:
        pytest.skip("the SIMT bring-up kernel runs at most 64 rows")
    g = torch.Generator().manual_seed(12 + N)
    X = (torch.randn(x_rows(M), K, generator=g)).to(dtype)
    Wg = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    Wu = (torch.randn(N, K, generator=g) * 0.08).to(dtype)
    gate = F.linear(X[:M].float(), Wg.float()).to(dtype)
    up = F.linear(X[:M].float(), Wu.float()).to(dtype)
    want = F.silu(gate) * up
    Wil = interleave64(Wg, Wu).cuda()
    Xd = X.cuda()
    out = torch.zeros(x_rows(M), N, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    check(lib, lib.eb200_k_gemm(DT[dtype], mode, 5, ptr(Wil), None, ptr(Xd), ptr(out), None, None, M, N, K, splitk, None))
    err = (out[:M].float().cpu() - want.float()).abs()
    tol = 1e-3 + 3.2 * ULP[dtype] * want.float().abs() + ULP[dtype] * up.float().abs() * 0.02
    assert bool((err <= tol).all()), f"gemm_swiglu_il: {int((err > tol).sum())} bad, max err {float(err.max())}"
    if M < out.shape[0]:
        assert float(out[M:].abs().max()) == 0.0
    if mode != 1 and N % 128 == 0 and M <= 64:
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
@pytest.mark.parametrize("M,N,K,splitk", [(10, 256, 512, 1), (60, 512, 256, 2), (60, 4096, 1024, 4)] + PREFILL_CASES)
def test_gemm_residual(lib, M, N, K, splitk, dtype, mode):
    g = torch.Generator().manual_seed(11)
    X = (torch.randn(x_rows(M), K, generator=g) * 0.5).to(dtype)
    W = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
    res = torch.randn(x_rows(M), N, generator=g).to(dtype)
    proj = F.linear(X[:M].float(), W.float()).to(dtype)
    want = res[:M] + proj  # x + o_proj(a): two roundings
    out = res.clone().cuda()
    check(lib, lib.eb200_k_gemm(DT[dtype], mode, 1, ptr(W.cuda()), None, ptr(X.cuda()), ptr(out), ptr(out), None, M, N, K, splitk, None))
    # 1 ulp of the projection (it may flip before the add) + 1 ulp of the sum
    err = (out[:M].float().cpu() - want.float()).abs()
    tol = 1e-3 + ULP[dtype] * (proj.float().abs() + want.float().abs())
    assert bool((err <= tol).all()), f"gemm_residual: {int((err > tol).sum())} bad, max err {float(err.max())}"
    assert torch.equal(out[M:].cpu(), res[M:])  # rows beyond M are never written


def test_gemm_and_qkv_rope_refuse_what_the_prefill_does_not_run_at_256_rows(lib):
    """Above 64 rows the entry points run only what the prompt prefill runs; everything else fails before any launch, so the
    output buffer keeps its contents."""
    dtype = torch.bfloat16
    N, K = 256, 256
    W, X = torch.zeros(3 * 128, K, dtype=dtype, device="cuda"), torch.zeros(256, K, dtype=dtype, device="cuda")  # W: N rows, or q/k/v heads
    out = torch.full((256, N), 7.0, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    refused = {  # what: (simt, epilogue, W2, M)
        "store": (0, 0, None, 65), "two-matrix SwiGLU": (0, 2, W, 65), "fp32 partials": (0, 4, None, 65),
        "SIMT kernel": (1, 1, None, 65), "M > 256": (0, 1, None, 257), "M = 0": (0, 1, None, 0),
    }
    for what, (simt, epi, W2, M) in refused.items():
        rc = lib.eb200_k_gemm(0, simt, epi, ptr(W), ptr(W2), ptr(X), ptr(out), ptr(out), None, M, N, K, 1, None)
        assert rc != 0, f"eb200_k_gemm ran {what}"
        assert lib.eb200_last_error().decode(), what
    cos = torch.ones(2048, 64, dtype=dtype, device="cuda")
    kc = torch.full((1, 1024, 128), 7.0, dtype=dtype, device="cuda")
    for what, (simt, M, kv_base) in {"SIMT kernel": (1, 65, 0), "M > 256": (0, 257, 0), "cache rows past kv_cap": (0, 200, 900)}.items():
        rc = lib.eb200_k_qkv_rope(0, simt, ptr(W), ptr(X), ptr(out), ptr(kc), ptr(kc), ptr(cos), ptr(cos), None, M, 1, 1, K, 1024,
                                  kv_base, 1, None)
        assert rc != 0, f"eb200_k_qkv_rope ran {what}"
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((kc == 7.0).all()), "a refused call wrote its output"


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


QKV_CASES = [  # M, nh, nkv, K, splitk, kv_base, position form: "pos" = pos[m] (the cycle's), "prefill" = kv_base + m
    pytest.param(10, 2, 1, 256, 1, 37, "pos", id="10-2-1-256-1"), pytest.param(60, 4, 2, 512, 2, 37, "pos", id="60-4-2-512-2"),
    pytest.param(7, 2, 2, 512, 1, 37, "pos", id="7-2-2-512-1"),
    # the prompt prefill's 256-row launch, kv_base 0 / 256 / past 1000 in both position forms
    (65, 2, 1, 256, 1, 0, "prefill"), (70, 2, 2, 512, 3, 256, "pos"), (128, 4, 2, 512, 2, 1029, "prefill"), (129, 2, 1, 1024, 8, 0, "pos"),
    (192, 2, 2, 256, 4, 256, "prefill"), (255, 4, 2, 768, 3, 1029, "pos"), (256, 2, 1, 512, 1, 1029, "prefill"),
    (100, 2, 1, 1024, 8, 256, "pos"), (256, 4, 1, 1024, 8, 0, "prefill"),
]


@pytest.mark.parametrize("simt", MODES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,nh,nkv,K,splitk,kv_base,form", QKV_CASES)
def test_qkv_rope_kv_append(lib, M, nh, nkv, K, splitk, kv_base, form, dtype, simt):
    if simt == 1 and M > 64:
        pytest.skip("the SIMT bring-up kernel runs at most 64 rows")
    R = x_rows(M)
    g = torch.Generator().manual_seed(13)
    X = torch.randn(R, K, generator=g).to(dtype)
    Wq = (torch.randn(nh * 128, K, generator=g) * 0.06).to(dtype)
    Wk = (torch.randn(nkv * 128, K, generator=g) * 0.06).to(dtype)
    Wv = (torch.randn(nkv * 128, K, generator=g) * 0.06).to(dtype)
    n_pos = 2048
    cap = 256 if M <= 64 else 1536
    pos = torch.randint(0, 200 if M <= 64 else n_pos, (R,), generator=g, dtype=torch.int32)
    if form == "prefill":
        pos = torch.arange(kv_base, kv_base + R, dtype=torch.int32)
    cos, sin = orc.rope_table(128, n_pos, 500000.0)
    cosT, sinT = cos.to(dtype), sin.to(dtype)
    q = F.linear(X[:M].float(), Wq.float()).to(dtype).view(1, M, nh, 128).transpose(1, 2)
    k = F.linear(X[:M].float(), Wk.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2)
    v = F.linear(X[:M].float(), Wv.float()).to(dtype).view(1, M, nkv, 128).transpose(1, 2)
    qr, kr = orc.apply_rope(q, k, cosT, sinT, pos[:M].long()[None])
    Wqkv = torch.cat([Wq, Wk, Wv]).cuda()
    q_out = torch.zeros(R, nh * 128, dtype=dtype, device="cuda")
    kc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
    vc = torch.zeros(nkv, cap, 128, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_qkv_rope(DT[dtype], simt, ptr(Wqkv), ptr(X.cuda()), ptr(q_out), ptr(kc), ptr(vc),
                                    ptr(cosT[:, :64].contiguous().cuda()), ptr(sinT[:, :64].contiguous().cuda()),
                                    ptr(pos.cuda()) if form == "pos" else None, M, nh, nkv, K, cap, kv_base, splitk, None))
    if M <= 64:  # the cycle-form cases keep the plain 1-ulp bar they were written with
        close(q_out[:M].view(M, nh, 128).transpose(0, 1), qr[0], dtype, "q rope")
        close(kc[:, kv_base:kv_base + M], kr[0], dtype, "k rope/cache")
    else:
        close_rope(q_out[:M].view(M, nh, 128).transpose(0, 1), q[0], cosT, sinT, pos[:M].long(), qr[0], dtype, "q rope")
        close_rope(kc[:, kv_base:kv_base + M], k[0], cosT, sinT, pos[:M].long(), kr[0], dtype, "k rope/cache")
    close(vc[:, kv_base:kv_base + M], v[0], dtype, "v cache")
    # cache rows outside [kv_base, kv_base + M) and q rows beyond M are never written
    for t in (kc[:, :kv_base], kc[:, kv_base + M:], vc[:, :kv_base], vc[:, kv_base + M:], q_out[M:]):
        assert not bool(t.any())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("epi", ["residual", "swiglu", "qkv_rope"])
def test_256_rows_equal_64_row_launches_bit_for_bit(lib, epi, dtype):
    """One 256-row launch over rows [0, M) against separate launches (64 or 16 rows, like the 64-row prompt chunks and the cycle)
    on each 64-row block of X, with the same splitk: each output element sums the same products in the same k-block and rank
    order, so the two must agree bit for bit.  This is what makes the engine's 256-row and 64-row prefills identical."""
    g = torch.Generator(device="cuda").manual_seed(21)
    K, nh, nkv, kv_base = 1024, 4, 2, 300
    N = {"residual": 1024, "swiglu": 512, "qkv_rope": (nh + 2 * nkv) * 128}[epi]
    rows = 2 * N if epi == "swiglu" else N
    X = torch.randn(256, K, generator=g, device="cuda").to(dtype)
    W = (torch.randn(rows, K, generator=g, device="cuda") * 0.05).to(dtype)
    res = torch.randn(256, N, generator=g, device="cuda").to(dtype)
    cos, sin = (t.to(dtype)[:, :64].contiguous().cuda() for t in orc.rope_table(128, 1024, 500000.0))
    torch.cuda.synchronize()

    def run(r0, M, splitk, out, q_out, kc, vc):
        """Rows [r0, r0 + M) of X in one launch."""
        x = ptr(X[r0:])
        if epi == "qkv_rope":
            return lib.eb200_k_qkv_rope(DT[dtype], 0, ptr(W), x, ptr(q_out[r0:]), ptr(kc), ptr(vc), ptr(cos), ptr(sin), None, M, nh, nkv,
                                        K, 1024, kv_base + r0, splitk, None)
        if epi == "residual":
            return lib.eb200_k_gemm(DT[dtype], 0, 1, ptr(W), None, x, ptr(out[r0:]), ptr(out[r0:]), None, M, N, K, splitk, None)
        return lib.eb200_k_gemm(DT[dtype], 0, 5, ptr(W), None, x, ptr(out[r0:]), None, None, M, N, K, splitk, None)

    for M, splitk in [(256, 1), (256, 4), (200, 2), (129, 3), (65, 8), (100, 8)]:
        results = []
        for blocks in (False, True):
            out = res.clone() if epi == "residual" else torch.zeros(256, N, dtype=dtype, device="cuda")
            q_out = torch.zeros(256, nh * 128, dtype=dtype, device="cuda")
            kc = torch.zeros(nkv, 1024, 128, dtype=dtype, device="cuda")
            vc = torch.zeros(nkv, 1024, 128, dtype=dtype, device="cuda")
            torch.cuda.synchronize()
            for r0 in (range(0, M, 64) if blocks else [0]):
                check(lib, run(r0, min(64, M - r0) if blocks else M, splitk, out, q_out, kc, vc))
            results.append((out, q_out, kc, vc))
        for what, a, b in zip(("out", "q", "K cache", "V cache"), *results):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (
                f"{epi} M={M} splitk={splitk}: {what} of the 256-row launch differs from the 64-row launches in "
                f"{int((a != b).sum())} elements, max {float((a.float() - b.float()).abs().max()):.3g}")


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
@pytest.mark.parametrize("V,dtype", [(512, torch.bfloat16), (32000, torch.float16), (128256, torch.bfloat16), (32003, torch.float16)],
                         ids=["512-bf16", "32000-fp16", "128256-bf16", "32003-fp16"])
def test_sample_posterior_matches_oracle(lib, V, dtype, seed, temperature, top_p, top_k):
    """Decisions, uniforms drawn and the bonus token against tests/sampling_ref.posterior (the oracle's
    evaluate_posterior_sampling on the rows as the stats kernel warped them; the thresholds of the rows the walk reads are
    held to the float64 reference here, all of them by tests/test_sampling_gpu.py)."""
    from tests import sampling_ref as sr
    g = torch.Generator().manual_seed(200 + seed)
    k, depth, total = 10, 6, 60
    scores, tokens, parents = _random_pool(k, depth, seed, torch.float32)
    scores = scores + torch.arange(scores.numel()) * 1e-7
    tokens = torch.randint(0, 40, (scores.numel(),), generator=g)  # small token range so candidates get real probability
    draft_tokens, retrieve, _, _ = orc.finalize_tree(scores, tokens, parents, torch.tensor([3]), k, total - 1, True)
    logits_nodes = (torch.randn(total, V, generator=g) * 1.5).to(dtype)
    # the draft's token range is likely under the target too, about as likely at every vocabulary size
    logits_nodes[:, :40] += 4.0 + math.log(V / 512)
    lg_d = logits_nodes.cuda()
    cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
    st = torch.zeros(total, 3)
    check(lib, lib.eb200_k_sample_stats(DT[dtype], ptr(lg_d), total, V, temperature, top_p, top_k, ptr(st)))
    thr = st[:, 2].double()
    lt = sr.temperature_warp(logits_nodes, temperature)
    for attempt in range(10):  # redraw uniforms that fall within rounding distance of an acceptance probability
        uniforms = torch.rand(64, generator=g)
        w_best, w_acc, w_p, w_used, ambiguous = sr.posterior(lt, thr, cands, retrieve, uniforms.tolist())
        if not ambiguous:
            break
    assert not ambiguous
    best, acc, bonus, used = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    check(lib, lib.eb200_k_sample_posterior(DT[dtype], ptr(lg_d), V, ptr(draft_tokens[0].int().contiguous()),
                                            ptr(retrieve.int().contiguous()), total, retrieve.shape[0], retrieve.shape[1], temperature, top_p,
                                            top_k, ptr(uniforms.contiguous()), 64, C.byref(best), C.byref(acc), C.byref(bonus), C.byref(used)))
    assert (best.value, acc.value) == (w_best, w_acc)
    assert used.value == w_used
    for node in retrieve[w_best, :w_acc + 1].tolist():  # the rows the walk and the bonus draw read
        adm = sr.RowRef(lt[node]).admissible(top_p, top_k)
        assert float(thr[node]) in adm, (node, float(thr[node]), sorted(adm)[:4])
    ok = sr.bracket(w_p, float(uniforms[used.value - 1]), sr.cdf_delta_rel(V))
    assert bool(ok[bonus.value]), (f"bonus {bonus.value} (p = {float(w_p[bonus.value]):.3g}) outside the bracket "
                                   f"{torch.nonzero(ok).flatten()[:8].tolist()}")

"""Parity of the lm_head launch (eagle_b200/csrc/mega.cu: whole 128-row weight tiles per CTA) on the H100, through the C ABI.

The kernel replaces ea_model.py:190 + utils.py:362 (lm_head + arg-max) in the verify pass, and the lm_head alone (direct store
of the logits) in the sampling path.  The stored logits are held to 1 ulp of the model dtype + 1e-3 against fp32 math; the
arg-max is exact, including torch.argmax's first-index rule on ties.
"""
import pytest
import torch

from tests.test_kernels_gpu import _KEEP, DT, check, close, lib, ptr  # noqa: F401  (lib is a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def release_kept_tensors():
    """ptr() keeps the last 64 tensors it was given alive.  Here those are lm_head-sized weights (1 GB each at V = 128256):
    release them when this module ends, so that the modules after it find the device memory free (the FP8 Llama-3-70B
    engine of tests/test_fp8_gpu.py needs nearly all of an 80 GB card)."""
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def dev_randn(shape, g, scale, dtype):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


# ----------------------------------------------------------------------------------------------
# single GEMM through the lm_head launch: direct store (mode 1), fused arg-max (mode 2)
# ----------------------------------------------------------------------------------------------
CHAIN_GEMM_CASES = [
    # M, N, K   (tiny problems leave most CTAs without a tile; odd tile counts; the benchmark's projection shapes)
    (1, 256, 256), (10, 512, 256), (60, 256, 2048), (64, 1024, 512), (7, 384, 768), (33, 200, 320),
    (60, 4096, 4096), (60, 6144, 4096), (60, 4096, 14336), (10, 32000, 4096), (10, 4096, 12288),
    # the sampling path's verify lm_head (FIN_STORE_DIRECT, all 60 rows of logits) at Llama-2-13B and Llama-3-8B width, and the
    # prefill's one-row lm_head at 13B width
    (60, 32000, 5120), (60, 128256, 4096), (1, 32000, 5120),
]


@pytest.mark.parametrize("mode", [1])  # direct store; mode 2 (fused arg-max) is tested below
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
    # three launches back to back: the counters reset themselves between launches
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

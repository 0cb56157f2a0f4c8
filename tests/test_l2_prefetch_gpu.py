"""L2 weight prefetch (kernels.h L2Prefetch) on the H100: it only moves weight bytes into L2 earlier, so every output is bit for
bit what the same kernels compute without it.

1. Kernel level (eb200_k_prefetch): the cluster GEMM and RMSNorm, prefetching another matrix, against the plain kernels.  Tiny,
   ragged (N % 128, K % 64 != 0) and Llama-3-8B shapes; plans that prefetch nothing, part of the matrix, more rows than it
   has, and that start below row 0.
2. End to end: an 8-layer Llama-3-8B-width engine (EAGLE-3 head, correlated weights so that drafts are accepted), dynamic and
   static tree, run in two subprocesses with EB200_L2_PREFETCH=0 and =1 (the switch is read once per process).
   Every cycle's tree, verify result and committed tokens must be identical.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {torch.bfloat16: 0, torch.float16: 1}


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def rand(shape, seed, dtype, scale=0.02):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


# (PN, PK, p_splitk) of the prefetched matrix: tiny, ragged, Llama-3-8B o_proj / gate_up / down_proj under the engine's split-K
PREFETCHED = [(256, 256, 1), (200, 320, 2), (4096, 4096, 4), (28672, 4096, 1), (4096, 14336, 4)]
# (j0, j1): nothing, nothing (j1 < j0), the first k-block row, part, more rows than any split has, starting below row 0
PLANS = [(0, 0), (3, 1), (0, 1), (1, 5), (0, 1 << 20), (-4, 2)]


@pytest.mark.parametrize("pn,pk,psk", PREFETCHED)
@pytest.mark.parametrize("j0,j1", PLANS)
@pytest.mark.parametrize("M,N,K,splitk,epi", [(10, 200, 320, 1, 0), (60, 4096, 4096, 4, 1), (16, 6144, 4096, 4, 0)])
def test_gemm_with_prefetch_is_unchanged(lib, pn, pk, psk, j0, j1, M, N, K, splitk, epi):
    dtype = torch.bfloat16
    W, X, P = rand((N, K), 1, dtype), rand((64, K), 2, dtype, 1.0), rand((pn, pk), 3, dtype)
    res = rand((M, N), 4, dtype, 1.0) if epi == 1 else None
    want = res.clone() if epi == 1 else torch.empty(M, N, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_gemm(DT[dtype], 2, epi, ptr(W), None, ptr(X), ptr(want), ptr(want) if epi == 1 else None, None, M, N, K, splitk, None))
    got = res.clone() if epi == 1 else torch.empty(M, N, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_prefetch(DT[dtype], 0, epi, ptr(W), ptr(X), ptr(got), ptr(got) if epi == 1 else None, M, N, K, splitk, 0.0,
                                    ptr(P), pn, pk, psk, j0, j1, None))
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize("pn,pk,psk", PREFETCHED)
@pytest.mark.parametrize("j0,j1", PLANS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rmsnorm_with_prefetch_is_unchanged(lib, pn, pk, psk, j0, j1, dtype):
    rows, H = 60, 4096
    x, w, P = rand((rows, H), 5, dtype, 1.0), rand((H,), 6, dtype, 1.0), rand((pn, pk), 7, dtype)
    want = torch.empty(rows, H, dtype=dtype, device="cuda")
    check(lib, lib.eb200_k_rmsnorm(DT[dtype], ptr(x), ptr(w), ptr(want), rows, H, 1e-5, None))
    got = torch.empty_like(want)
    check(lib, lib.eb200_k_prefetch(DT[dtype], 1, 0, ptr(w), ptr(x), ptr(got), None, rows, H, 0, 1, 1e-5, ptr(P), pn, pk, psk, j0, j1, None))
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_prefetch_rejects_bad_arguments(lib):
    P = torch.zeros(128, 64, dtype=torch.bfloat16, device="cuda")
    for bad in [dict(kernel=2), dict(p_splitk=0), dict(p_splitk=9), dict(pn=0)]:
        a = dict(kernel=1, p_splitk=1, pn=128)
        a.update(bad)
        rc = lib.eb200_k_prefetch(0, a["kernel"], 0, ptr(P), ptr(P), ptr(P), None, 1, 64, 0, 1, 1e-5, ptr(P), a["pn"], 64, a["p_splitk"], 0, 1,
                                  None)
        assert rc != 0, bad


# ----------------------------------------------------------------------------------------------
# end to end, prefetch on vs off
# ----------------------------------------------------------------------------------------------
RUN = r"""
import argparse, json, sys
import torch
import bench
args = argparse.Namespace(model="llama3-8b", dtype="bf16", tree=sys.argv[1], fixture="correlated", layers=8, temperature=0.0)
m, tcfg, hcfg, eagle3 = bench.build_engine(args, 0, 0, 1)
from eagle_b200 import synthetic as syn
used = syn.draft_vocab_ids(tcfg["vocab_size"], 32000)
prompt = used[torch.randint(0, used.numel(), (300,), generator=torch.Generator().manual_seed(0))][None].cuda()
out = {"first": m.prefill(prompt), "cycles": []}
for _ in range(24):
    dt, ri, tm, tp = m.get_tree()
    toks, nxt = m.step()
    am, best, acc, n = m.get_verify()
    out["cycles"].append({"tree": dt.tolist(), "retrieve": ri.tolist(), "mask": tm.flatten().nonzero().flatten().tolist(), "pos": tp.tolist(),
                          "argmax": am.tolist(), "best": best, "accept": acc, "tokens": toks, "next": nxt})
ids, new_token, idx = m.eagenerate(prompt, max_new_tokens=96, log=True)
out["ids"], out["new_token"], out["idx"] = ids.tolist(), int(new_token), int(idx)
print("RESULT " + json.dumps(out))
"""


def run(tree, prefetch):
    env = dict(os.environ, EB200_L2_PREFETCH=prefetch)
    p = subprocess.run([sys.executable, "-s", "-c", RUN, tree], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    return json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][len("RESULT "):])


@pytest.mark.parametrize("tree", ["dynamic", "static"])
def test_generation_identical_with_and_without_prefetch(tree):
    off, on = run(tree, "0"), run(tree, "1")
    assert max(c["accept"] for c in off["cycles"]) >= 2, "the fixture must accept drafts"
    assert on["first"] == off["first"]
    for c, (a, b) in enumerate(zip(off["cycles"], on["cycles"])):
        assert a == b, f"cycle {c} differs"
    assert (on["ids"], on["new_token"], on["idx"]) == (off["ids"], off["new_token"], off["idx"])

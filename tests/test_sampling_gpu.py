"""The sampling path on the H100 at the engine's vocabulary sizes, against the float64 reference of tests/sampling_ref.py
(held to the oracle's warpers by tests/test_sampling_ref_cpu.py):

* row_softmax_stats_kernel (eb200_k_sample_stats): max bit for bit, the keep-threshold one of the reference's admissible
  values (never NaN, never above max), the normaliser within the reference's rounding bound;
* the first-token draw of sample_row0 (eb200_k_sample_token): the token lies in the reference's inverse-CDF bracket,
  including uniforms on a per-thread chunk edge of sample_commit_kernel and inside a chunk whose only kept token is its last;
* the sampling posterior (eb200_k_sample_posterior) with every level-1 candidate rejected, duplicates, removed candidates;
* losslessness with the warpers: the first committed token over 20 000 seeded trials against the float64 warped target.

Row families: flat Gaussian, peaked (p = 1 - 1e-6), tie-heavy (a few values, thousands of tokens each), masked (-inf
entries), +-0.0 at the threshold, all-equal, and top-p binding at the second token."""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

from tests import sampling_ref as sr

pytestmark = pytest.mark.gpu

DT = {torch.bfloat16: 0, torch.float16: 1}
SHAPES = [(32000, torch.float16), (32000, torch.bfloat16), (128256, torch.bfloat16), (128256, torch.float16),
          (32003, torch.bfloat16), (32003, torch.float16)]
TEMPERATURES = [1.0, 0.7, 1.3, 0.05]
TOP_PS = [0.0, 1e-8, 2e-8, 3e-8, 0.02, 0.6, 0.9, 0.999, 1.0]
FP32_TINY = 2.0 ** -126  # smallest normal fp32
MASKED_CHUNK = 100  # in the masked row, this chunk of sample_commit_kernel keeps only its last token


def top_ks(V):
    return [0, 1, 10, 50, V - 1, V, V + 5]


@pytest.fixture(scope="module")
def lib():
    from eagle_b200 import _lib
    return _lib.load()


def check(lib, rc):
    assert rc == 0, lib.eb200_last_error().decode()


_KEEP = []


def ptr(t):
    _KEEP.append(t)
    if len(_KEEP) > 64:
        del _KEEP[:-64]
    return C.c_void_p(t.data_ptr())


def family_rows(V, dtype, seed=0):
    """[R][V] rows of every family, in the model dtype, and their names."""
    g = torch.Generator().manual_seed(1000 + V + seed)
    rows, names = [], []

    def add(name, x):
        rows.append(x.to(dtype))
        names.append(name)

    for i in range(2):
        add(f"flat{i}", torch.randn(V, generator=g))
    x = torch.randn(V, generator=g, dtype=torch.float64)
    top = int(torch.randint(0, V, (1,), generator=g))
    x[top] = math.log(torch.exp(x).sum() * 1e6)  # p(top) = 1 - 1e-6
    add("peaked", x)
    levels = torch.tensor([-3.0, -1.0, 0.0, 0.5, 1.25])
    add("ties", levels[torch.randint(0, 5, (V,), generator=g)])
    x = torch.randn(V, generator=g)
    x[torch.rand(V, generator=g) < 0.3] = -math.inf
    per = sr.per_thread(V)
    x[MASKED_CHUNK * per:(MASKED_CHUNK + 1) * per - 1] = -math.inf
    x[(MASKED_CHUNK + 1) * per - 1] = float(x[torch.isfinite(x)].max()) + 1.0  # the chunk's last token is the row maximum
    add("masked", x)
    x = -(torch.rand(V, generator=g) * 3 + 1)  # (-4, -1]
    idx = torch.randperm(V, generator=g)
    x[idx[:5]] = 2.0
    x[idx[5:305]] = 0.0
    x[idx[305:605]] = -0.0
    add("zeros", x)
    add("equal", torch.full((V,), 0.5))
    x = torch.randn(V, generator=g) * 0.5 - math.log(V) - 2.0
    a, b = torch.randperm(V, generator=g)[:2].tolist()
    x[a], x[b] = 0.0, -0.4  # p(a) ~ 0.55, p(b) ~ 0.37, the rest ~ 0.08: top-p 0.6 and 0.9 bind at the second token
    add("second", x)
    return torch.stack(rows), names


def stats(lib, xd, dtype, t, p, k):
    out = np.zeros((xd.shape[0], 3), dtype=np.float32)
    check(lib, lib.eb200_k_sample_stats(DT[dtype], ptr(xd), xd.shape[0], xd.shape[1], t, p, k, out.ctypes.data_as(C.c_void_p)))
    return out


def sample_token(lib, row_d, dtype, t, p, k, u):
    tok = C.c_int32()
    check(lib, lib.eb200_k_sample_token(DT[dtype], ptr(row_d), row_d.numel(), t, p, k, u, C.byref(tok)))
    return tok.value


def stats_problem(ref, got, top_p, top_k):
    """None when the kernel's (max, sum, thr) agree with the reference, else what is wrong."""
    mx, s, thr = (float(v) for v in got)
    adm = ref.admissible(top_p, top_k)
    if mx != ref.max:
        return f"max {mx!r} != {ref.max!r}"
    if math.isnan(thr) or thr > mx:
        return f"thr {thr!r} (max {mx!r})"
    if thr not in adm:
        return f"thr {thr!r} not admissible {sorted(adm)[:4]}"
    if abs(s - adm[thr]) > sr.stats_delta_rel(ref.V) * adm[thr]:
        return f"sum {s!r} vs {adm[thr]!r} at thr {thr!r}"
    return None


def _fail(bad, what):
    assert not bad, f"{len(bad)} {what}; first: " + "\n".join(bad[:20])


@pytest.mark.parametrize("V,dtype", SHAPES)
def test_row_stats_match_the_float64_reference(lib, V, dtype):
    x, names = family_rows(V, dtype)
    xd = x.cuda()
    bad = []
    for t in TEMPERATURES:
        refs = [sr.RowRef(lt) for lt in sr.temperature_warp(x, t)]
        for p in TOP_PS:
            for k in top_ks(V):
                got = stats(lib, xd, dtype, t, p, k)
                for r, ref in enumerate(refs):
                    why = stats_problem(ref, got[r], p, k)
                    if why:
                        bad.append(f"{names[r]} T={t} top_p={p} top_k={k}: {why}")
    _fail(bad, "rows out of the reference")


def _chunk_uniforms(w, V):
    """Uniforms that put u S on the end of the per-thread chunk nearest the median, and inside the first chunk whose only
    eligible token is its last (None when there is none)."""
    per = sr.per_thread(V)
    c = torch.cumsum(w, 0)
    s = float(c[-1])
    ends = c[torch.clamp(torch.arange(1, sr.CHUNKS + 1) * per, max=V) - 1] / s
    inner = (ends > 0) & (ends < 1)
    edge = float(ends[inner][torch.argmin((ends[inner] - 0.5).abs())]) if inner.any() else 0.5
    only_last = None
    pad = torch.zeros(sr.CHUNKS * per, dtype=torch.float64)
    pad[:V] = w
    chunks = pad.view(sr.CHUNKS, per) > 0
    for ch in torch.nonzero((chunks.sum(1) == 1) & chunks[:, -1]).flatten().tolist():
        last = (ch + 1) * per - 1
        if last < V and per > 1:
            only_last = (float(c[last]) - float(w[last]) / 2) / s
            break
    return edge, only_last


@pytest.mark.parametrize("V,dtype", SHAPES)
def test_first_token_draw_lies_in_the_inverse_cdf_bracket(lib, V, dtype):
    x, names = family_rows(V, dtype)
    xd = x.cuda()
    ks = top_ks(V)
    d_rel = sr.cdf_delta_rel(V)
    bad, n_only_last = [], 0
    # 36 combinations: every temperature, top_p and top_k value, 36 of the 63 (top_p, top_k) pairs
    for i in range(36):
        t, p, k = TEMPERATURES[i % 4], TOP_PS[i % 9], ks[i % 7]
        got = stats(lib, xd, dtype, t, p, k)
        for r, lt in enumerate(sr.temperature_warp(x, t)):
            ref = sr.RowRef(lt)
            why = stats_problem(ref, got[r], p, k)
            if why:
                bad.append(f"{names[r]} T={t} top_p={p} top_k={k}: stats {why}")
                continue
            w = ref.weights(float(got[r][2]))
            edge, only_last = _chunk_uniforms(w, V)
            us = [0.0, 1e-7, 0.5, 1 - 2.0 ** -24, 1.0, edge] + ([only_last] if only_last is not None else [])
            n_only_last += only_last is not None
            # u = 0 takes the first token whose weight is positive in fp32; weights below the fp32 range (T = 0.05 puts
            # most of a peaked row under e^-400) may be skipped
            first_fp32 = int(torch.nonzero(w >= FP32_TINY)[0])
            for u in us:
                u32 = float(np.float32(u))
                tok = sample_token(lib, xd[r], dtype, t, p, k, u32)
                ok = sr.bracket(w, u32, d_rel)
                if not (0 <= tok < V and bool(ok[tok])) or (u32 == 0.0 and tok > first_fp32):
                    adm = torch.nonzero(ok).flatten()[:6].tolist()
                    bad.append(f"{names[r]} T={t} top_p={p} top_k={k} u={u32!r}: token {tok}, bracket {adm}, "
                               f"eligible {tok < V and bool(w[min(tok, V - 1)] > 0)}")
    _fail(bad, "draws outside the bracket")
    assert n_only_last >= 36, "the masked row's only-last chunk was not exercised"


def _tree(level1_tokens, level2=()):
    """Root 0, level-1 nodes 1..n with the given tokens, level-2 nodes under node 1.  Returns draft_tokens [T],
    retrieve [n_leaf][max_depth] (node ids, -1 padding), candidates (tokens, -1 padding)."""
    draft = [0] + list(level1_tokens) + list(level2)
    n1 = len(level1_tokens)
    rows = [[0, 1, n1 + 1 + j] for j in range(len(level2))] or [[0, 1, -1]]
    rows += [[0, i, -1] for i in range(2, n1 + 1)]
    retrieve = torch.tensor(rows)
    draft_t = torch.tensor(draft)
    cands = torch.where(retrieve >= 0, draft_t[retrieve.clamp(min=0)], torch.full_like(retrieve, -1))
    return draft_t, retrieve, cands


def run_posterior(lib, xd, dtype, V, draft, retrieve, t, p, k, uniforms):
    best, acc, bonus, used = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    u = torch.as_tensor(uniforms, dtype=torch.float32).contiguous()
    check(lib, lib.eb200_k_sample_posterior(DT[dtype], ptr(xd), V, ptr(draft.int().contiguous()), ptr(retrieve.int().contiguous()),
                                            draft.numel(), retrieve.shape[0], retrieve.shape[1], t, p, k, ptr(u), u.numel(),
                                            C.byref(best), C.byref(acc), C.byref(bonus), C.byref(used)))
    return best.value, acc.value, bonus.value, used.value


def _root_row(V, dtype, g, masked_tokens, boost=4.5):
    x = torch.randn(V, generator=g)
    hi = torch.randperm(V, generator=g)[:40]
    x[hi] = boost + torch.rand(40, generator=g)  # a few dozen tokens of real probability: the warpers keep several
    x[list(masked_tokens)] = -math.inf
    return x.to(dtype), hi.tolist()


@pytest.mark.parametrize("temperature,top_p,top_k", [(1.0, 0.0, 0), (0.7, 0.9, 20), (1.3, 0.6, 50), (1.0, 1e-8, 0)])
@pytest.mark.parametrize("V,dtype", [(32000, torch.float16), (128256, torch.bfloat16), (32003, torch.bfloat16)])
def test_posterior_rejecting_every_level1_candidate(lib, V, dtype, temperature, top_p, top_k):
    """u = 1.0 for every level-1 decision: the target's top token, kept tokens and a removed token (p = 0) are all rejected,
    a duplicated token is skipped without a draw, and the bonus comes from what is left."""
    g = torch.Generator().manual_seed(77 + V)
    removed = int(torch.randint(0, V, (1,), generator=g))
    root, hi = _root_row(V, dtype, g, [removed])
    lt_root = sr.temperature_warp(root, temperature)
    top = int(torch.argmax(lt_root))
    kept = [h for h in hi if h != top]
    kept.sort(key=lambda h: -float(lt_root[h]))
    low = int(torch.randint(0, V, (1,), generator=g))
    while low in hi or low in (top, removed):
        low = int(torch.randint(0, V, (1,), generator=g))
    # level 1: top, removed (-inf), a kept token, top again (duplicate node), an ordinary token (removed by top-k / top-p
    # where they are on); node 1 has two level-2 children, so its node is visited twice at level 1 as well
    draft, retrieve, cands = _tree([top, removed, kept[0], top, low], level2=[kept[1], kept[2]])
    T = draft.numel()
    x = torch.cat((root[None], torch.randn(T - 1, V, generator=g).to(dtype)))
    xd = x.cuda()
    thr = torch.tensor(stats(lib, xd, dtype, temperature, top_p, top_k)[:, 2], dtype=torch.float64)
    ref = sr.RowRef(lt_root)
    assert float(thr[0]) in ref.admissible(top_p, top_k), (float(thr[0]), sorted(ref.admissible(top_p, top_k)))
    uniforms = [1.0] * 4 + [0.37]
    w_best, w_acc, w_p, w_used, amb = sr.posterior(sr.temperature_warp(x, temperature), thr, cands, retrieve, uniforms)
    # top-p 1e-8 keeps the maximum only: p(top) = exp(0) / 1 = 1 exactly in fp32 too, accepted even at u = 1
    only_top = int((lt_root >= thr[0]).sum()) == 1
    assert only_top or not amb
    best, acc, bonus, used = run_posterior(lib, xd, dtype, V, draft, retrieve, temperature, top_p, top_k, uniforms)
    assert (best, acc, used) == (w_best, w_acc, w_used)
    ok = sr.bracket(w_p, uniforms[used - 1], sr.cdf_delta_rel(V))
    assert bool(ok[bonus]), f"bonus {bonus} outside the bracket {torch.nonzero(ok).flatten()[:6].tolist()}"
    if only_top:
        assert acc == 1
        return
    # four distinct level-1 tokens, one draw each (the duplicates draw nothing), all rejected; one draw for the bonus
    assert (acc, used) == (0, 5)
    for tok in (top, removed, kept[0], low):
        assert w_p[tok] == 0.0
    assert bonus not in (top, removed, kept[0], low), f"bonus {bonus} is a rejected candidate"


def _equal_mass_buckets(p, n=16):
    """Bucket of every token with p > 0: n buckets of about equal float64 mass in index order."""
    c = torch.cumsum(p, 0) - p / 2
    return torch.clamp((c * n).long(), max=n - 1)


@pytest.mark.parametrize("V,dtype,temperature,top_p,top_k,trials", [(32000, torch.float16, 1.0, 0.0, 0, 20000),
                                                                    (128256, torch.bfloat16, 0.7, 0.9, 20, 20000),
                                                                    (32000, torch.bfloat16, 1.0, 2e-8, 0, 2000)])
def test_first_committed_token_is_distributed_as_the_warped_target(lib, V, dtype, temperature, top_p, top_k, trials):
    """Losslessness at the kernel level: the token committed first (the accepted level-1 candidate, or the bonus token
    when nothing is accepted) follows the warped target distribution, whatever the candidates are.  chi-square over 16
    equal-mass buckets, df <= 15, bound 44.3 (p = 1e-4).  At top_p = 2e-8 only the maximum is kept: every trial must
    commit it."""
    g = torch.Generator().manual_seed(5 + V)
    removed = int(torch.randint(0, V, (1,), generator=g))
    root, hi = _root_row(V, dtype, g, [removed] if top_k == 0 else [], boost=8.0 if top_k == 0 else 4.5)
    lt_root = sr.temperature_warp(root, temperature)
    order = sorted(hi, key=lambda h: -float(lt_root[h]))
    if top_k:
        removed = order[-1]  # outside the top 20
    level1 = [order[0], order[3], removed, order[1], order[3], order[7]]  # kept, removed and a duplicate
    draft, retrieve, cands = _tree(level1, level2=[order[2]])
    T = draft.numel()
    x = torch.cat((root[None], torch.randn(T - 1, V, generator=g).to(dtype)))
    xd = x.cuda()
    thr0 = float(stats(lib, xd, dtype, temperature, top_p, top_k)[0, 2])
    ref = sr.RowRef(lt_root)
    adm = ref.admissible(top_p, top_k)
    p = ref.weights(thr0 if thr0 in adm else min(adm))  # the kernel's threshold is asserted after the trials
    p = p / p.sum()
    assert p[removed] == 0.0
    uniforms = torch.rand(trials, 8, generator=torch.Generator().manual_seed(11))
    counts = torch.zeros(V, dtype=torch.int64)
    t0 = time.perf_counter()
    for i in range(trials):
        best, acc, bonus, _ = run_posterior(lib, xd, dtype, V, draft, retrieve, temperature, top_p, top_k, uniforms[i])
        counts[int(draft[retrieve[best, 1]]) if acc >= 1 else bonus] += 1
    wall = time.perf_counter() - t0
    outside = torch.nonzero((counts > 0) & (p == 0)).flatten().tolist()
    assert not outside, f"tokens outside the kept set were committed: {outside[:10]}"
    b = _equal_mass_buckets(p)
    obs = torch.zeros(16, dtype=torch.float64).index_add_(0, b, counts.double())
    exp = torch.zeros(16, dtype=torch.float64).index_add_(0, b, p * trials)
    used = exp > 0
    chi2 = float(((obs[used] - exp[used]) ** 2 / exp[used]).sum())
    print(f"\nlosslessness V={V} {dtype} T={temperature} top_p={top_p} top_k={top_k}: chi2 = {chi2:.2f} over "
          f"{int(used.sum())} buckets, {trials} trials in {wall:.1f} s")
    assert chi2 < 44.3, (chi2, obs[used].tolist(), exp[used].tolist())
    assert thr0 in adm, (thr0, sorted(adm)[:4])

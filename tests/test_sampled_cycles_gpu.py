"""Sampled decoding cycle by cycle: every decision of the engine against a float64 posterior evaluated on the engine's OWN
verify logits, and those logits, the draft trees and the committed KV against a shadow of the CPU oracle driven by the engine's
decisions.

Why not token parity with the oracle: a bf16 logit near 12 carries an ulp of 0.06, which moves an acceptance probability by
several percent, so two correct implementations sharing one uniform stream part ways within a few cycles.  Instead each cycle
is checked in two halves:

* decisions -- the stats kernel's thresholds on the engine's verify logits (model dtype, read back exactly) must be admissible
  for the float64 reference (tests/sampling_ref.py); tests/sampling_ref.posterior on those rows, with the injected uniforms
  from the cursor the previous cycles left, must give the engine's (best, accept_length) exactly, its committed tokens, and a
  bonus token inside the inverse-CDF bracket of the uniform it drew.  The cursor advances by the uniforms the reference used,
  so a cursor that drifts, a bonus drawn from the wrong node's residual, or verify rows out of node order show up as a wrong
  decision in a later cycle;
* state -- the shadow oracle (tests/sampled_cycles_ref.py) verifies over the engine's tree, so its logits align row for row
  with the engine's: every row within relative L2 distance 0.05 (a wrong row, position or stale KV row moves a row by O(1)).
  It then compacts its KV with the engine's decisions and grows its own sampling-mode tree, whose top-score chain the
  engine's next tree must contain wherever the chain's scores clear the selection cut-offs by more than rounding.  After the run the committed target KV is held to the shadow's and to a fresh engine that
  prefills the committed ids (tests/test_prefill_gpu.py's bars), eagenerate must reproduce the stepwise ids from the same
  uniform stream (captured graph and the asynchronous cycle pipeline), and an engine called with another warper in between
  must still match.

Each case must exercise a rejection followed by an acceptance in one level, an empty accept with a residual bonus, and an
accept of two or more tokens, where its fixture can reach them (CASES says which cannot and why).  The uniform streams are
seeded and were picked on the H100 to reach those paths; decisions within rounding distance of a threshold fail the case
(none occur with these seeds)."""
import ctypes as C

import numpy as np
import pytest
import torch

from eagle_b200 import static_trees
from oracle import eagle_oracle as orc
from tests import sampling_ref as sr
from tests.fixtures import report, to_cfg
from tests.sampled_cycles_ref import Shadow, certain_chain, top_score_chain, tree_paths
from tests.test_prefill_gpu import kv_bars, planes, target_rope_terms
from tests.test_tree_geometry_gpu import DEEP, ULP, engine, prompt_of, tid, weights

pytestmark = pytest.mark.gpu

N_UNIFORMS = 4096  # eb200_set_uniforms' capacity
DT = {torch.bfloat16: 0, torch.float16: 1}
OTHER_WARPER = dict(temperature=3.0, top_p=0.95, top_k=50)  # hot: its output differs from every case's
# cumulative draft scores are log-probabilities summed in the model dtype (bf16 spacing 0.125 at 16..32): a node whose score
# clears the tree's and its level's cut-offs by this much is in the engine's tree whatever the rounding
CHAIN_MARGIN = 0.5


def sample_stats(lib, x, temperature, top_p, top_k):
    """eb200_k_sample_stats on model-dtype rows [R, V]: float64 thresholds [R]."""
    xd = x.contiguous().cuda()
    out = np.zeros((x.shape[0], 3), dtype=np.float32)
    torch.cuda.synchronize()
    rc = lib.eb200_k_sample_stats(DT[x.dtype], C.c_void_p(xd.data_ptr()), x.shape[0], x.shape[1], temperature, top_p, top_k,
                                  out.ctypes.data_as(C.c_void_p))
    assert rc == 0, lib.eb200_last_error().decode()
    return torch.from_numpy(out[:, 2].astype(np.float64))


def sampled_prefill(m, prompt, gen, new_tokens, max_length):
    """eb200_prefill in sampling mode (EaModel.prefill is the greedy one): the first token."""
    from eagle_b200 import _lib
    ids = prompt.to(torch.int64).contiguous()
    gp = m._gen_params(gen["temperature"], gen.get("top_p", 0.0), gen.get("top_k", 0), new_tokens, max_length, False)
    first = C.c_int64()
    _lib.check(m.lib.eb200_prefill(m._h, ids.data_ptr(), ids.shape[1], C.byref(gp), C.byref(first)))
    return int(first.value)


def check_thresholds(lt, thr, nodes, top_p, top_k, what):
    for node in nodes:
        adm = sr.RowRef(lt[node]).admissible(top_p, top_k)
        assert float(thr[node]) in adm, f"{what}: threshold of node {node} {float(thr[node])!r} not admissible {sorted(adm)[:4]}"


def run_sampled_case(m, ref, prompt, gen, what, new_tokens=40, max_length=512, uniform_seed=0, fresh=None, min_cycles=1,
                     cover=("rej_then_acc", "empty_residual", "acc2")):
    """The harness.  m: engine; ref: OracleEaModel of the same weights and tree; gen: temperature / top_p / top_k; fresh: a
    callable building another engine of the same weights (the committed-KV and warper checks); cover: the paths the run must
    exercise (a rejection followed by an acceptance in one level, an empty accept with a residual bonus, an accept of two or
    more tokens).  Returns the report dict."""
    from eagle_b200 import _lib
    lib = _lib.load()
    temperature, top_p, top_k = gen["temperature"], gen.get("top_p", 0.0), gen.get("top_k", 0)
    V, dtype, T = m.vocab_size, m.dtype, m._cfg.total_token
    uniforms = torch.rand(N_UNIFORMS, generator=torch.Generator().manual_seed(uniform_seed)).tolist()  # exact fp32 values
    P = prompt.shape[1]
    m.set_uniforms(uniforms)
    first = sampled_prefill(m, prompt, gen, new_tokens, max_length)

    # ---- first token: row 0 of the verify logits holds the prefill's last-row logits
    x0 = m.debug_read("verify_logits")[:1, :V].to(dtype)
    lt0 = sr.temperature_warp(x0, temperature)
    thr0 = sample_stats(lib, x0, temperature, top_p, top_k)
    check_thresholds(lt0, thr0, [0], top_p, top_k, f"{what} first token")
    w0 = sr.RowRef(lt0[0]).weights(float(thr0[0]))
    ok = sr.bracket(w0, uniforms[0], sr.cdf_delta_rel(V))
    assert bool(ok[first]), f"{what}: first token {first} outside the bracket {torch.nonzero(ok).flatten()[:6].tolist()}"
    shadow = Shadow(ref, sampling=True)
    want0 = shadow.prefill(prompt, max_length).float()
    d0 = float((x0[0].float() - want0).norm() / want0.norm())
    assert d0 < 0.05, f"{what}: prefill logits row at relative distance {d0:.4f} from the oracle's"
    shadow.first_token(first)

    offset, ids, new_token = 1, prompt[0].tolist(), 0
    limit = max_length - (T - 1) - 10
    accs, used_per_cycle, n_rej, n_residual, n_rej_then_acc, n_empty_residual = [], [], 0, 0, 0, 0
    worst_row, worst_elem, shared_nodes, chain_found, chain_len, chain_certain = d0, 0.0, [], [], [], []
    while True:
        c = len(accs)
        dt, ri, tm, tp = m.get_tree()
        # the oracle's tree, grown from the same decisions: its top-score chain is in the engine's tree as far as the chain's
        # scores clear the selection cut-offs by CHAIN_MARGIN (below that a rounding-level tie may pick another node; the
        # chain is then followed further and what is found is reported)
        paths = set(tree_paths(dt, tm))
        chain = top_score_chain(shadow.tree[0], shadow.tree[2])
        certain = certain_chain(shadow.tree[0], shadow.tree[2], shadow.scores, CHAIN_MARGIN)
        missing = [p for p in certain if p not in paths]
        assert not missing, f"{what} cycle {c}: the engine's tree lacks the oracle's top-score chain node {missing[0]}"
        chain_found.append(next((i for i, p in enumerate(chain) if p not in paths), len(chain)))
        chain_len.append(len(chain))
        chain_certain.append(len(certain))
        shared_nodes.append(len(paths & set(tree_paths(shadow.tree[0], shadow.tree[2]))))
        toks, nxt = m.step()
        _, best, acc, n = m.get_verify()
        x = m.debug_read("verify_logits")[:, :V].to(dtype)
        assert x.shape[0] == T

        # ---- decisions against the float64 posterior on the engine's own logits
        lt = sr.temperature_warp(x, temperature)
        thr = sample_stats(lib, x, temperature, top_p, top_k)
        cands = torch.cat((dt, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, ri]
        draws = []
        w_best, w_acc, w_p, used, amb = sr.posterior(lt, thr, cands, ri, uniforms[offset:], draws=draws)
        assert not amb, f"{what} cycle {c}: a decision lies within rounding distance of its acceptance probability"
        assert (best, acc) == (w_best, w_acc), f"{what} cycle {c}: (best, accept_length) ({best}, {acc}), reference ({w_best}, {w_acc})"
        check_thresholds(lt, thr, ri[best, : acc + 1].tolist(), top_p, top_k, f"{what} cycle {c}")
        assert toks == cands[best, : acc + 1].tolist(), f"{what} cycle {c}: committed tokens {toks}"
        ok = sr.bracket(w_p, uniforms[offset + used - 1], sr.cdf_delta_rel(V))
        assert bool(ok[nxt]), f"{what} cycle {c}: bonus {nxt} outside the bracket {torch.nonzero(ok).flatten()[:6].tolist()}"
        offset += used
        assert offset < N_UNIFORMS, f"{what}: the run needs more than {N_UNIFORMS} uniforms"
        ids += toks
        assert n == len(ids), f"{what} cycle {c}: committed length {n}, expected {len(ids)}"
        residual = bool(draws) and not draws[-1][1]
        n_rej += sum(1 for _, a in draws if not a)
        n_residual += residual
        n_rej_then_acc += sum(1 for (la, a), (lb, b) in zip(draws, draws[1:]) if la == lb and not a and b)
        n_empty_residual += acc == 0 and residual
        accs.append(acc)
        used_per_cycle.append(used)

        # ---- state: the shadow oracle verifies the engine's tree and takes the engine's decisions
        want = shadow.verify(dt, tm, tp).float()
        got = x.float()
        d = (got - want).norm(dim=-1) / want.norm(dim=-1).clamp_min(1e-6)
        assert float(d.max()) < 0.05, f"{what} cycle {c}: verify logits rows {(d >= 0.05).nonzero().flatten()[:8].tolist()} differ from the oracle's"
        worst_row = max(worst_row, float(d.max()))
        worst_elem = max(worst_elem, float(((got - want).abs() / (1e-3 + 2 * ULP[dtype] * want.abs())).max()))
        shadow.commit(dt, ri, best, acc, nxt)
        assert shadow.ids[0].tolist() == ids

        new_token += acc + 1
        if new_token > new_tokens or len(ids) > limit:
            break

    # ---- committed target KV against the shadow oracle's and a fresh prefill's
    n = len(ids)
    ids_t = torch.tensor([ids])
    nkv = ref.target.cfg.num_key_value_heads
    kv = planes(m, "target_kv", n)
    want_kv = shadow.kv.data[:, 0, :, :n].float().reshape(-1, n, 128)
    terms = target_rope_terms(ref, ids_t)
    f_or, rows_or, worst_or = kv_bars(kv, want_kv, 2 * nkv, dtype, "committed target KV vs the oracle", terms)
    fails = list(f_or)
    kv_fresh = None
    if fresh is not None:
        f = fresh()
        # a fresh engine's first sampled call, with the other warper (compared below with the same call on the used engine)
        f.set_uniforms(uniforms)
        other_fresh = f.eagenerate(prompt.cuda(), max_new_tokens=new_tokens, max_length=max_length, **OTHER_WARPER).cpu()
        f.prefill(ids_t.cuda())
        f_fr, rows_fr, worst_fr = kv_bars(kv, planes(f, "target_kv", n), 2 * nkv, dtype, "committed target KV vs a fresh prefill", terms)
        fails += f_fr
        kv_fresh = float(rows_fr.max())
        del f
    assert not fails, f"{what}: " + "; ".join(fails)

    # ---- eagenerate from the same uniform stream: the captured graph and the asynchronous pipeline give the stepwise ids
    m.set_uniforms(uniforms)
    a1, w_new, w_idx = m.eagenerate(prompt.cuda(), max_new_tokens=new_tokens, max_length=max_length, log=True, **gen)
    assert a1[0].cpu().tolist() == ids, f"{what}: eagenerate differs from the stepwise run"
    assert (w_new, w_idx) == (new_token, len(accs) - 1)
    if fresh is not None:
        # warper A, then B, then A on one engine: no captured sampling parameter may survive a call
        other = m.eagenerate(prompt.cuda(), max_new_tokens=new_tokens, max_length=max_length, **OTHER_WARPER).cpu()
        assert other.tolist() == other_fresh.tolist(), f"{what}: warper B after A differs from a fresh engine's"
        assert other.tolist() != a1.cpu().tolist(), f"{what}: the second warper must change the output to discriminate"
        a2 = m.eagenerate(prompt.cuda(), max_new_tokens=new_tokens, max_length=max_length, **gen).cpu()
        assert a2[0].tolist() == ids, f"{what}: warper A after B differs from the first call"

    rep = dict(cycles=len(accs), accs=accs, rejections=n_rej, residual_bonuses=n_residual, uniforms=offset,
               worst_row=worst_row, worst_elem=worst_elem, kv_oracle=float(rows_or.max()), kv_oracle_layer0=worst_or,
               kv_fresh=kv_fresh, shared=min(shared_nodes), rej_then_acc=n_rej_then_acc, empty_residual=n_empty_residual,
               chain=f"{sum(chain_found)}/{sum(chain_len)}", chain_asserted=sum(chain_certain))
    report(f"sampled cycles {what}: {len(accs)} cycles, accept lengths {accs}; {n_rej} rejections, {n_residual} residual bonuses; "
           f"{offset} uniforms used; verify logits worst row distance {worst_row:.4f}, worst element {worst_elem:.2f} x (1e-3 + 2 ulp); "
           f"committed KV worst row distance {rep['kv_oracle']:.4f} to the oracle (layer 0 {worst_or:.2f} x bar), "
           f"{kv_fresh if kv_fresh is None else round(kv_fresh, 4)} to a fresh prefill; fewest shared tree nodes {rep['shared']}, "
           f"oracle top-score chain nodes found {rep['chain']} ({rep['chain_asserted']} asserted); {n_rej_then_acc} rejections followed by an acceptance, "
           f"{n_empty_residual} empty accepts with a residual bonus")
    print("\n" + f"{what}: {rep}")
    assert len(accs) >= min_cycles, f"{what}: only {len(accs)} cycles"
    assert "rej_then_acc" not in cover or n_rej_then_acc >= 1, f"{what}: no rejection followed by an acceptance"
    assert "empty_residual" not in cover or n_empty_residual >= 1, f"{what}: no empty accept with a residual bonus: {accs}"
    assert "acc2" not in cover or max(accs) >= 2, f"{what}: no accept of two or more tokens: {accs}"
    return rep


ALL = ("rej_then_acc", "empty_residual", "acc2")
CASES = [
    # name, fixture, tree (None: the fixture's own), sampling settings, uniform seed, paths the run must exercise.  Two fixtures
    # cannot reach all three: the random weights of e3_rand_bf16 give the draft's candidates no target mass at top_k 20 of 1024,
    # so every cycle ends in a residual bonus (24 of 24 seeds tried); at T = 1, top_k = 5 the sharp e3_gqa_bf16 target keeps a
    # single token of real mass, so its decisions are the same for every uniform stream and no level accepts after a rejection.
    ("corr-T2", "e3_corr_bf16", None, dict(temperature=2.0), 12, ALL),
    ("corr-deep-T2", "e3_corr_bf16", DEEP, dict(temperature=2.0), 8, ALL),
    ("e1-T15-p09", "e1_corr_fp16", None, dict(temperature=1.5, top_p=0.9), 24, ALL),
    ("rand-T07-p09-k20", "e3_rand_bf16", None, dict(temperature=0.7, top_p=0.9, top_k=20), 4, ("empty_residual",)),
    ("gqa-T1-k5", "e3_gqa_bf16", None, dict(temperature=1.0, top_k=5), 5, ("empty_residual", "acc2")),
    ("corr-static-T2", "e3_corr_bf16", "static", dict(temperature=2.0), 2, ALL),
]


@pytest.mark.parametrize("name,base,tree,gen,seed,cover", CASES, ids=[c[0] for c in CASES])
def test_sampled_cycles_against_the_float64_posterior_and_the_oracle(name, base, tree, gen, seed, cover):
    from eagle_b200.synthetic import fixture_models
    w = weights(base)
    tcfg, tW, hcfg, hW, eagle3, dtype = w
    if tree == "static":
        kw = dict(top_k=10, tree_choices=static_trees.mc_sim_7b_63)
        oref = dict(top_k=10, tree_choices=[list(c) for c in static_trees.mc_sim_7b_63])
    else:
        kw = dict(tree if tree is not None else fixture_models(base)[6])
        oref = kw
    make = lambda: engine(w, {}, **kw)  # noqa: E731
    ref = orc.OracleEaModel(to_cfg(tcfg), tW, to_cfg(hcfg), hW, eagle3, **oref)
    run_sampled_case(make(), ref, prompt_of(base, w), gen, f"{name} ({base} {tid(kw) if 'total_token' in kw else 'mc_sim_7b_63'})",
                     uniform_seed=seed, fresh=make, cover=cover)

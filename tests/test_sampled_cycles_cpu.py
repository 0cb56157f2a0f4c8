"""The shadow cycle of tests/sampled_cycles_ref.py against OracleEaModel.eagenerate itself.

tests/test_sampled_cycles_gpu.py runs the oracle's cycle body with the ENGINE's decisions (best candidate, accept length, bonus
token) to keep the oracle's KV and draft tree in step with the engine.  That is only a reference if the split body, fed the
oracle's own decisions, is the oracle: same seeded `rand` stream for the posterior, same torch.multinomial call order, and then
identical ids, (new_token, idx) and cycle records."""
import random

import pytest
import torch

from eagle_b200.synthetic import FIXTURES, make_prompt
from oracle import eagle_oracle as orc
from tests.fixtures import build_oracle
from tests.sampled_cycles_ref import Shadow, top_score_chain, tree_paths


def shadow_generate(ref, prompt, temperature, top_p, top_k, max_new_tokens, max_length, rand):
    warp = lambda lg: orc.warp_logits(lg, temperature, top_p, int(top_k))  # noqa: E731
    sh = Shadow(ref, sampling=True)
    last = sh.prefill(prompt, max_length)
    token = torch.multinomial(torch.softmax(warp(last[None]), dim=1), 1)
    sh.first_token(int(token))
    records, new_token, idx = [], 0, 0
    limit = max_length - ref.head.total_tokens - 10
    for idx in range(limit):
        dt, ri, tm, tp = sh.tree
        tree_logits = sh.verify(dt, tm, tp)
        cands = torch.cat((dt, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, ri]
        best, acc, sample_p = orc.evaluate_posterior_sampling(tree_logits[ri], cands, warp, rand)
        token = torch.multinomial(sample_p, 1)[None]
        records.append(dict(draft_tokens=dt.clone(), retrieve=ri.clone(), tree_mask=tm.clone(), tree_pos=tp.clone(),
                            node_argmax=torch.argmax(tree_logits, dim=-1), best=int(best), accept_length=int(acc), bonus=int(token)))
        sh.commit(dt, ri, int(best), int(acc), int(token))
        new_token += int(acc) + 1
        if new_token > max_new_tokens or sh.ids.shape[1] > limit:
            break
    return sh.ids, new_token, idx, records


@pytest.mark.parametrize("fx", ["e3_corr_bf16", "e1_corr_fp16"])
def test_shadow_cycle_reproduces_the_oracle(fx):
    ref, (tcfg, *_rest) = build_oracle(fx)
    plen, pseed, _, _ = FIXTURES[fx]
    prompt = make_prompt(tcfg["vocab_size"], plen, pseed)
    gen = dict(temperature=2.0, top_p=0.0, top_k=0, max_new_tokens=40, max_length=512)
    ref.cycle_log = []
    torch.manual_seed(3)
    want, w_new, w_idx = ref.eagenerate(prompt, log=True, rand=random.Random(5).random, **gen)
    log, ref.cycle_log = ref.cycle_log, None
    torch.manual_seed(3)
    ids, new_token, idx, records = shadow_generate(ref, prompt, rand=random.Random(5).random, **gen)
    assert ids.tolist() == want.tolist()
    assert (new_token, idx) == (w_new, w_idx)
    assert len(records) == len(log)
    for c, (got, rec) in enumerate(zip(records, log)):
        for k, v in rec.items():
            same = torch.equal(got[k], v) if torch.is_tensor(v) else got[k] == v
            assert same, f"cycle {c}: {k} differs"
    accs = [r["accept_length"] for r in log]
    # at T = 2 the run is no longer the greedy one: empty and multi-token accepts both occur
    assert min(accs) == 0 and max(accs) >= 2, accs


def test_top_score_chain_follows_first_children():
    # root 0; level 1: nodes 1, 2 (children of 0); level 2: 3 (child of 2), 4 (child of 1), 5 (child of 1)
    parent = [-1, 0, 0, 2, 1, 1]
    T = len(parent)
    m = torch.eye(T)
    for i in range(1, T):
        m[i] += m[parent[i]]
    dt = torch.tensor([[7, 11, 12, 13, 14, 15]])
    assert top_score_chain(dt, m[None, None]) == [(7,), (7, 11), (7, 11, 14)]
    assert tree_paths(dt, m)[3] == (7, 12, 13)

"""The fp16 EAGLE-1 configurations at model width: Llama-2-13B (benchmark configuration 3, sampled at temperature 1) and
Vicuna-7B (configuration 0, greedy), each with two target layers, against the CPU oracle.

These run what no fixture reaches: fp16 at H = 4096 / 5120, MHA with 32 / 40 kv heads, I = 11008 / 13824, rope theta 1e4,
V = 32000, and an EAGLE-1 head (fc over 2H with bias) whose draft reads the target lm_head.  The weights are
eagle_b200.synthetic.correlated_llama2_eagle1's: a permutation-bigram target and a copy head wrong after a quarter of the
tokens.  The engines are loaded the way from_pretrained loads a checkpoint, with the head's own embed_tokens
(load_emb_from_target=False), which is what makes the draft wrong where its table is rotated.  A 300-token prompt runs as a
256-row and a 44-row prefill chunk.  Each test builds its own weights and frees them with its engines at its end; at most two
engines are alive at once (the harness's fresh engine next to the one under test)."""
import pytest
import torch

from eagle_b200.synthetic import make_prompt
from oracle import eagle_oracle as orc
from tests.fixtures import report, to_cfg
from tests.test_prefill_gpu import kv_bars, planes, target_rope_terms
from tests.test_sampled_cycles_gpu import run_sampled_case
from tests.test_tree_geometry_gpu import compare_cycles, frontier_logits_bar

pytestmark = pytest.mark.gpu

TREE = dict(total_token=60, depth=6, top_k=10)
P, MAX_LEN = 300, 512
DTYPE = torch.float16


def pair(name, head_scale=None, seed=30):
    """(make_engine, oracle, prompt): make_engine builds an engine from the device copies of the weights."""
    from eagle_b200 import EaModel, synthetic as syn
    tcfg, tW, hcfg, hW = syn.correlated_llama2_eagle1(name, 2, DTYPE, "cuda", head_scale=head_scale, seed=seed)

    def make():
        m = EaModel(tcfg, hcfg, use_eagle3=False, torch_dtype=DTYPE, max_length=MAX_LEN, **TREE)
        m.load_target_state_dict(tW)
        m.load_head_state_dict(hW, load_emb_from_target=False)  # the head's own (partly rotated) table, as from_pretrained
        return m.finalize()

    ref = orc.OracleEaModel(to_cfg(tcfg), {k: v.cpu() for k, v in tW.items()}, to_cfg(hcfg), {k: v.cpu() for k, v in hW.items()},
                            False, **TREE)
    return make, ref, make_prompt(tcfg["vocab_size"], P, seed + 3)


def test_llama2_13b_shape_sampled_cycles():
    """Configuration 3 on one GPU: a soft target sampled at temperature 1, run through the whole sampled-cycle harness of
    tests/test_sampled_cycles_gpu.py for at least 16 cycles.  head_scale 30 / H: at this width the two random layers add about
    as much to the residual stream as the embedding carries, which lowers the bigram logit below head_scale * H; 30 / H puts the
    target's top-1 mass near 0.8 at T = 1, so most cycles accept draft tokens (up to the full depth) and about a third end in a
    residual bonus.  A rejection followed by an acceptance in one level cannot occur here: after the draft's top candidate the
    others carry target mass of the order of 1e-5 each (the remaining 0.2 spread over 32000 tokens)."""
    make, ref, prompt = pair("llama2-13b", head_scale=30.0 / 5120)
    m = make()
    run_sampled_case(m, ref, prompt, dict(temperature=1.0), "llama2-13b width fp16 T=1", new_tokens=96, max_length=MAX_LEN,
                     uniform_seed=13, fresh=make, min_cycles=16, cover=("empty_residual", "acc2"))
    del m, make, ref
    torch.cuda.empty_cache()


def test_vicuna_7b_shape_greedy():
    """Configuration 0: greedy cycles identical to the oracle (ids, accept lengths, committed tokens, verify arg-max of the
    shared nodes), the prefill K/V within tests/test_prefill_gpu.py's bars, and the last tree level's draft logits (the target
    lm_head over the EAGLE-1 head's output) within 1e-3 + one fp16 ulp, paired by row as in tests/test_tree_geometry_gpu.py."""
    make, ref, prompt = pair("vicuna-7b")
    m = make()
    accs, n_cmp = compare_cycles(m, ref, prompt, TREE, "vicuna-7b width fp16 greedy", new_tokens=48, max_length=MAX_LEN)
    assert max(accs) >= 2 and min(accs) <= 1, f"the rotated head rows must make accept lengths vary: {accs}"

    # ---- prefill K/V
    kv = ref._kv(MAX_LEN)
    ref.target.forward(prompt, kv)
    want = kv.data[:, 0, :, :P].float().reshape(-1, P, 128)
    m.prefill(prompt.cuda())
    fails, rows, worst_kv = kv_bars(planes(m, "target_kv", P), want, 2 * ref.target.cfg.num_key_value_heads, DTYPE, "target KV",
                                    target_rope_terms(ref, prompt))
    assert not fails, "; ".join(fails)

    # ---- last-level draft logits after one cycle
    ref.head.trace = {}
    ref.eagenerate(prompt, max_new_tokens=0, max_length=MAX_LEN, log=True)
    want = ref.head.trace["level_raw"][-1].float()
    ref.head.trace = None
    k = TREE["top_k"]
    m.prefill(prompt.cuda())
    m.step()
    got = m.debug_read("draft_logits")[:k]
    assert got.shape == want.shape
    pairs, n_bad, n_all, worst = frontier_logits_bar(got, want, DTYPE)
    assert len(pairs) >= 3, f"only {len(pairs)} of {k} frontier rows are fed the same node in both implementations"
    report(f"vicuna-7b width fp16 greedy: accept lengths {accs}, {n_cmp} verify nodes compared; prefill KV worst row distance "
           f"{float(rows.max()):.4f}, layer 0 {worst_kv:.2f} x bar; last-level draft logits {len(pairs)} rows, {n_bad}/{n_all} beyond "
           f"1e-3 + 1 ulp, worst {worst:.2f} x")
    assert n_bad <= n_all * 1e-3 and worst <= 3.0, f"{n_bad}/{n_all} draft logits beyond 1e-3 + 1 ulp; worst {worst:.2f}x"
    del m, make, ref
    torch.cuda.empty_cache()

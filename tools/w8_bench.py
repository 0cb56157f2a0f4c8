#!/usr/bin/env python
"""Int8 target weights (load_in_8bit) vs bf16 on bench.py's headline workload, in one process on one GPU.

Workload: Llama-3-8B shapes + EAGLE-3 head, bf16, 512-token prompt, 256 new tokens, greedy, dynamic tree (total_token=60,
depth=6, top_k=10); random-init (default) or `--fixture correlated` weights, generated exactly like bench.py.  Two engines
are built from the same weights: an int8 engine (the target's decoder projections as int8 + fp32 row scales) and a bf16
engine loaded with W' = dequantize(quantize(W)), the values the int8 engine multiplies by.  So the two must produce identical
ids, which the run checks on the timed calls themselves.

Timing: after warm-up, `--rounds` rounds of one `--steps`-call window per engine, alternating which engine goes first, each
window timed with CUDA events on the engine's stream (bench.timed_steps).  Prefill is timed separately (3 prefills).
A separate profiled pass (per-launch CUDA events) gives the verify GEMMs' achieved bytes/s and their share of 3.35 TB/s.
Bytes are algorithmic: every weight once per verify pass, the head once per draft pass (bench.weight_bytes_per_cycle);
int8 projections count 1 byte per weight plus 4 bytes per row.  The card's name and power limit are read in the same run.

    python tools/w8_bench.py [--fixture random|correlated] [--rounds 3] [--steps 2] [--warmup 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from eagle_b200 import EaModel, quant, synthetic as syn  # noqa: E402

HBM_PEAK_GBS = 3350.0  # NVIDIA H100 SXM data sheet


def log(msg):
    print(f"[w8_bench] {msg}", file=sys.stderr, flush=True)


def card():
    q = "name,power.limit,power.max_limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, plim, pmax, smmax = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "power_max_limit": pmax, "sm_max_clock": smmax}
    except Exception as ex:  # the numbers below are then reported without their context
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def target_weights(args, tcfg, hcfg, dev):
    """(name, tensor) of the target and the head, generated like bench.build_engine (random: streamed per tensor)."""
    dtype = torch.bfloat16
    if args.fixture == "correlated":
        _, tW, _, hW = syn.correlated_llama3_eagle3(tcfg["num_hidden_layers"], dtype, dev)
        for k in list(tW):
            yield k, tW.pop(k)
        for k in list(hW):
            w = hW.pop(k)
            if k not in ("embed_tokens.weight", "t2d"):  # as EaModel.load_head_state_dict: the head embeds with the target's table
                yield "head." + k, w
        return
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    for which, name, shape, kind in bench.weight_specs(tcfg, hcfg, True):
        if kind == "normal":
            w = (torch.randn(shape, generator=gen, device=dev, dtype=torch.float32) * 0.02).to(dtype)
        else:
            w = torch.ones(shape, dtype=dtype, device=dev) if kind == "ones" else torch.zeros(shape, dtype=dtype, device=dev)
        yield (name if which == "t" else "head." + name), w
    d2t, _ = syn.make_d2t(tcfg["vocab_size"], hcfg["draft_vocab_size"])
    yield "head.d2t", d2t


def build_pair(args):
    tcfg, hcfg, _ = bench.model_configs(argparse.Namespace(model="llama3-8b", layers=0))
    if args.fixture == "correlated":
        hcfg = syn.head_config("llama3-8b", True, draft_vocab_size=32000, num_key_value_heads=tcfg["num_attention_heads"])
    kw = dict(use_eagle3=True, torch_dtype=torch.bfloat16, device=0, max_length=2048, **bench.TREE)
    m8 = EaModel(tcfg, hcfg, load_in_8bit=True, **kw)
    mb = EaModel(tcfg, hcfg, **kw)
    for name, w in target_weights(args, tcfg, hcfg, "cuda:0"):
        if quant.is_target_projection(name):
            q, scb = quant.quantize_int8_rowwise(w)
            m8._load(name, q)
            m8._load(name[: -len("weight")] + "SCB", scb)
            mb._load(name, quant.dequantize_int8_rowwise(q, scb, torch.bfloat16))
        else:
            m8._load(name, w)
            mb._load(name, w)
        del w
    torch.cuda.empty_cache()
    return m8.finalize(), mb.finalize(), tcfg, hcfg


def bytes_per_cycle(tcfg, hcfg, int8):
    """Algorithmic weight bytes of one cycle (bench.weight_bytes_per_cycle), with int8 projections at 1 B/weight + 4 B/row."""
    cyc, verify = bench.weight_bytes_per_cycle(tcfg, hcfg, True, bench.TREE["depth"])
    if not int8:
        return cyc, verify
    saved = 0
    for which, name, shape, kind in bench.weight_specs(tcfg, hcfg, True):
        if which == "t" and quant.is_target_projection(name):
            saved += shape[0] * shape[1] - 4 * shape[0]
    return cyc - saved, verify - saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fixture", default="random", choices=["random", "correlated"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="eagenerate calls per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("w8_bench.py: no CUDA device (eagle_b200 has no CPU path)")
    torch.cuda.set_device(0)
    info = card()
    log(f"card: {info}")
    log(f"building the int8 and the bf16-on-W' engines ({args.fixture} weights)")
    m8, mb, tcfg, hcfg = build_pair(args)
    engines = {"int8": m8, "bf16": mb}
    V = tcfg["vocab_size"]
    if args.fixture == "correlated":
        used = syn.draft_vocab_ids(V, 32000)
        prompt = used[torch.randint(0, used.numel(), (bench.PROMPT_LEN,), generator=torch.Generator().manual_seed(0))][None].cuda()
    else:
        prompt = torch.randint(0, V - 200, (1, bench.PROMPT_LEN), generator=torch.Generator().manual_seed(0)).cuda()
    for name, m in engines.items():
        for _ in range(max(1, args.warmup)):
            m.eagenerate(prompt, max_new_tokens=bench.NEW_TOKENS, max_length=2048)
    acc = {k: dict(ms=0.0, new=0, cycles=0, windows=[]) for k in engines}
    last = {}
    for r in range(args.rounds):
        order = ["int8", "bf16"] if r % 2 == 0 else ["bf16", "int8"]
        for name in order:
            ms, new, cyc, lst = bench.timed_steps(engines[name], prompt, args.steps, None, {})
            a = acc[name]
            a["ms"] += ms
            a["new"] += new
            a["cycles"] += cyc
            a["windows"].append(round(new / (ms / 1e3), 2))
            last[name] = lst
        log(f"round {r}: " + ", ".join(f"{k} {acc[k]['windows'][-1]} tok/s" for k in engines))
    parity = (last["int8"][0].cpu().tolist() == last["bf16"][0].cpu().tolist() and last["int8"][1:] == last["bf16"][1:])
    res = {}
    for name, m in engines.items():
        stream = m.cuda_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        for _ in range(3):
            m.prefill(prompt)
        e1.record(stream)
        torch.cuda.synchronize()
        prefill_ms = e0.elapsed_time(e1) / 3
        a = acc[name]
        steps = args.rounds * args.steps
        cycle_ms = (a["ms"] / steps - prefill_ms) / max(1.0, a["cycles"] / steps)
        cyc_bytes, verify_bytes = bytes_per_cycle(tcfg, hcfg, name == "int8")
        m.reset_stats()
        m.set_profiling(True)
        for _ in range(2):
            m.eagenerate(prompt, max_new_tokens=bench.NEW_TOKENS, max_length=2048)
        ps = m.stats()
        m.set_profiling(False)
        vach = ps["verify_gemm_bytes"] / 1e9 / (ps["verify_gemm_ms"] / 1e3) if ps["verify_gemm_ms"] > 0 else 0.0
        res[name] = {"tok_s": round(a["new"] / (a["ms"] / 1e3), 2), "tok_s_windows": a["windows"], "ms_per_cycle": round(cycle_ms, 3),
                     "tau": round(a["new"] / max(1, a["cycles"]), 3), "prefill_ms": round(prefill_ms, 3),
                     "bytes_per_cycle_gb": round(cyc_bytes / 1e9, 3), "verify_bytes_per_cycle_gb": round(verify_bytes / 1e9, 3),
                     "verify_gemm": {"achieved_gbs": round(vach, 1), "share_of_3350_gbs": round(vach / HBM_PEAK_GBS, 4),
                                     "ms_per_cycle": round(ps["verify_gemm_ms"] / max(1, ps["cycles"]), 3),
                                     "how": "per-launch CUDA events in 2 profiled (eager) eagenerate calls after the timed rounds"}}
    line = {"tool": "w8_bench", "workload": f"llama3-8b+eagle3 bf16 bs1 {bench.PROMPT_LEN}in/{bench.NEW_TOKENS}out greedy "
                                            f"dynamic-tree(60,6,10) {args.fixture}-init",
            "card": info, "rounds": args.rounds, "steps_per_window": args.steps, "ids_identical_int8_vs_bf16_on_Wprime": parity,
            "int8": res["int8"], "bf16": res["bf16"], "speedup_tok_s": round(res["int8"]["tok_s"] / res["bf16"]["tok_s"], 4)}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")
    if not parity:
        raise SystemExit("w8_bench.py: the int8 engine's ids differ from the bf16 engine's on W'")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Int8 (load_in_8bit), 4-bit (nf4 / fp4) or FP8 (FineGrainedFP8Config) target weights vs bf16 on bench.py's headline workload, in one process on one GPU.

Workload: Llama-3-8B shapes + EAGLE-3 head, bf16, 512-token prompt, 256 new tokens, greedy, dynamic tree (total_token=60,
depth=6, top_k=10); random-init (default) or `--fixture correlated` weights, generated exactly like bench.py.  Two engines
are built from the same weights: a quantized engine (the target's decoder projections as int8 + fp32 row scales, or with
`--quant nf4|fp4` as bitsandbytes 4-bit codes + fp32 absmax per 64 weights, with `--quant fp8` as float8_e4m3fn + one fp32
scale per 128 x 128 block) and a bf16 engine loaded with
W' = dequantize(quantize(W)), the values the quantized engine multiplies by.  So the two must produce identical ids, which the
run checks on the timed calls themselves.

Timing: after warm-up, `--rounds` rounds of one `--steps`-call window per engine, alternating which engine goes first, each
window timed with CUDA events on the engine's stream (bench.timed_steps).  Prefill is timed separately (3 prefills).
A separate profiled pass (per-launch CUDA events) gives the verify GEMMs' achieved bytes/s and their share of 3.35 TB/s.
Bytes are algorithmic: every weight once per verify pass, the head once per draft pass (bench.weight_bytes_per_cycle);
int8 projections count 1 byte per weight plus 4 bytes per row, 4-bit ones half a byte per weight plus 4 bytes per 64 weights,
FP8 ones 1 byte per weight plus 16 bytes per 128 x 128 block (the kernel's padded scale layout).
The card's name and power limit are read in the same run.

`--model llama3-70b` (4-bit or FP8: no bf16 twin fits on one card) builds one quantized engine with random weights, quantized per
tensor on the device, and reports tok/s, tau, prefill, the engine's measured device footprint and how many generated tokens of
greedy eagenerate equal naivegenerate's on the timed prompt.

    python tools/w8_bench.py [--quant int8|nf4|fp4|fp8] [--model llama3-8b|llama3-70b] [--fixture random|correlated] [--rounds 3]
                             [--steps 2] [--warmup 2] [--out FILE]
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


def target_weights(args, tcfg, hcfg, dev, chunk_rows=None):
    """(name, tensor) of the target and the head, generated like bench.build_engine (random: streamed per tensor).  chunk_rows:
    draw random tensors that many rows at a time (other values than bench.py's, but no full-size fp32 temporary: a 70B FP8
    engine leaves a few GB of the card free)."""
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
        if kind == "normal" and chunk_rows and len(shape) == 2:
            w = torch.empty(shape, dtype=dtype, device=dev)
            for r in range(0, shape[0], chunk_rows):
                n = min(chunk_rows, shape[0] - r)
                w[r: r + n] = (torch.randn((n, shape[1]), generator=gen, device=dev, dtype=torch.float32) * 0.02).to(dtype)
        elif kind == "normal":
            w = (torch.randn(shape, generator=gen, device=dev, dtype=torch.float32) * 0.02).to(dtype)
        else:
            w = torch.ones(shape, dtype=dtype, device=dev) if kind == "ones" else torch.zeros(shape, dtype=dtype, device=dev)
        yield (name if which == "t" else "head." + name), w
    d2t, _ = syn.make_d2t(tcfg["vocab_size"], hcfg["draft_vocab_size"])
    yield "head.d2t", d2t


def quant_kwargs(q):
    if q == "fp8":
        return dict(quantization_config={"quant_method": "fp8", "activation_scheme": "dynamic", "weight_block_size": [128, 128]})
    return dict(load_in_8bit=True) if q == "int8" else dict(quantization_config={"load_in_4bit": True, "bnb_4bit_quant_type": q})


def quantize_pair(q, w):
    """(the quantized engine's tensors as (suffix, tensor) pairs, W')."""
    if q == "int8":
        qw, scb = quant.quantize_int8_rowwise(w)
        return [("weight", qw), ("SCB", scb)], quant.dequantize_int8_rowwise(qw, scb, torch.bfloat16)
    if q == "fp8":
        qw, scale_inv = quant.quantize_fp8_block(w)
        return [("weight", qw), ("weight_scale_inv", scale_inv)], quant.dequantize_fp8_block(qw, scale_inv, torch.bfloat16)
    packed, absmax = quant.quantize_4bit(w, q)
    return [("weight", packed), ("weight.absmax", absmax)], quant.dequantize_4bit(packed, absmax, q, torch.bfloat16)


def build_pair(args):
    tcfg, hcfg, _ = bench.model_configs(argparse.Namespace(model="llama3-8b", layers=0))
    if args.fixture == "correlated":
        hcfg = syn.head_config("llama3-8b", True, draft_vocab_size=32000, num_key_value_heads=tcfg["num_attention_heads"])
    kw = dict(use_eagle3=True, torch_dtype=torch.bfloat16, device=0, max_length=2048, **bench.TREE)
    mq = EaModel(tcfg, hcfg, **quant_kwargs(args.quant), **kw)
    mb = EaModel(tcfg, hcfg, **kw)
    for name, w in target_weights(args, tcfg, hcfg, "cuda:0"):
        if quant.is_target_projection(name):
            parts, wd = quantize_pair(args.quant, w)
            for suffix, t in parts:
                mq._load(name[: -len("weight")] + suffix, t)
            mb._load(name, wd)
        else:
            mq._load(name, w)
            mb._load(name, w)
        del w
    torch.cuda.empty_cache()
    return mq.finalize(), mb.finalize(), tcfg, hcfg


def bytes_per_cycle(tcfg, hcfg, q):
    """Algorithmic weight bytes of one cycle (bench.weight_bytes_per_cycle), with int8 projections at 1 B/weight + 4 B/row and
    4-bit ones at 0.5 B/weight + 4 B per 64 weights, FP8 ones at 1 B/weight + 16 B per 128 x 128 block (q: None for bf16)."""
    cyc, verify = bench.weight_bytes_per_cycle(tcfg, hcfg, True, bench.TREE["depth"])
    if not q:
        return cyc, verify
    saved = 0
    for which, name, shape, kind in bench.weight_specs(tcfg, hcfg, True):
        if which == "t" and quant.is_target_projection(name):
            nk = shape[0] * shape[1]
            saved += (nk - 4 * shape[0] if q == "int8" else nk - 16 * (nk // (128 * 128)) if q == "fp8"
                      else 2 * nk - (nk // 2 + 4 * (nk // 64)))
    return cyc - saved, verify - saved


def run_70b(args, info):
    """One 4-bit / FP8 Llama-3-70B + EAGLE-3 engine with random weights (quantized per tensor on the device)."""
    tcfg, hcfg, _ = bench.model_configs(argparse.Namespace(model="llama3-70b", layers=0))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    m = EaModel(tcfg, hcfg, use_eagle3=True, torch_dtype=torch.bfloat16, device=0, max_length=2048, **quant_kwargs(args.quant), **bench.TREE)
    for name, w in target_weights(args, tcfg, hcfg, "cuda:0", chunk_rows=8192):
        if quant.is_target_projection(name):
            m._load_target(name, w)
        else:
            m._load(name, w)
        del w
    m.finalize()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    footprint = free0 - torch.cuda.mem_get_info()[0]
    prompt = torch.randint(0, tcfg["vocab_size"] - 200, (1, bench.PROMPT_LEN), generator=torch.Generator().manual_seed(0)).cuda()
    for _ in range(max(1, args.warmup)):
        m.eagenerate(prompt, max_new_tokens=bench.NEW_TOKENS, max_length=2048)
    ms, new, cyc, last = 0.0, 0, 0, None
    windows = []
    for _ in range(args.rounds):
        w_ms, w_new, w_cyc, last = bench.timed_steps(m, prompt, args.steps, None, {})
        ms, new, cyc = ms + w_ms, new + w_new, cyc + w_cyc
        windows.append(round(w_new / (w_ms / 1e3), 2))
    naive = m.naivegenerate(prompt, max_new_tokens=bench.NEW_TOKENS, max_length=2048)
    n = min(last[0].shape[1], naive.shape[1])
    same = (last[0][0, :n] == naive[0, :n]).long().cumprod(0)
    lossless = bool(same.all())
    parting = None
    if not lossless:
        # where the two greedy paths part: the target's logits there, recomputed by a prefill of the common prefix
        j = int(same.sum())
        first = m.prefill(last[0][:, :j])
        logits = m.debug_read("verify_logits")[0]
        top = logits.topk(2)
        ulp = 2.0 ** (float(torch.floor(torch.log2(top.values[0].abs().clamp_min(1e-30)))) - 7)  # bf16 spacing at the top logit
        a_tok, b_tok = int(last[0][0, j]), int(naive[0, j])
        parting = {"position": j - bench.PROMPT_LEN, "eagenerate_token": a_tok, "naivegenerate_token": b_tok, "prefill_argmax": first,
                   "logit_eagenerate_token": float(logits[a_tok]), "logit_naivegenerate_token": float(logits[b_tok]),
                   "top2_tokens": top.indices.tolist(), "top2_logits": top.values.tolist(),
                   "top2_gap_bf16_ulps": float((top.values[0] - top.values[1]) / ulp)}
    stream = m.cuda_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    for _ in range(3):
        m.prefill(prompt)
    e1.record(stream)
    torch.cuda.synchronize()
    line = {"tool": "w8_bench", "workload": f"llama3-70b+eagle3 {args.quant} bs1 {bench.PROMPT_LEN}in/{bench.NEW_TOKENS}out greedy "
                                            f"dynamic-tree(60,6,10) random-init", "card": info, "rounds": args.rounds,
            "steps_per_window": args.steps, "tok_s": round(new / (ms / 1e3), 2), "tok_s_windows": windows,
            "tau": round(new / max(1, cyc), 3), "prefill_ms": round(e0.elapsed_time(e1) / 3, 3),
            "device_footprint_gb": round(footprint / 1e9, 3), "eagenerate_equals_naivegenerate": lossless,
            "identical_generated_prefix": int(same.sum()) - bench.PROMPT_LEN, "generated": n - bench.PROMPT_LEN, "parting": parting}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quant", default="int8", choices=["int8", "nf4", "fp4", "fp8"])
    ap.add_argument("--model", default="llama3-8b", choices=["llama3-8b", "llama3-70b"])
    ap.add_argument("--fixture", default="random", choices=["random", "correlated"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="eagenerate calls per timed window")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("w8_bench.py: no CUDA device (eagle_b200 has no CPU path)")
    if args.model == "llama3-70b" and (args.quant == "int8" or args.fixture != "random"):
        raise SystemExit("w8_bench.py: --model llama3-70b runs 4-bit or FP8 (--quant nf4|fp4|fp8) random-init weights only")
    torch.cuda.set_device(0)
    info = card()
    log(f"card: {info}")
    q = args.quant
    if args.model == "llama3-70b":
        return run_70b(args, info)
    log(f"building the {q} and the bf16-on-W' engines ({args.fixture} weights)")
    mq, mb, tcfg, hcfg = build_pair(args)
    engines = {q: mq, "bf16": mb}
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
        order = [q, "bf16"] if r % 2 == 0 else ["bf16", q]
        for name in order:
            ms, new, cyc, lst = bench.timed_steps(engines[name], prompt, args.steps, None, {})
            a = acc[name]
            a["ms"] += ms
            a["new"] += new
            a["cycles"] += cyc
            a["windows"].append(round(new / (ms / 1e3), 2))
            last[name] = lst
        log(f"round {r}: " + ", ".join(f"{k} {acc[k]['windows'][-1]} tok/s" for k in engines))
    parity = (last[q][0].cpu().tolist() == last["bf16"][0].cpu().tolist() and last[q][1:] == last["bf16"][1:])
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
        cyc_bytes, verify_bytes = bytes_per_cycle(tcfg, hcfg, None if name == "bf16" else q)
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
            "card": info, "rounds": args.rounds, "steps_per_window": args.steps, f"ids_identical_{q}_vs_bf16_on_Wprime": parity,
            q: res[q], "bf16": res["bf16"], "speedup_tok_s": round(res[q]["tok_s"] / res["bf16"]["tok_s"], 4)}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")
    if not parity:
        raise SystemExit(f"w8_bench.py: the {q} engine's ids differ from the bf16 engine's on W'")


if __name__ == "__main__":
    main()

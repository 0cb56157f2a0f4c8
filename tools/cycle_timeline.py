"""Per-kernel timeline of bench.py's headline cycle on the GPU: where the time of a draft -> verify -> accept cycle goes.

Builds the workload exactly as bench.py does (bench.build_engine: Llama-3-8B + EAGLE-3 shapes, bf16, random weights), prefills the
512-token prompt, warms up, then runs a few cycles (`EaModel.step`, CUDA-graph replay) under torch.profiler with CUDA activities.
Under programmatic dependent launch a kernel starts while its predecessor still runs, so a kernel's duration (start to end)
includes time it spends waiting on griddepcontrol.wait, and durations overlap.  The timeline therefore also gives each kernel's
EXPOSED time: from the later of its start and the previous kernel's end to its own end.  Exposed times and gaps add up to the
span, so they say where the cycle's time goes.  Prints, per cycle:
  * per projection (verify: qkv, o, gate/up, down; draft: fc, qkv, o, gate/up, down, lm_head): launches, mean duration, mean
    exposed time and the achieved bandwidth N*K*2 / exposed time (weight bytes only);
  * per other kernel name: launches, mean duration and mean exposed time;
  * the exposed time of GEMM and non-GEMM kernels, and the gaps between consecutive kernels (gaps above 50 us, the host round
    trip between two cycles, are summed separately);
  * the card name, power limit and SM clock, read with nvidia-smi in the same run.
The trace (chrome JSON) and the summary are written to --out (default: a directory under the system temp dir).  Run it with
and without EB200_L2_PREFETCH=1 (the L2 weight prefetch, off by default) for an A/B picture.

    python tools/cycle_timeline.py [--cycles 8] [--warmup-cycles 20] [--out DIR] [--tree dynamic|static]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402

HOST_GAP_US = 50.0


def card():
    q = "name,power.limit,power.max_limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")]))
    except Exception as ex:  # the numbers are still printed, without the card
        return {"error": repr(ex)}


def projections(tcfg, hcfg):
    """(N, K) of every projection of the cycle, as the engine stores them (q/k/v fused, gate/up interleaved into one matrix)."""
    H, I, hd = tcfg["hidden_size"], tcfg["intermediate_size"], 128
    Hh, Ih = hcfg["hidden_size"], hcfg["intermediate_size"]
    return {
        "verify.qkv": ((tcfg["num_attention_heads"] + 2 * tcfg["num_key_value_heads"]) * hd, H),
        "verify.o": (H, H), "verify.gate_up": (2 * I, H), "verify.down": (H, I),
        "draft.fc": (Hh, 3 * H), "draft.qkv": ((hcfg["num_attention_heads"] + 2 * hcfg["num_key_value_heads"]) * hd, 2 * Hh),
        "draft.o": (Hh, Hh), "draft.gate_up": (2 * Ih, Hh), "draft.down": (Hh, Ih), "draft.lm_head": (hcfg["draft_vocab_size"], Hh),
    }


def label(name, grid, prev_gemm, shapes):
    """Projection of a skinny_gemm_wgmma launch from its template arguments <T, MPAD, EPI, ...> and grid (n-tiles, split-K)."""
    m = re.search(r"skinny_gemm_wgmma<[^,]+,\s*(\d+),\s*(\d+)", name)
    if not m:
        return None
    mpad, epi = int(m.group(1)), int(m.group(2))
    side = "verify" if mpad == 64 else "draft"
    if epi == 3:
        return side + ".qkv"
    if epi in (2, 5):
        return side + ".gate_up"
    if epi in (1, 4):  # residual: o_proj follows the qkv (through attention), down_proj follows gate/up
        return side + (".o" if prev_gemm and prev_gemm.endswith(".qkv") else ".down")
    # store: fc (N = Hh tiles) or the draft lm_head
    tiles = grid[0] if grid else 0
    return "draft.fc" if tiles * 128 <= shapes["draft.fc"][0] else "draft.lm_head"


def short(name):
    return re.sub(r"<.*", "", re.sub(r"^void\s+", "", re.sub(r"\(.*", "", name))).replace("eb::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=8)
    ap.add_argument("--warmup-cycles", type=int, default=20)
    ap.add_argument("--tree", default="dynamic", choices=["dynamic", "static"])
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "eagle_b200_timeline"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cycle_timeline.py: no CUDA device")
    args = argparse.Namespace(model="llama3-8b", dtype="bf16", tree=a.tree, fixture="random", layers=0, temperature=0.0)
    m, tcfg, hcfg, eagle3 = bench.build_engine(args, 0, 0, 1)
    prompt = torch.randint(0, tcfg["vocab_size"] - 200, (1, bench.PROMPT_LEN), generator=torch.Generator().manual_seed(0)).cuda()
    m.prefill(prompt)
    for _ in range(a.warmup_cycles):
        m.step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.cycles):
            m.step()
        torch.cuda.synchronize()
    os.makedirs(a.out, exist_ok=True)
    tag = "pf_on" if os.environ.get("EB200_L2_PREFETCH") == "1" else "pf_off"
    trace = os.path.join(a.out, f"trace_{tag}_{a.tree}.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X" and e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    shapes = projections(tcfg, hcfg)
    n = a.cycles
    per = defaultdict(lambda: [0, 0.0, 0.0])  # key -> [launches, summed duration us, summed exposed us]
    gemm_us = other_us = gap_us = host_gap_us = 0.0
    prev_gemm, end = None, None
    for e in ev:
        name, dur = e["name"], float(e["dur"])
        grid = e.get("args", {}).get("grid")
        lab = label(name, grid, prev_gemm, shapes)
        if lab:
            prev_gemm = lab
        key = lab or short(name)
        exposed = e["ts"] + dur - max(e["ts"], end if end is not None else e["ts"])
        exposed = max(0.0, exposed)
        per[key][0] += 1
        per[key][1] += dur
        per[key][2] += exposed
        if lab or "gemm" in name:
            gemm_us += exposed
        else:
            other_us += exposed
        if end is not None:
            g = max(0.0, e["ts"] - end)
            if g > HOST_GAP_US:
                host_gap_us += g
            else:
                gap_us += g
        end = max(end or 0.0, e["ts"] + dur)
    span_us = (end - ev[0]["ts"]) if ev else 0.0
    rows = []
    for key, (cnt, us, ex) in sorted(per.items(), key=lambda kv: -kv[1][2]):
        r = {"kernel": key, "launches_per_cycle": round(cnt / n, 2), "mean_us": round(us / cnt, 2), "mean_exposed_us": round(ex / cnt, 2),
             "exposed_us_per_cycle": round(ex / n, 1)}
        if key in shapes and ex > 0:
            N, K = shapes[key]
            r["gbs"] = round(N * K * 2 / (ex / cnt * 1e-6) / 1e9, 1)
        rows.append(r)
    out = {"prefetch": tag, "tree": a.tree, "cycles": n, "kernels_seen": len(ev), "card": card(),
           "per_cycle_ms": {"span": round(span_us / n / 1e3, 3), "gemm_exposed": round(gemm_us / n / 1e3, 3),
                            "non_gemm_exposed": round(other_us / n / 1e3, 3),
                            "gaps": round(gap_us / n / 1e3, 3), "host_gaps": round(host_gap_us / n / 1e3, 3)},
           "kernels": rows, "trace": trace}
    for r in rows:
        print(f"{r['kernel'][:40]:40s} {r['launches_per_cycle']:7.2f}/cycle {r['mean_us']:9.2f} us {r['mean_exposed_us']:9.2f} us exposed "
              f"{r['exposed_us_per_cycle']:9.1f} us/cycle"
              + (f" {r['gbs']:8.1f} GB/s" if "gbs" in r else ""))
    print(json.dumps({k: v for k, v in out.items() if k != "kernels"}))
    with open(os.path.join(a.out, f"timeline_{tag}_{a.tree}.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

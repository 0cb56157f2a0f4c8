"""Tensor-parallel parity on >= 2 H100s: the target sharded 2-way over NCCL/NVLink (draft head replicated) must emit
exactly the tokens of the reference (golden vectors), i.e. of the single-GPU engine.  Skipped with fewer than 2 GPUs; run
with `python -m pytest tests/test_tp_gpu.py -m gpu` on a machine with two.  Each rank is a separate process with a hard
deadline (a rank that dies would otherwise leave its peer blocked in a collective)."""
import json
import os
import socket
import subprocess
import sys
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import json, os, sys, traceback
sys.path.insert(0, os.environ["EB_ROOT"])
import torch, torch.distributed as dist
rank, world, fx = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), os.environ["EB_FX"]
out = {"rank": rank}
try:
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)   # only carries the 128-byte NCCL id
    from eagle_b200 import EaModel
    from oracle.make_golden import fixture_models
    from tests.fixtures import load_golden
    g = load_golden(fx)
    tcfg, tW, hcfg, hW, eagle3, dtype, tree = fixture_models(fx)
    m = EaModel.from_state_dicts(tcfg, tW, hcfg, hW, use_eagle3=eagle3, torch_dtype=dtype, max_length=512, device=rank,
                                 tp_rank=rank, tp_size=world, **tree)
    out["built"] = True
    out["tp_fused"] = bool(getattr(m, "tp_fused", False))
    ids, new_token, idx = m.eagenerate(g["prompt"].cuda(rank), log=True, **g["gen_kw"])
    out["ids_ok"] = ids.cpu().tolist() == g["ids"].tolist()
    out["log_ok"] = (new_token, idx) == (g["new_token"], g["idx"])
    naive = m.naivegenerate(g["prompt"].cuda(rank), max_new_tokens=g["gen_kw"]["max_new_tokens"], max_length=g["gen_kw"]["max_length"])
    out["naive_ok"] = naive.cpu().tolist() == g["naive_ids"].tolist()
except Exception:
    out["error"] = traceback.format_exc()[-1500:]
try:
    torch.cuda.synchronize()
    dist.barrier()  # no rank frees its peer window while the other may still be inside its last cycle
except Exception:
    pass
print("RESULT " + json.dumps(out), flush=True)
os._exit(0)
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("fused,two_shot_min", [("1", "8"), ("1", "2"), ("0", "8")],
                         ids=["nvlink-one-shot", "nvlink-two-shot", "nccl-allreduce"])
@pytest.mark.parametrize("fx", ["e3_gqa_bf16", "e1_corr_fp16", "e3_tp8_bf16"])
def test_tp2_matches_reference(fx, fused, two_shot_min):
    """All three tensor-parallel data paths -- the one-shot exchange kernel over NVLink peer windows (default below 8 ranks),
    the row-owner two-shot kernel (default from 8 ranks, forced here with EB200_TP_TWO_SHOT_MIN=2) and the NCCL all-reduce
    path (EB200_TP_FUSED=0) -- must reproduce the reference's tokens."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), EB_FX=fx, EB_ROOT=ROOT,
                   EB200_TP_FUSED=fused, EB200_TP_TWO_SHOT_MIN=two_shot_min)
        procs.append(subprocess.Popen([sys.executable, "-c", WORKER], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    deadline = time.time() + 150
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=max(1, deadline - time.time()))
        except subprocess.TimeoutExpired:
            p.kill()
            o, _ = p.communicate()
            o += "\nTIMEOUT"
        outs.append(o)
    res = []
    for o in outs:
        lines = [l for l in o.splitlines() if l.startswith("RESULT ")]
        assert lines, "rank produced no result:\n" + o[-2000:]
        res.append(json.loads(lines[-1][7:]))
    for r in res:
        assert "error" not in r, r["error"]
        assert r.get("ids_ok") and r.get("log_ok") and r.get("naive_ok"), r
        if fused == "1":
            assert r.get("tp_fused"), "NVLink peer windows did not open on this box: " + json.dumps(r)

"""Tensor-parallel plumbing: one process per GPU (torchrun), torch.distributed only carries the 128-byte NCCL unique id;
the collectives themselves are issued by libeagle_b200.so on its own stream (NCCL over NVLink / NVSwitch).

The reference has no tensor parallelism (its multi-GPU mode is accelerate layer placement, ea_model.py:104-118);
sharding follows the usual column/row-parallel split of a Llama block (SURVEY.md 8e): q/k/v by heads and gate/up by rows,
o_proj/down_proj by columns with one all-reduce each, vocab-parallel lm_head with an arg-max exchange; the draft head is
replicated on every rank (zero communication)."""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib


def shard_of(name: str, rows: int, cols: int, tp_rank: int, tp_size: int):
    """(row0, n_rows, col0, n_cols) kept by `tp_rank` for the target tensor `name` (same function the engine applies)."""
    out = (C.c_int64 * 4)()
    _lib.check(_lib.load().eb200_tp_shard(name.encode(), rows, cols, tp_rank, tp_size, out))
    return tuple(int(x) for x in out)


def broadcast_unique_id(group=None, device=None) -> torch.Tensor:
    """Rank 0 creates the ncclUniqueId, everyone receives it through the existing process group (gloo or nccl)."""
    import torch.distributed as dist
    buf = torch.zeros(128, dtype=torch.uint8)
    if dist.get_rank(group) == 0:
        _lib.check(_lib.load().eb200_tp_unique_id(buf.data_ptr()))
    if dist.get_backend(group) == "nccl":
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        t = buf.to(dev)
        dist.broadcast(t, src=0, group=group)
        buf = t.cpu()
    else:
        dist.broadcast(buf, src=0, group=group)
    return buf


def init_engine_tp(model, group=None):
    """Join the engine of `model` (an EaModel built with tp_rank/tp_size) to the tensor-parallel communicator, then open the
    NVLink peer windows: every rank exports a CUDA IPC handle of its window, the handles are all-gathered through the existing
    process group, and each engine maps the others' windows.  `model.tp_fused` tells whether the peer path is active (it is
    not when the GPUs of the job have no peer access: the engine then keeps the NCCL all-reduce path and says so)."""
    import warnings

    import torch.distributed as dist
    dev = torch.device("cuda", model.device)
    buf = broadcast_unique_id(group, dev)
    _lib.check(model.lib.eb200_tp_init(model._h, buf.data_ptr()))
    world = dist.get_world_size(group)
    mine = torch.zeros(64, dtype=torch.uint8)
    _lib.check(model.lib.eb200_tp_ipc_handle(model._h, mine.data_ptr()))
    if dist.get_backend(group) == "nccl":
        out = torch.zeros(world, 64, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(out, mine.to(dev), group=group)
        handles = out.cpu().contiguous()
    else:
        lst = [torch.zeros(64, dtype=torch.uint8) for _ in range(world)]
        dist.all_gather(lst, mine, group=group)
        handles = torch.stack(lst).contiguous()
    rc = model.lib.eb200_tp_open_peers(model._h, handles.data_ptr(), world)
    ok = torch.tensor([1 if rc == 0 else 0], device=dev if dist.get_backend(group) == "nccl" else None)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
    if rc != 0:
        warnings.warn("eagle_b200: NVLink peer windows unavailable (" + model.lib.eb200_last_error().decode("utf-8", "replace") +
                      "); tensor parallelism falls back to NCCL all-reduce")
    if int(ok[0]) != 1 and rc == 0:
        raise _lib.EngineError("tensor-parallel peers disagree about NVLink peer access; set EB200_TP_FUSED=0 on every rank")
    model.tp_fused = bool(rc == 0 and os.environ.get("EB200_TP_FUSED", "1") != "0")
    dist.barrier(group=group)  # every window is zero-initialised and mapped before anyone writes into a peer

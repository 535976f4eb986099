"""Multi-GPU plumbing for partition-range sharding (SURVEY §8e).

One process per GPU; rank g owns the partitions [g*ceil(P/G), (g+1)*ceil(P/G)) of every stage:
it keeps only those IR spectra, recomputes the (tiny) input spectra itself from the broadcast
input, and produces a PARTIAL spectrum sum.  Between the FDL sweep and the inverse FFT the
engine calls back into `attach_reduce`'s hook, which sums the partial spectra of all ranks into
rank 0 with ONE collective per launch group (ncclReduce over NVLink under the "nccl" backend).
Only rank 0 runs the inverse FFT / overlap-add and produces audio.

Tail layout (Engine(..., shard_head=False)): rank 0 keeps the head stage whole and only the stages >= 1 are split.
The hook then runs once per completed tail block (never for the head), and `attach_p2p` attaches the tail slot
exchange instead: every rank stores its partial tail spectrum into rank 0's slots over peer memory, off the path of the
real-time call.

The "gloo" branch exists for the world_size-2 CPU tests: with the emulation build of the C ABI
the "device" pointers are host memory, so the same hook reduces them with gloo.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
import torch.distributed as dist


class _CudaView:
    """Zero-copy __cuda_array_interface__ view of n float32 at a raw device pointer."""

    def __init__(self, ptr: int, n: int):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}


def attach_reduce(engine, device: int | None = None, group=None, root: int = 0) -> None:
    """Installs the reduce hook on a sharded Engine (engine.shard_count == world size)."""
    backend = dist.get_backend(group)
    if backend == "nccl":
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        streams = {}

        def hook(ptr: int, n: int, stream_ptr: int) -> int:
            # the engine hands over the stream the partial spectra were produced on (its post stream):
            # the reduce is ordered after the sweep and before the inverse FFT on that stream
            st = streams.get(stream_ptr)
            if st is None:
                st = streams[stream_ptr] = torch.cuda.ExternalStream(stream_ptr, device=dev)
            t = torch.as_tensor(_CudaView(ptr, n), device=dev)
            with torch.cuda.stream(st):
                dist.reduce(t, dst=root, op=dist.ReduceOp.SUM, group=group)
            return 0
    else:
        def hook(ptr: int, n: int, _stream: int) -> int:
            buf = (ctypes.c_float * n).from_address(ptr)
            t = torch.from_numpy(np.ctypeslib.as_array(buf))
            dist.reduce(t, dst=root, op=dist.ReduceOp.SUM, group=group)
            return 0
    engine.set_reduce(hook)


def attach_p2p(engine, group=None) -> tuple:
    """Enables the fused slot-exchange path on a sharded uniform Engine, or the tail slot exchange on an Engine created
    with shard_head=False (any stage schedule).  torch.distributed only moves the
    CUDA IPC blobs (plumbing) — the data path makes no NCCL call.  Every rank executes the same collectives
    whether or not its own export / import works, and all ranks end on the SAME path:
    returns (True, "") if the exchange is active everywhere, else (False, reason) with the exchange detached."""
    world = dist.get_world_size(group)
    blob, err = None, ""
    try:
        blob = engine.p2p_export(mode=0)
    except Exception as ex:                       # e.g. CUDA IPC not permitted in this container
        err = f"export: {ex}"
    gathered = [None] * world
    dist.all_gather_object(gathered, (blob, err), group=group)
    if all(b is not None for b, _ in gathered):
        try:
            engine.p2p_import([b for b, _ in gathered])
        except Exception as ex:
            err = f"import: {ex}"
    else:
        err = err or next(e for b, e in gathered if b is None)
    oks = [None] * world
    dist.all_gather_object(oks, err, group=group)
    bad = [e for e in oks if e]
    if bad:
        engine.p2p_detach()
        return False, bad[0]
    return True, ""

"""Rank 0's real-time call latency of REEV-R's quad two-stage handle with the tail stage sharded over G GPUs.

  torchrun --nproc-per-node G tools/tail_shard_bench.py [--calls 2000]
      one rank per GPU: the head-sharded layout with the NCCL reduce hook and the tail layout (shard_head = 0) with
      the slot exchange over CUDA IPC (mode 0), both at G = world size
  python tools/tail_shard_bench.py [--shards 2 4 8] [--calls 2000]
      without torchrun: the G shards of the tail layout run as threads of this process on ONE device (raw-pointer
      exchange, host barrier at every tail block) — the results are labelled "in-process shards on one device"; the
      NCCL reduce needs one process per GPU and is reported as not measured

Workload: 4 convolvers (LL, RR, LR, RL), head 128 / tail 8192 (StereoConvolver.cpp:15 for a 128-sample host block),
120 s IRs at 48 kHz, host calls of 128 samples.  Every rank gets the same input and the same call lengths.  Rank 0's
call is timed on the host clock around b200conv_process (which returns after its synchronise); median / min / max over
`--calls` calls after `--warmup` untimed ones, plus b200conv_launch_count per call and the parity of rank 0's output
against the unsharded engine on the same input.  Prints one JSON line with the card's name and power limit, read in the
same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SRATE, HEAD, TAIL, BLOCK, IR_SECONDS, CH = 48000.0, 128, 8192, 128, 120.0, 4


def power_limit_w(dev=0):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(dev)],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 4), "min_ms": round(float(a.min()), 4),
            "max_ms": round(float(a.max()), 4), "n": int(a.size)}


class Calls:
    """Pointer arrays of every 128-sample call into one input / one output buffer (no allocation while timing)."""

    def __init__(self, xs, n_calls):
        self.y = np.zeros((CH, n_calls * BLOCK), np.float32)
        self.ins, self.outs = [], []
        for i in range(n_calls):
            a, b = (C.c_void_p * CH)(), (C.c_void_p * CH)()
            for c in range(CH):
                a[c] = xs[c].ctypes.data + 4 * i * BLOCK
                b[c] = self.y[c].ctypes.data + 4 * i * BLOCK
            self.ins.append(a)
            self.outs.append(b)

    def run(self, e, warmup, timed):
        lat, launches = [], []
        for i in range(len(self.ins)):
            l0 = e.launch_count
            t = time.perf_counter()
            e.process_into(self.ins[i], self.outs[i], BLOCK)
            dt = (time.perf_counter() - t) * 1e3
            if timed and i >= warmup:
                lat.append(dt)
                launches.append(e.launch_count - l0)
        return lat, launches


def summary(lat, launches, y, ref):
    err = float(np.max(np.abs(y.astype(np.float64) - ref)) / np.max(np.abs(ref)))
    return {"rank0_call": stats(lat), "launches_per_call_median": float(np.median(launches)),
            "launches_per_call_max": int(max(launches)), "parity_vs_unsharded": err}


def in_process_tail(Engine, irs, xs, n_calls, warmup, G):
    """G tail-layout shards as threads of this process on device 0 (raw pointers, host barrier)."""
    box, bar, host_bar = [None] * G, threading.Barrier(G), threading.Barrier(G)
    res, errs = {}, []

    def worker(rank):
        try:
            e = Engine(CH, device=0, shard_rank=rank, shard_count=G, shard_head=False)
            assert e.init_twostage(HEAD, TAIL, irs)

            def allgather(blob):
                box[rank] = blob
                bar.wait(600)
                out = list(box)
                bar.wait(600)
                return out
            e.p2p_attach(allgather, mode=1, host_barrier=lambda: (host_bar.wait(600), 0)[1])
            calls = Calls(xs, n_calls)
            bar.wait(600)
            lat, launches = calls.run(e, warmup, rank == 0)
            if rank == 0:
                res.update(lat=lat, launches=launches, y=calls.y)
            bar.wait(600)
            e.close()
        except Exception as ex:
            errs.append(repr(ex))
            bar.abort()
            host_bar.abort()

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(G)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    if errs:
        raise RuntimeError(errs[0])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--shards", type=int, nargs="*", default=[2, 4, 8])
    a = ap.parse_args()

    import torch
    from reevr_b200 import Engine
    from reevr_b200.synth import synth_input, synth_ir

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl")
    dev = rank if world > 1 else 0
    n_calls = a.warmup + a.calls
    irs = [synth_ir(int(IR_SECONDS * SRATE), c) for c in range(CH)]
    xs = [synth_input(n_calls * BLOCK, c) for c in range(CH)]
    res = {"workload": f"quad two-stage head {HEAD} tail {TAIL}, {IR_SECONDS:g} s IRs at {SRATE / 1000:g} kHz, "
                       f"host calls of {BLOCK} samples",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev),
           "callback_period_ms": round(BLOCK / SRATE * 1e3, 4)}

    # unsharded handle (rank 0's device)
    ref = None
    if rank == 0:
        u = Engine(CH, device=dev)
        assert u.init_twostage(HEAD, TAIL, irs)
        calls = Calls(xs, n_calls)
        lat, launches = calls.run(u, a.warmup, True)
        ref = calls.y.astype(np.float64)
        res["unsharded"] = summary(lat, launches, calls.y, ref)
        u.close()

    if world > 1:
        from reevr_b200.distributed import attach_p2p, attach_reduce
        res["mode"] = f"one process per GPU, {world} GPUs"
        for key, shard_head in (("head_sharded_nccl_reduce", True), ("tail_sharded_slot_exchange", False)):
            e = Engine(CH, device=dev, shard_rank=rank, shard_count=world, shard_head=shard_head)
            assert e.init_twostage(HEAD, TAIL, irs)
            attach_reduce(e)
            if not shard_head:
                ok, why = attach_p2p(e)
                if not ok:
                    res[key] = f"not measured: slot exchange unavailable ({why})"
                    e.close()
                    continue
            calls = Calls(xs, n_calls)
            dist.barrier()
            lat, launches = calls.run(e, a.warmup, rank == 0)
            dist.barrier()
            if rank == 0:
                res[key] = {"G": world, **summary(lat, launches, calls.y, ref)}
            e.close()
        for G in a.shards:
            if G != world:
                res.setdefault("tail_sharded_other_G", {})[str(G)] = "not measured"
        dist.destroy_process_group()
    else:
        res["mode"] = "in-process shards on one device (threads, host barrier at every tail block); multi-GPU not measured"
        res["head_sharded_nccl_reduce"] = "not measured (needs one process per GPU)"
        out = {}
        for G in a.shards:
            r = in_process_tail(Engine, irs, xs, n_calls, a.warmup, G)
            out[str(G)] = summary(r["lat"], r["launches"], r["y"], ref)
        res["tail_sharded_slot_exchange_in_process"] = out
    if rank == 0:
        print(json.dumps(res))


if __name__ == "__main__":
    main()

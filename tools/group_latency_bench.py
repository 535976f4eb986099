"""Fixed-latency members per audio callback: N own b200conv_process calls against one b200conv_group_process whose group
latency makes the members share their head-block steps (b200conv_group_set_latency).

Members: REEV-R's quad two-stage shape (head 128, tail 8192, 10 s IRs) with routing [0, 1, 0, 1] and the quad mixdown.
Cases: N in {1, 8, 32} members, latency 2 * 128, host blocks of 128 and 32 samples.  Every callback is paced at the
audio rate (host block / 48 kHz) and does both legs on two sets of handles with the same IRs and input: first the N
own calls on the twins (each given the latency by its own set_latency), then the group call on the members.  Each leg
is timed with the host clock; a fixed-latency call returns once its output is copied, which is D samples behind.  The
first `--warm` callbacks are untimed.  Reported per case: median / p99 microseconds per callback of each leg, group and
member launches per callback, latency_waits per member of each leg (counted over the timed callbacks), and the largest
difference between the two legs' outputs.  The card's name and power limit are read in the same run.  Needs a GPU.

  python tools/group_latency_bench.py [--warm 200] [--calls 1500] [--sizes 1,8,32] [--blocks 128,32] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from reevr_b200.convolver import Engine, Group  # noqa: E402
from reevr_b200.synth import synth_input, synth_ir  # noqa: E402

SR = 48000
IR_10S = 480000
HEAD, TAIL, D = 128, 8192, 256
QUAD_MAP, QUAD_MIX = [0, 1, 0, 1], [[1, 0, 0, 1], [0, 1, 1, 0]]


def quad(seed):
    e = Engine(4)
    assert e.init_twostage(HEAD, TAIL, [synth_ir(IR_10S, 4 * seed + c) for c in range(4)])
    e.set_routing(QUAD_MAP, QUAD_MIX)
    return e


def table(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


class Case:
    def __init__(self, n, block):
        self.block = block
        self.members = [quad(i) for i in range(n)]
        self.twins = [quad(i) for i in range(n)]
        for e in self.twins:
            e.set_latency(D)
        self.group = Group(self.members)
        self.group.set_latency(D)
        self.lib = self.members[0]._l
        self.xin = [[np.zeros(block, np.float32) for _ in range(2)] for _ in range(n)]
        self.y_own = [[np.zeros(block, np.float32) for _ in range(2)] for _ in range(n)]
        self.y_group = [[np.zeros(block, np.float32) for _ in range(2)] for _ in range(n)]
        self.p_in = [table(x) for x in self.xin]
        self.p_own = [table(y) for y in self.y_own]
        self.p_group = [table(y) for y in self.y_group]
        self.g_in = (C.c_void_p * n)(*[C.cast(p, C.c_void_p) for p in self.p_in])
        self.g_out = (C.c_void_p * n)(*[C.cast(p, C.c_void_p) for p in self.p_group])
        self.src = [[synth_input(HEAD * 64, 7 * i + c) for c in range(2)] for i in range(n)]

    def feed(self, k):
        off = (k * self.block) % (HEAD * 63)
        for x, s in zip(self.xin, self.src):
            for a, b in zip(x, s):
                a[:] = b[off:off + self.block]

    def own(self):
        for e, pi, po in zip(self.twins, self.p_in, self.p_own):
            if self.lib.b200conv_process(e._h, pi, po, self.block):
                raise RuntimeError(self.lib.b200conv_last_error(e._h).decode())

    def grouped(self):
        if self.lib.b200conv_group_process(self.group._g, C.cast(self.g_in, C.POINTER(C.c_void_p)),
                                           C.cast(self.g_out, C.POINTER(C.c_void_p)), self.block):
            raise RuntimeError(self.lib.b200conv_group_last_error(self.group._g).decode())

    def diff(self):
        return max(float(np.max(np.abs(a - b))) for yo, yg in zip(self.y_own, self.y_group) for a, b in zip(yo, yg))

    def close(self):
        self.group.close()
        for e in self.members + self.twins:
            e.close()


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "p99_us": round(float(np.percentile(a, 99)), 1)}


def run_case(n, block, warm, calls):
    c = Case(n, block)
    period = block / SR
    t_own, t_group, l_group, l_members, l_twins, dmax = [], [], [], [], [], 0.0
    t_next = time.perf_counter()
    for k in range(warm + calls):
        if k == warm:
            w_members = [e.latency_waits for e in c.members]
            w_twins = [e.latency_waits for e in c.twins]
        while time.perf_counter() < t_next:
            pass
        c.feed(k)
        g0 = c.group.launch_count
        m0 = sum(e.launch_count for e in c.members)
        o0 = sum(e.launch_count for e in c.twins)
        t0 = time.perf_counter()
        c.own()
        t1 = time.perf_counter()
        c.grouped()
        t2 = time.perf_counter()
        if k >= warm:
            t_own.append((t1 - t0) * 1e6)
            t_group.append((t2 - t1) * 1e6)
            l_group.append(c.group.launch_count - g0)
            l_members.append(sum(e.launch_count for e in c.members) - m0)
            l_twins.append(sum(e.launch_count for e in c.twins) - o0)
            dmax = max(dmax, c.diff())
        t_next += period
        t_next = max(t_next, time.perf_counter())       # a late callback does not start a burst of catch-up calls
    waits_group = [e.latency_waits - w for e, w in zip(c.members, w_members)]
    waits_own = [e.latency_waits - w for e, w in zip(c.twins, w_twins)]
    c.close()
    return {"members": n, "host_block": block, "latency": D, "calls": calls,
            "own_calls": stats(t_own), "group_call": stats(t_group),
            "own_launches_per_callback": round(float(np.mean(l_twins)), 3),
            "group_launches_per_callback": round(float(np.mean(l_group)), 3),
            "group_member_launches_per_callback": round(float(np.mean(l_members)), 3),
            "latency_waits_own_max": max(waits_own), "latency_waits_group_max": max(waits_group),
            "max_abs_diff_group_vs_own": dmax}


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm", type=int, default=200)
    ap.add_argument("--calls", type=int, default=1500)
    ap.add_argument("--sizes", default="1,8,32")
    ap.add_argument("--blocks", default="128,32")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("group_latency_bench.py needs a CUDA device")
    results = [{"card": card()}]
    print(json.dumps(results[0]), flush=True)
    for block in [int(b) for b in a.blocks.split(",")]:
        for n in [int(s) for s in a.sizes.split(",")]:
            results.append(run_case(n, block, a.warm, a.calls))
            print(json.dumps(results[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

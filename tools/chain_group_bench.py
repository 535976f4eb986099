"""Send / wet chain calls of N handles per audio callback: N single b200conv_chain_process calls against one
b200conv_chain_group_process.

Every callback is paced at the audio rate (host block / 48 kHz) and does both, on two sets of handles with the same IRs,
chain configurations and input: first the N single calls on the twins, then the group call on the members, each timed
with the host clock (the call returns with its output complete).  The first `--warm` callbacks are untimed.  Reported
per leg: median / p99 / max microseconds per callback, group launches per callback, and the largest difference between
the group's and the single calls' outputs.  The chains run both cuts (12 and 24 dB), a predelay and both envelopes; the
"nocut" leg switches the cuts off, which leaves the send kernels without their serial scan, to show whether that scan
sets the floor of a group call.

  python tools/chain_group_bench.py [--warm 200] [--calls 2000] [--legs quad128,quad480,mixed,nocut] [--out FILE]
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
CUTS = dict(srate=float(SR), lowcut_hz=120.0, lowcut_slope=1, highcut_hz=9000.0, highcut_slope=2, predelay=480,
            width=0.8, drygain=0.7, wetgain=0.5, true_stereo=True)
NOCUT = dict(CUTS, lowcut_hz=20.0, highcut_hz=20000.0)


def quad(head, tail, seed):
    return lambda: (Engine(4), lambda e: e.init_twostage(head, tail, [synth_ir(IR_10S, 4 * seed + c) for c in range(4)]))


def stereo(head, tail, seed):
    return lambda: (Engine(2), lambda e: e.init_twostage(head, tail, [synth_ir(IR_10S, 2 * seed + c) for c in range(2)]))


def stereo_uniform(block, parts, seed):
    return lambda: (Engine(2), lambda e: e.init_uniform(block, [synth_ir(block * parts - 3, 2 * seed + c) for c in range(2)]))


def build(recipe, cfg):
    e, init = recipe()
    assert init(e)
    e.chain_configure(**cfg)
    return e


def table(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


class Leg:
    def __init__(self, recipes, block, cfg):
        self.block = block
        self.members = [build(r, cfg) for r in recipes]
        self.twins = [build(r, cfg) for r in recipes]
        self.group = Group(self.members)
        self.lib = self.members[0]._l
        m, n = len(self.members), block
        self.dry = [[np.zeros(n, np.float32) for _ in range(2)] for _ in range(m)]
        self.env = [[np.zeros(n, np.float32) for _ in range(m)] for _ in range(2)]       # ysend, yrev per member
        self.y_single = [[np.zeros(n, np.float32) for _ in range(2)] for _ in range(m)]
        self.y_group = [[np.zeros(n, np.float32) for _ in range(2)] for _ in range(m)]
        self.p_dry = [table(x) for x in self.dry]
        self.p_single = [table(y) for y in self.y_single]
        self.p_group = [table(y) for y in self.y_group]
        self.g_dry = (C.c_void_p * m)(*[C.cast(p, C.c_void_p) for p in self.p_dry])
        self.g_out = (C.c_void_p * m)(*[C.cast(p, C.c_void_p) for p in self.p_group])
        self.g_env = [table(e) for e in self.env]
        self.src = [[synth_input(block * 64, 7 * i + c) for c in range(2)] for i in range(m)]
        t = np.arange(block * 64)
        self.src_env = [0.5 + 0.5 * np.abs(np.sin(t * 1e-3)), 0.25 + 0.75 * np.abs(np.cos(t * 7e-4))]

    def feed(self, k):
        off = (k % 63) * self.block
        for x, s in zip(self.dry, self.src):
            for a, b in zip(x, s):
                a[:] = b[off:off + self.block]
        for es, s in zip(self.env, self.src_env):
            for a in es:
                a[:] = s[off:off + self.block]

    def single(self):
        for i, (e, pd, po) in enumerate(zip(self.twins, self.p_dry, self.p_single)):
            if self.lib.b200conv_chain_process(e._h, pd, self.env[0][i].ctypes.data, self.env[1][i].ctypes.data, po,
                                               self.block):
                raise RuntimeError(self.lib.b200conv_last_error(e._h).decode())

    def grouped(self):
        pp = C.POINTER(C.c_void_p)
        if self.lib.b200conv_chain_group_process(self.group._g, C.cast(self.g_dry, pp), C.cast(self.g_env[0], pp),
                                                 C.cast(self.g_env[1], pp), C.cast(self.g_out, pp), self.block):
            raise RuntimeError(self.lib.b200conv_group_last_error(self.group._g).decode())

    def diff(self):
        return max(float(np.max(np.abs(a - b))) for ys, yg in zip(self.y_single, self.y_group) for a, b in zip(ys, yg))

    def close(self):
        self.group.close()
        for e in self.members + self.twins:
            e.close()


def stats(us):
    a = np.asarray(us)
    return {"median_us": round(float(np.median(a)), 1), "p99_us": round(float(np.percentile(a, 99)), 1),
            "max_us": round(float(np.max(a)), 1)}


def run_leg(name, recipes, block, warm, calls, cfg=CUTS):
    leg = Leg(recipes, block, cfg)
    period = block / SR
    t_single, t_group, launches, dmax = [], [], [], 0.0
    t_next = time.perf_counter()
    for k in range(warm + calls):
        while time.perf_counter() < t_next:
            pass
        leg.feed(k)
        l0 = leg.group.launch_count
        t0 = time.perf_counter()
        leg.single()
        t1 = time.perf_counter()
        leg.grouped()
        t2 = time.perf_counter()
        if k >= warm:
            t_single.append((t1 - t0) * 1e6)
            t_group.append((t2 - t1) * 1e6)
            launches.append(leg.group.launch_count - l0)
            dmax = max(dmax, leg.diff())
        t_next += period
        t_next = max(t_next, time.perf_counter())       # a late callback does not start a burst of catch-up calls
    leg.close()
    return {"leg": name, "handles": len(recipes), "host_block": block, "calls": calls, "single": stats(t_single),
            "group": stats(t_group), "group_launches_per_callback": round(float(np.mean(launches)), 3),
            "max_abs_diff_vs_single": dmax}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        q = f"unavailable: {ex}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warm", type=int, default=200)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--legs", default="quad128,quad480,mixed,nocut")
    ap.add_argument("--sizes", default="1,2,4,8,16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    results = [{"card": card()}]
    sizes = [int(s) for s in a.sizes.split(",")]
    legs = a.legs.split(",")
    for n in sizes:
        if "quad128" in legs:
            results.append(run_leg("quad 128/8192, 10 s IRs", [quad(128, 8192, i) for i in range(n)], 128, a.warm, a.calls))
        if "quad480" in legs:
            results.append(run_leg("quad 512/8192, 10 s IRs, 480-sample calls", [quad(512, 8192, i) for i in range(n)], 480,
                                   a.warm, a.calls))
    if "mixed" in legs:
        results.append(run_leg("mixed: quad 128/8192, stereo 128/8192, stereo split-mode uniform 256 x 1100 (alone)",
                               [quad(128, 8192, 0), stereo(128, 8192, 1), stereo_uniform(256, 1100, 2)], 128,
                               a.warm, a.calls))
    if "nocut" in legs:
        n = max(sizes)
        results.append(run_leg("quad 128/8192, 10 s IRs, cuts off (no send scan)", [quad(128, 8192, i) for i in range(n)],
                               128, a.warm, a.calls, NOCUT))
    for r in results:
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE ONLY — ctypes loader for the oracle of the IR hot swap inside the chain (b200conv_chain_swap):
the plain-C restatement of processBlock's warmer, warm-up, crossfade and swap (oracle/hotswap_oracle.c, built into
oracle/libhotswap.so by oracle/hotswap.mk).

Only tests/, __graft_entry__.build() and tools/ may import this module.  The product package (reevr_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libhotswap.so")
_SOURCES = ("hotswap_oracle.c", "chain_oracle.c", "partconv_oracle.c")
_lib = None


def build(quiet: bool = True) -> None:
    out = subprocess.run(["make", "-C", _HERE, "-f", "hotswap.mk", "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("hot-swap oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


def _load() -> C.CDLL:
    global _lib
    if _lib is None:
        stale = not os.path.exists(_SO) or any(
            os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, s)) for s in _SOURCES)
        if stale:
            build()
        l = C.CDLL(_SO)
        l.oc_hs_create.restype = C.c_void_p
        l.oc_hs_create.argtypes = [C.c_double, C.c_float, C.c_int, C.c_float, C.c_int, C.c_int, C.c_float, C.c_float,
                                   C.c_float, C.c_int]
        l.oc_hs_destroy.restype = None
        l.oc_hs_destroy.argtypes = [C.c_void_p]
        for fn in ("oc_hs_set_live", "oc_hs_arm"):
            f = getattr(l, fn)
            f.restype = C.c_int
        l.oc_hs_set_live.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t]
        l.oc_hs_arm.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        for fn in ("oc_hs_state", "oc_hs_swapped"):
            f = getattr(l, fn)
            f.restype = C.c_int
            f.argtypes = [C.c_void_p]
        l.oc_hs_process.restype = None
        l.oc_hs_process.argtypes = [C.c_void_p] + [C.c_void_p] * 6 + [C.c_size_t]
        _lib = l
    return _lib


def _irs(irs):
    keep = [np.ascontiguousarray(a, dtype=np.float32) for a in irs]
    n = keep[0].size
    assert all(a.size == n for a in keep), "equally long IR channels"
    return keep, (C.c_void_p * len(keep))(*[a.ctypes.data for a in keep]), n


class HotSwapChain:
    """processBlock's send / wet chain with the convolver hot swap, one host callback per process() call."""

    def __init__(self, srate, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=0, predelay=0,
                 width=1.0, drygain=1.0, wetgain=1.0, true_stereo=True):
        self._l = _load()
        self._h = self._l.oc_hs_create(float(srate), lowcut_hz, lowcut_slope, highcut_hz, highcut_slope, predelay, width,
                                       drygain, wetgain, int(true_stereo))

    def set_live(self, head: int, tail: int, irs) -> None:
        keep, ptrs, n = _irs(irs)
        assert self._l.oc_hs_set_live(self._h, len(keep), head, tail, ptrs, n)

    def arm(self, head: int, tail: int, irs, host_block: int) -> None:
        """the load set holds the new IR and the next callback warms it up (loadState = kReady)"""
        keep, ptrs, n = _irs(irs)
        assert self._l.oc_hs_arm(self._h, len(keep), head, tail, ptrs, n, host_block)

    @property
    def state(self) -> int:
        """0 idle, 1 ready, 2 fading"""
        return int(self._l.oc_hs_state(self._h))

    @property
    def swapped(self) -> bool:
        """the last process() call completed the swap"""
        return bool(self._l.oc_hs_swapped(self._h))

    def process(self, dryL, dryR, ysend, yrev):
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in (dryL, dryR, ysend, yrev)]
        n = xs[0].size
        outs = [np.empty(n, np.float32) for _ in range(2)]
        self._l.oc_hs_process(self._h, *[a.ctypes.data for a in xs], outs[0].ctypes.data, outs[1].ctypes.data, n)
        return outs[0], outs[1]

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.oc_hs_destroy(self._h)
            self._h = None

"""TEST INFRASTRUCTURE ONLY — ctypes loaders for the checkers of the IR recalculation (b200conv_ir_recalc):

* ``ir_recalc`` / ``ir_recalc_len`` / ``decay_lut``: the plain-C restatement of Impulse::recalcImpulse
  (oracle/recalc_oracle.c, built into oracle/librecalc.so by oracle/recalc.mk);
* ``ref_ir_recalc``: the UNMODIFIED reference Impulse::recalcImpulse compiled from /root/reference into
  oracle/_ref/librefimpulse.so (oracle/ref_impulse_shim.cpp, oracle/recalc.mk).

Only tests/, __graft_entry__.build() and tools/ may import this module.  The product package (reevr_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_RECALC_SO = os.path.join(_HERE, "librecalc.so")
_REF_IMPULSE_SO = os.path.join(_HERE, "_ref", "librefimpulse.so")
_SOURCES = ("recalc_oracle.c", "chain_oracle.c", "partconv_oracle.c")
_libs: dict = {}


def build(quiet: bool = True) -> None:
    """Compile librecalc.so and, when /root/reference is present, _ref/librefimpulse.so."""
    out = subprocess.run(["make", "-C", _HERE, "-f", "recalc.mk", "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("recalc oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


def _lib(which: str) -> C.CDLL:
    if which not in _libs:
        stale = not os.path.exists(_RECALC_SO) or any(
            os.path.getmtime(_RECALC_SO) < os.path.getmtime(os.path.join(_HERE, s)) for s in _SOURCES)
        if stale:
            build()
        _libs[which] = C.CDLL(_RECALC_SO)
    return _libs[which]


class EqBand(C.Structure):
    """SVF::EQBand (src/dsp/SVF.h:28-33); mode = SVF::Mode 0..9 (LP BP HP LS HS PK BS HP6 LP6 Off)."""
    _fields_ = [("mode", C.c_int), ("freq", C.c_float), ("q", C.c_float), ("gain", C.c_float)]


def _bands(bands):
    bands = list(bands or [])
    arr = (EqBand * max(len(bands), 1))(*[EqBand(int(m), f, q, g) for m, f, q, g in bands])
    return len(bands), arr


def decay_lut(bands, srate: float, decay_rate: float) -> np.ndarray:
    """Impulse::applyDecayEQ's 2049-entry table from the bands (recalc_oracle.c::oc_decay_lut)."""
    lib = _lib("recalc")
    lib.oc_decay_lut.restype = None
    lib.oc_decay_lut.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_float, C.c_void_p]
    nb, arr = _bands(bands)
    lut = np.empty(2049, np.float64)
    lib.oc_decay_lut(C.addressof(arr), nb, float(srate), float(decay_rate), lut.ctypes.data)
    return lut


def ir_recalc_len(n: int, ir_srate: float, srate: float, stretch=0.0, trim_left=0.0, trim_right=0.0, **_) -> int:
    lib = _lib("recalc")
    lib.oc_ir_recalc_len.restype = C.c_size_t
    lib.oc_ir_recalc_len.argtypes = [C.c_size_t, C.c_double, C.c_double, C.c_float, C.c_float, C.c_float]
    return int(lib.oc_ir_recalc_len(n, float(ir_srate), float(srate), stretch, trim_left, trim_right))


def ir_recalc(irs, ir_srate=48000.0, srate=48000.0, stretch=0.0, autogain=True, reverse=False, trim_left=0.0, trim_right=0.0,
              gain=1.0, param_eq=(), decay_eq=(), decay_rate=1.0, clip=True, attack=0.0, decay=0.0):
    """C restatement of Impulse::recalcImpulse (recalc_oracle.c::oc_ir_recalc); irs = {LL, RR[, LR, RL]};
    bands: (mode, freq, q, gain) tuples.  Returns the recalculated channels."""
    lib = _lib("recalc")
    lib.oc_ir_recalc.restype = C.c_size_t
    lib.oc_ir_recalc.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_double, C.c_double, C.c_float, C.c_int, C.c_int,
                                 C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_float,
                                 C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_size_t]
    raws = [np.ascontiguousarray(a, dtype=np.float32) for a in irs]
    n = raws[0].size
    cap = max(ir_recalc_len(n, ir_srate, srate, stretch, trim_left, trim_right), 1)
    outs = [np.empty(cap, np.float32) for _ in raws]
    npq, pq = _bands(param_eq)
    ndc, dc = _bands(decay_eq)
    rp = (C.c_void_p * len(raws))(*[a.ctypes.data for a in raws])
    op = (C.c_void_p * len(raws))(*[a.ctypes.data for a in outs])
    m = lib.oc_ir_recalc(rp, len(raws), n, float(ir_srate), float(srate), stretch, int(autogain), int(reverse), trim_left,
                         trim_right, gain, npq, C.addressof(pq), ndc, C.addressof(dc), decay_rate, int(clip), attack, decay,
                         op, cap)
    assert m <= cap
    return [o[:m].copy() for o in outs]


def ref_impulse_available() -> bool:
    if os.path.exists(_REF_IMPULSE_SO):
        return True
    if os.path.isfile("/root/reference/src/dsp/Impulse.cpp"):
        build()
        return os.path.exists(_REF_IMPULSE_SO)
    return False


def ref_ir_recalc(irs, ir_srate=48000.0, srate=48000.0, stretch=0.0, reverse=False, trim_left=0.0, trim_right=0.0, gain=1.0,
                  param_eq=(), decay_eq=(), decay_rate=1.0, attack=0.0, decay=0.0):
    """The UNMODIFIED Impulse::recalcImpulse (oracle/ref_impulse_shim.cpp); auto gain and clip are always on there."""
    if "refimpulse" not in _libs:
        if not ref_impulse_available():
            raise RuntimeError("oracle/_ref/librefimpulse.so not built and /root/reference absent")
        l = C.CDLL(_REF_IMPULSE_SO)
        l.ref_impulse_recalc.restype = C.c_size_t
        l.ref_impulse_recalc.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_double, C.c_double, C.c_float, C.c_int,
                                         C.c_float, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                         C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_size_t]
        _libs["refimpulse"] = l
    l = _libs["refimpulse"]
    raws = [np.ascontiguousarray(a, dtype=np.float32) for a in irs]
    n = raws[0].size
    cap = max(ir_recalc_len(n, ir_srate, srate, stretch, trim_left, trim_right), 1)
    outs = [np.empty(cap, np.float32) for _ in raws]

    def flat(bands):
        v = np.array([x for b in (bands or []) for x in b] or [0.0], np.float32)
        return len(bands or []), v
    npq, pq = flat(param_eq)
    ndc, dc = flat(decay_eq)
    rp = (C.c_void_p * len(raws))(*[a.ctypes.data for a in raws])
    op = (C.c_void_p * len(raws))(*[a.ctypes.data for a in outs])
    m = l.ref_impulse_recalc(rp, len(raws), n, float(ir_srate), float(srate), stretch, int(reverse), trim_left, trim_right,
                             gain, npq, pq.ctypes.data, ndc, dc.ctypes.data, decay_rate, attack, decay, op, cap)
    assert m <= cap, (m, cap)
    return [o[:m].copy() for o in outs]

"""TEST INFRASTRUCTURE ONLY — ctypes loader for the oracle of b200conv_chain_update: chain parameter changes without a
reset, restated from processBlock's onSlider and per-block reads (oracle/params_oracle.c, built into
oracle/libparams.so by oracle/params.mk), and the reference's own Filter with setSlope (oracle/_ref/libreffilterswitch.so,
built by the same recipe where the reference's sources are present).

Only tests/, __graft_entry__.build() and tools/ may import this module.  The product package (reevr_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.hotswap import HotSwapChain

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libparams.so")
_REF_SO = os.path.join(_HERE, "_ref", "libreffilterswitch.so")
_SOURCES = ("params_oracle.c", "hotswap_oracle.c", "chain_oracle.c", "partconv_oracle.c")
_CHAIN_ARGS = [C.c_float, C.c_int, C.c_float, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_libs = {}


def build(quiet: bool = True) -> None:
    out = subprocess.run(["make", "-C", _HERE, "-f", "params.mk", "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("chain-parameter oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


def _load() -> C.CDLL:
    if "oc" not in _libs:
        stale = not os.path.exists(_SO) or any(
            os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, s)) for s in _SOURCES)
        if stale:
            build()
        l = C.CDLL(_SO)
        # the hot-swap restatement's entry points, as oracle/hotswap.py declares them
        l.oc_hs_destroy.restype = None
        l.oc_hs_destroy.argtypes = [C.c_void_p]
        for fn in ("oc_hs_set_live", "oc_hs_arm", "oc_hs_state", "oc_hs_swapped", "oc_hs_delay_size", "oc_chain_delay_size"):
            getattr(l, fn).restype = C.c_int
        l.oc_hs_set_live.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t]
        l.oc_hs_arm.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        for fn in ("oc_hs_state", "oc_hs_swapped", "oc_hs_delay_size", "oc_chain_delay_size"):
            getattr(l, fn).argtypes = [C.c_void_p]
        l.oc_hs_process.restype = None
        l.oc_hs_process.argtypes = [C.c_void_p] + [C.c_void_p] * 6 + [C.c_size_t]
        # the additions of params_oracle.c
        l.oc_hs_create_ref.restype = C.c_void_p
        l.oc_hs_create_ref.argtypes = [C.c_double] + _CHAIN_ARGS + [C.c_int]
        l.oc_hs_set_params.restype = None
        l.oc_hs_set_params.argtypes = [C.c_void_p] + _CHAIN_ARGS + [C.c_int]
        l.oc_chain_create_ref.restype = C.c_void_p
        l.oc_chain_create_ref.argtypes = [C.c_float] + _CHAIN_ARGS
        l.oc_chain_set.restype = None
        l.oc_chain_set.argtypes = [C.c_void_p] + _CHAIN_ARGS
        l.oc_chain_destroy.restype = None
        l.oc_chain_destroy.argtypes = [C.c_void_p]
        l.oc_chain_send.restype = None
        l.oc_chain_send.argtypes = [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_size_t]
        l.oc_filter_create.restype = C.c_void_p
        l.oc_filter_create.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
        l.oc_filter_set.restype = None
        l.oc_filter_set.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float]
        l.oc_filter_run.restype = None
        l.oc_filter_run.argtypes = [C.c_void_p, _f32p, _f32p, C.c_size_t]
        l.oc_filter_destroy.argtypes = [C.c_void_p]
        _libs["oc"] = l
    return _libs["oc"]


def _chain_args(cfg):
    return (cfg["lowcut_hz"], cfg["lowcut_slope"], cfg["highcut_hz"], cfg["highcut_slope"], cfg["predelay"],
            cfg["width"], cfg["drygain"], cfg["wetgain"])


def _cfg(srate, lowcut_hz=20.0, lowcut_slope=0, highcut_hz=20000.0, highcut_slope=0, predelay=0, width=1.0,
         drygain=1.0, wetgain=1.0, true_stereo=True):
    return dict(srate=srate, lowcut_hz=lowcut_hz, lowcut_slope=lowcut_slope, highcut_hz=highcut_hz,
                highcut_slope=highcut_slope, predelay=predelay, width=width, drygain=drygain, wetgain=wetgain,
                true_stereo=true_stereo)


class ParamHotSwapChain(HotSwapChain):
    """HotSwapChain on the reference's delay line (D = (int)(2 * srate), grown past the predelay), with set(**cfg):
    onSlider + the per-block reads, effective from the next process() call."""

    def __init__(self, srate, **kw):
        self._l = _load()
        self._srate = srate
        c = _cfg(srate, **kw)
        self._h = self._l.oc_hs_create_ref(float(srate), *_chain_args(c), int(c["true_stereo"]))

    def set(self, srate, **kw):
        assert srate == self._srate, "a new rate is prepareToPlay"
        c = _cfg(srate, **kw)
        self._l.oc_hs_set_params(self._h, *_chain_args(c), int(c["true_stereo"]))

    @property
    def delay_size(self) -> int:
        """the delay line's length D"""
        return int(self._l.oc_hs_delay_size(self._h))


class ParamChain:
    """The send side of the chain (filters + predelay) on the reference's delay line, with set(**cfg)."""

    def __init__(self, srate, **kw):
        self._l = _load()
        self._srate = srate
        self._h = self._l.oc_chain_create_ref(float(srate), *_chain_args(_cfg(srate, **kw)))

    def set(self, srate, **kw):
        assert srate == self._srate, "a new rate is prepareToPlay"
        self._l.oc_chain_set(self._h, *_chain_args(_cfg(srate, **kw)))

    def send(self, dryL, dryR, ysend):
        xs = [np.ascontiguousarray(a, dtype=np.float32) for a in (dryL, dryR, ysend)]
        a, b = np.empty_like(xs[0]), np.empty_like(xs[1])
        self._l.oc_chain_send(self._h, *xs, a, b, xs[0].size)
        return a, b

    @property
    def delay_size(self) -> int:
        return int(self._l.oc_chain_delay_size(self._h))

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.oc_chain_destroy(self._h)
            self._h = None


class SwitchFilter:
    """The restated Filter with set(slope, srate, freq, q) = setSlope + init without reset (onSlider)."""

    def __init__(self, slope: int, mode: int, srate: float, freq: float, q: float):
        self._l = _load()
        self._h = self._l.oc_filter_create(slope, mode, srate, freq, q)

    def set(self, slope: int, srate: float, freq: float, q: float) -> None:
        self._l.oc_filter_set(self._h, slope, srate, freq, q)

    def run(self, x) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        self._l.oc_filter_run(self._h, x, y, x.size)
        return y

    def __del__(self):
        if getattr(self, "_h", None):
            self._l.oc_filter_destroy(self._h)
            self._h = None


def ref_switch_filter_available() -> bool:
    if not os.path.exists(_REF_SO):
        build()
    return os.path.exists(_REF_SO)


class RefSwitchFilter(SwitchFilter):
    """The unmodified reference Filter: setSlope + init, no reset (oracle/_ref/libreffilterswitch.so)."""

    def __init__(self, slope: int, mode: int, srate: float, freq: float, q: float):
        if "ref" not in _libs:
            if not ref_switch_filter_available():
                raise RuntimeError("oracle/_ref/libreffilterswitch.so not built and the reference's sources absent")
            l = C.CDLL(_REF_SO)
            l.ref_filter_create.restype = C.c_void_p
            l.ref_filter_create.argtypes = [C.c_int, C.c_int]
            l.ref_filter_destroy.argtypes = [C.c_void_p]
            l.ref_filter_init.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float]
            l.ref_filter_reset.argtypes = [C.c_void_p, C.c_float]
            l.ref_filter_set_slope.argtypes = [C.c_void_p, C.c_int]
            l.ref_filter_run.argtypes = [C.c_void_p, _f32p, _f32p, C.c_size_t]
            _libs["ref"] = l
        self._r = _libs["ref"]
        self._p = self._r.ref_filter_create(slope, mode)
        self._r.ref_filter_init(self._p, srate, freq, q)
        self._r.ref_filter_reset(self._p, 0.0)

    def set(self, slope: int, srate: float, freq: float, q: float) -> None:
        self._r.ref_filter_set_slope(self._p, slope)
        self._r.ref_filter_init(self._p, srate, freq, q)

    def run(self, x) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        self._r.ref_filter_run(self._p, x, y, x.size)
        return y

    def __del__(self):
        if getattr(self, "_p", None):
            self._r.ref_filter_destroy(self._p)
            self._p = None


"""Python bindings of the Adaptive AOV oracle (oracle/_build/liboracle_adaptive_aov.so, built from
oracle_adaptive_aov/adaptive_aov.cpp) — TEST INFRASTRUCTURE, like oracle/pyoracle.py.

``AdaptiveAovOracleScene`` is an ``AdaptiveOracleScene`` backed by that library (the Adaptive-sampler oracle with the AOV records
added), so it has every oracle and Adaptive method plus ``render_samples_adaptive_aov`` with the signature of
``tray_rust_b200.api.Scene.render_samples_adaptive_aov``.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_adaptive import pyadaptive as A
from tray_rust_b200 import _ffi as F
from tray_rust_b200.api import _cfg


def load():
    lib = O.load_oracle("adaptive_aov")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_adaptive_aov_ready"):
        a = A.load()
        for name in ("orc_render_adaptive", "orc_render_samples_adaptive", "orc_adaptive_schedule"):  # as pyadaptive declares them
            getattr(lib, name).argtypes = getattr(a, name).argtypes
        vp = C.c_void_p
        lib.orc_render_samples_adaptive_aov.argtypes = [vp, C.POINTER(F.RenderCfg), C.POINTER(F.Adaptive), C.c_size_t, vp, vp, vp, C.POINTER(F.Stats),
                                                        C.c_int]
        lib._adaptive_aov_ready = True
    return lib


class AdaptiveAovOracleScene(A.AdaptiveOracleScene):
    """The Adaptive-sampler oracle with the AOV record of every slot it takes (adaptive_aov.cpp)."""

    def __init__(self, desc, baseline=False):
        load()
        O.OracleScene.__init__(self, desc, libm="adaptive_aov", baseline=baseline)

    def render_samples_adaptive_aov(self, min_spp, max_spp, threads=0, **kw):
        """(samples as render_samples_adaptive, AOV records as AOV_SAMPLE_DTYPE in the same layout, unused slots zero; pixel_spp;
        Stats)."""
        cfg = _cfg(**kw)
        n = self._n_selected_blocks(cfg) * 64 * self.adaptive_schedule(min_spp, max_spp)[3]
        out, aov = np.zeros(n, F.SAMPLE_DTYPE), np.zeros(n, F.AOV_SAMPLE_DTYPE)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.orc_render_samples_adaptive_aov(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), n, F.ptr(out), F.ptr(aov),
                                                              F.ptr(spp), C.byref(st), threads))
        return out, aov, spp, st

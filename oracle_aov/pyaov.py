"""Python bindings of the AOV oracle (oracle/_build/liboracle_aov.so, built from oracle_aov/aov.cpp) — TEST INFRASTRUCTURE, like
oracle/pyoracle.py.

``AovOracleScene`` is a ``RefitOracleScene`` backed by that library (the ray-query oracle with the mesh refit and the AOV records
added), so it has every oracle, ray-query and refit method plus ``render_samples_aov`` with the signature of
``tray_rust_b200.api.Scene.render_samples_aov``.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_refit import pyrefit as R
from tray_rust_b200 import _ffi as F


def load():
    lib = O.load_oracle("aov")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_aov_ready"):
        r = R.load()
        for name in R._QUERY_FUNCS + ("orc_scene_refit_mesh",):  # as pyrefit declares them
            getattr(lib, name).argtypes = getattr(r, name).argtypes
        vp = C.c_void_p
        lib.orc_render_samples_aov.argtypes = [vp, C.POINTER(F.RenderCfg), C.c_size_t, vp, vp, C.POINTER(F.Stats)]
        lib._aov_ready = True
    return lib


class AovOracleScene(R.RefitOracleScene):
    """The ray-query oracle with Mesh refits and the AOV record of every camera sample (aov.cpp)."""

    def __init__(self, desc, baseline=False):
        load()
        O.OracleScene.__init__(self, desc, libm="aov", baseline=baseline)

    def render_samples_aov(self, **kw):
        """(samples as render_samples, AOV records as AOV_SAMPLE_DTYPE in the same order, Stats)."""
        cfg = O._cfg(**kw)
        n = self._n_samples(cfg)
        out, aov = np.zeros(n, F.SAMPLE_DTYPE), np.zeros(n, F.AOV_SAMPLE_DTYPE)
        st = F.Stats()
        self._check(self._lib.orc_render_samples_aov(self._h, C.byref(cfg), n, F.ptr(out), F.ptr(aov), C.byref(st)))
        return out, aov, st

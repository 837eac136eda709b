"""Python bindings of the Adaptive-sampler oracle (oracle/_build/liboracle_adaptive.so, built from
oracle_adaptive/adaptive.cpp) — TEST INFRASTRUCTURE, like oracle/pyoracle.py.

``AdaptiveOracleScene`` is an ``OracleScene`` backed by that library (the detmath oracle with the Adaptive sampler added), so
it has every oracle method plus ``render_adaptive``, ``render_samples_adaptive`` and ``adaptive_schedule`` with the
signatures of ``tray_rust_b200.api.Scene``.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from tray_rust_b200 import _ffi as F
from tray_rust_b200.api import _cfg


def load():
    lib = O.load_oracle("adaptive")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_adaptive_ready"):
        vp, sz = C.c_void_p, C.c_size_t
        lib.orc_render_adaptive.argtypes = [vp, C.POINTER(F.RenderCfg), C.POINTER(F.Adaptive), vp, vp, C.POINTER(F.Stats), C.c_int]
        lib.orc_render_samples_adaptive.argtypes = [vp, C.POINTER(F.RenderCfg), C.POINTER(F.Adaptive), sz, vp, vp, C.POINTER(F.Stats), C.c_int]
        lib.orc_adaptive_schedule.argtypes = [C.POINTER(F.Adaptive), vp]
        lib._adaptive_ready = True
    return lib


class AdaptiveOracleScene(O.OracleScene):
    """The oracle with thread_work driving sampler::Adaptive, literally (full per-pixel sample list, literal decision loop)."""

    def __init__(self, desc, baseline=False):
        load()
        super().__init__(desc, libm="adaptive", baseline=baseline)

    def adaptive_schedule(self, min_spp, max_spp):
        """Adaptive::new's rounded (min, max, step) and the largest per-pixel sample count."""
        out = np.zeros(4, np.uint32)
        self._check(self._lib.orc_adaptive_schedule(C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(out)))
        return tuple(int(x) for x in out)

    def render_adaptive(self, min_spp, max_spp, film=None, threads=0, **kw):
        """Returns (film, pixel_spp, Stats) like Scene.render_adaptive."""
        cfg = _cfg(**kw)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.orc_render_adaptive(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(film), F.ptr(spp), C.byref(st),
                                                  threads))
        return film, spp, st

    def render_samples_adaptive(self, min_spp, max_spp, threads=0, **kw):
        """Returns (records of (blocks, 64, max_per_pixel) flattened, unused slots zero; pixel_spp; Stats)."""
        cfg = _cfg(**kw)
        n = self._n_selected_blocks(cfg) * 64 * self.adaptive_schedule(min_spp, max_spp)[3]
        out = np.zeros(n, F.SAMPLE_DTYPE)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.orc_render_samples_adaptive(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), n, F.ptr(out), F.ptr(spp),
                                                          C.byref(st), threads))
        return out, spp, st

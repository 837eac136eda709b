"""Python binding of the motion-vector oracle (oracle/_build/liboracle_motion.so, built from oracle_motion/motion.cpp) — TEST
INFRASTRUCTURE, like oracle/pyoracle.py.

``MotionOracleScene`` is a ``QueryOracleScene`` backed by that library. It remembers the (start, end) of its last update_frame, which
an animated fov is sampled at, and adds ``motion_samples`` (the records of a LowDiscrepancy render, the order of
``Scene.render_samples_aov(motion=...)``) and ``motion_at`` (the records of caller camera samples).
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_queries import pyqueries as Q
from tray_rust_b200 import _ffi as F


def load():
    lib = O.load_oracle("motion")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_motion_ready"):
        q = Q.load()
        for name in ("orc_intersect_records", "orc_occluded", "orc_illumination", "orc_bsdf_eval", "orc_bsdf_sample", "orc_light_sample",
                     "orc_light_pdf", "orc_emitted", "orc_scene_lights", "orc_film_write"):  # as pyqueries declares them
            getattr(lib, name).argtypes = getattr(q, name).argtypes
        vp, sz = C.c_void_p, C.c_size_t
        lib.orc_motion_samples.argtypes = [vp, C.POINTER(F.RenderCfg), sz, F.f32, F.f32, F.f32, vp]
        lib.orc_motion_at.argtypes = [vp, sz, vp, F.f32, F.f32, F.f32, vp]
        lib._motion_ready = True
    return lib


class MotionOracleScene(Q.QueryOracleScene):
    """The ray-query oracle with include/trb.h "Motion vectors" (motion.cpp)."""

    def __init__(self, desc, baseline=False):
        load()
        O.OracleScene.__init__(self, desc, libm="motion", baseline=baseline)
        self._frame = (0.0, 0.0)

    def update_frame(self, frame=0, start=0.0, end=0.0):
        super().update_frame(frame, start, end)
        self._frame = (start, end)

    def frame_step(self):
        return float(np.float32(self._desc.film.scene_time) / np.float32(self._desc.film.frames))

    def _dt(self, dt):
        return -self.frame_step() if dt is None else float(dt)

    def motion_samples(self, dt=None, **kw):
        """MOTION_SAMPLE_DTYPE records of the render's camera samples (render_cfg keywords as render_samples), dt None: one frame back"""
        from tray_rust_b200.api import _cfg
        cfg = _cfg(**kw)
        n = self._n_samples(cfg)
        out = np.zeros(n, F.MOTION_SAMPLE_DTYPE)
        self._check(self._lib.orc_motion_samples(self._h, C.byref(cfg), n, self._dt(dt), *self._frame, F.ptr(out)))
        return out

    def motion_at(self, x, y, tm, dt=None):
        """MOTION_SAMPLE_DTYPE records of caller camera samples: raster positions x, y and time samples tm in [0, 1)"""
        xyt = np.ascontiguousarray(np.stack([np.asarray(x, np.float32), np.asarray(y, np.float32),
                                             np.broadcast_to(np.asarray(tm, np.float32), np.shape(x))], axis=-1), dtype=np.float32)
        out = np.zeros(len(xyt), F.MOTION_SAMPLE_DTYPE)
        self._check(self._lib.orc_motion_at(self._h, len(xyt), F.ptr(xyt), self._dt(dt), *self._frame, F.ptr(out)))
        return out

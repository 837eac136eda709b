"""Python binding of the variance temporal denoise oracle (oracle/_build/liboracle_variance_temporal.so, built from
oracle_variance_temporal/variance_temporal.cpp) — TEST INFRASTRUCTURE, like oracle_moment_gradient/pymomentgradient.py.

``History`` is an oracle history of this library. ``denoise_variance_temporal(scene, history, ...)`` and
``denoise_variance_temporal_gradient(scene, history, ...)`` take a ``Scene`` of this library after ``update_frame``;
``denoise_variance_temporal_lambda_frame`` takes an explicit ``oracle_gradient.pygradient.Frame`` and a caller lambda per stratum.
Every call returns (rgbw, motion, history_length, variance, lambda per pixel); the plain call's lambda is all 0.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_gradient.pygradient import Frame, make_frame  # noqa: F401  (the frame type this library takes)
from tray_rust_b200 import _ffi as F

_lib = None


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(O.oracle_path("variance_temporal"))
        vp = C.c_void_p
        lib.orc_gradient_history_create.argtypes = [C.POINTER(vp)]
        lib.orc_gradient_history_destroy.argtypes = [vp]
        lib.orc_gradient_history_reset.argtypes = [vp]
        lib.orc_denoise_variance_temporal_lambda_frame.argtypes = [F.u32, F.u32, C.POINTER(Frame), vp, C.POINTER(F.DenoiseFrame), vp,
                                                                   C.POINTER(F.DenoiseGradientParams), vp, vp, vp, vp, vp, vp]
        lib.orc_denoise_variance_temporal.argtypes = [vp, vp, C.POINTER(F.DenoiseFrame), vp, C.POINTER(F.DenoiseTemporalParams),
                                                      vp, vp, vp, vp]
        lib.orc_denoise_variance_temporal_gradient.argtypes = [vp, vp, C.POINTER(F.DenoiseFrame), vp, C.POINTER(F.DenoiseGradientParams),
                                                               F.u32, vp, vp, vp, vp, vp]
        lib.orc_scene_create.argtypes = [vp, C.POINTER(vp)]
        lib.orc_scene_update_frame.argtypes = [vp, F.u32, F.f32, F.f32]
        lib.orc_scene_destroy.argtypes = [vp]
        _lib = lib
    return _lib


class History:
    def __init__(self):
        h = C.c_void_p()
        load().orc_gradient_history_create(C.byref(h))
        self._h = h

    def reset(self):
        load().orc_gradient_history_reset(self._h)

    def __del__(self):
        if _lib is not None and getattr(self, "_h", None):
            _lib.orc_gradient_history_destroy(self._h)


class Scene:
    """An oracle scene in this library (its own copy of oracle.cpp)"""

    def __init__(self, desc):
        self._desc = desc
        h = C.c_void_p()
        rc = load().orc_scene_create(C.byref(desc), C.byref(h))
        if rc != F.TRB_OK:
            raise ValueError("orc_scene_create failed (status %d)" % rc)
        self._h = h
        self.width, self.height = desc.film.width, desc.film.height

    def update_frame(self, frame=0, start=0.0, end=0.0):
        load().orc_scene_update_frame(self._h, frame, start, end)

    def __del__(self):
        if _lib is not None and getattr(self, "_h", None):
            _lib.orc_scene_destroy(self._h)


def _call(fn, lead, mid, h, w, colour, aovs, prm, with_lambda=True):
    ins = [np.ascontiguousarray(a, dtype=np.float32) for a in (colour, aovs["albedo_w"], aovs["normal_w"])]
    near = np.ascontiguousarray(aovs["nearest"], dtype=np.uint64)
    lum = np.ascontiguousarray(aovs["lum_w"], dtype=np.float32)
    for a in ins + [lum]:
        assert a.shape == (h, w, 4)
    assert near.shape == (h, w)
    out, motion = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 2), np.float32)
    hl, var, lam = np.zeros((h, w), np.uint32), np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
    d_in = F.DenoiseFrame(*(a.ctypes.data for a in ins), near.ctypes.data)
    tail = [out.ctypes.data, motion.ctypes.data, hl.ctypes.data, var.ctypes.data] + ([lam.ctypes.data] if with_lambda else [])
    rc = fn(*lead, C.byref(d_in), lum.ctypes.data, C.byref(prm), *mid, *tail)
    if rc != F.TRB_OK:
        raise ValueError("the variance temporal denoise oracle refused the arguments (status %d)" % rc)
    return out, motion, hl, var, lam


def denoise_variance_temporal(scene, history, colour, aovs, **params):
    """orc_denoise_variance_temporal over host arrays (the inputs of Scene.denoise_variance_temporal)"""
    from tray_rust_b200.api import _temporal_params
    return _call(load().orc_denoise_variance_temporal, (scene._h, history._h), (), scene.height, scene.width, colour, aovs,
                 _temporal_params(params), with_lambda=False)


def denoise_variance_temporal_gradient(scene, history, colour, aovs, seed, **params):
    """orc_denoise_variance_temporal_gradient over host arrays (the inputs of Scene.denoise_variance_temporal_gradient)"""
    from tray_rust_b200.api import _gradient_params
    return _call(load().orc_denoise_variance_temporal_gradient, (scene._h, history._h), (seed % (1 << 32),), scene.height, scene.width,
                 colour, aovs, _gradient_params(params))


def denoise_variance_temporal_lambda_frame(frame, history, colour, aovs, lam_s, **params):
    """orc_denoise_variance_temporal_lambda_frame: the contract with a caller lambda per stratum over an explicit Frame; the image
    size is the films' shape"""
    from tray_rust_b200.api import _gradient_params
    h, w = colour.shape[:2]
    lam_s = np.ascontiguousarray(lam_s, np.float32)
    assert lam_s.shape == (((w + 2) // 3) * ((h + 2) // 3),)
    return _call(load().orc_denoise_variance_temporal_lambda_frame, (w, h, C.byref(frame), history._h), (lam_s.ctypes.data,), h, w, colour,
                 aovs, _gradient_params(params))

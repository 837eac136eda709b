"""Python binding of the temporal denoiser oracle (oracle/_build/liboracle_temporal.so, built from oracle_temporal/temporal.cpp) —
TEST INFRASTRUCTURE, like oracle_denoise/pydenoise.py.

``History`` is an oracle history. ``denoise_temporal(scene, history, ...)`` takes an oracle scene handle after
``orc_scene_update_frame`` (``oracle.pyoracle.OrcScene``); ``denoise_temporal_frame`` takes an explicit ``Frame`` instead.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from tray_rust_b200 import _ffi as F

_lib = None


class Frame(C.Structure):
    """orc_temporal_frame: row-major 4x4 px_to_cam, cam_mat (cam_world at shutter-open) and its inverse, the fov scaling, and the
    instances' world -> object (inv) and object -> world (mat) matrices, n x 16 floats each"""
    _fields_ = [("px_to_cam", F.f32 * 16), ("cam_mat", F.f32 * 16), ("cam_inv", F.f32 * 16), ("scaling", F.f32 * 3),
                ("n_instances", F.u32), ("inv", C.c_void_p), ("mat", C.c_void_p)]


def make_frame(px_to_cam, cam_mat, cam_inv, tan_fov, inv, mat):
    """A Frame over numpy matrices (inv / mat: (n, 4, 4)); the arrays are kept on the frame"""
    inv, mat = (np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 16) for a in (inv, mat))
    f = Frame()
    for name, m in (("px_to_cam", px_to_cam), ("cam_mat", cam_mat), ("cam_inv", cam_inv)):
        getattr(f, name)[:] = [float(x) for x in np.asarray(m, np.float32).ravel()]
    f.scaling[:] = [float(np.float32(tan_fov)), float(np.float32(tan_fov)), 1.0]
    f.n_instances = len(inv)
    f.inv, f.mat = inv.ctypes.data, mat.ctypes.data
    f._keep = (inv, mat)
    return f


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(O.oracle_path("temporal"))
        vp = C.c_void_p
        lib.orc_denoise_history_create.argtypes = [C.POINTER(vp)]
        lib.orc_denoise_history_destroy.argtypes = [vp]
        lib.orc_denoise_history_reset.argtypes = [vp]
        tail = [C.POINTER(F.DenoiseInput), C.POINTER(F.DenoiseTemporalParams), vp, vp, vp]
        lib.orc_denoise_temporal_frame.argtypes = [F.u32, F.u32, C.POINTER(Frame), vp] + tail
        lib.orc_denoise_temporal.argtypes = [vp, vp] + tail
        lib.orc_scene_create.argtypes = [vp, C.POINTER(vp)]
        lib.orc_scene_update_frame.argtypes = [vp, F.u32, F.f32, F.f32]
        lib.orc_scene_destroy.argtypes = [vp]
        _lib = lib
    return _lib


class History:
    def __init__(self):
        h = C.c_void_p()
        load().orc_denoise_history_create(C.byref(h))
        self._h = h

    def reset(self):
        load().orc_denoise_history_reset(self._h)

    def __del__(self):
        if _lib is not None and getattr(self, "_h", None):
            _lib.orc_denoise_history_destroy(self._h)


class Scene:
    """An oracle scene in this library (its own copy of oracle.cpp), for orc_denoise_temporal"""

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


def _call(fn, lead, h, w, colour_a, colour_b, aovs, params):
    from tray_rust_b200.api import _temporal_params
    ins = [np.ascontiguousarray(a, dtype=np.float32) for a in (colour_a, colour_b, aovs["albedo_w"], aovs["normal_w"])]
    near = np.ascontiguousarray(aovs["nearest"], dtype=np.uint64)
    for a in ins:
        assert a.shape == (h, w, 4)
    assert near.shape == (h, w)
    prm = _temporal_params(params)
    out, motion, hl = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 2), np.float32), np.zeros((h, w), np.uint32)
    d_in = F.DenoiseInput(*(a.ctypes.data for a in ins), near.ctypes.data)
    rc = fn(*lead, C.byref(d_in), C.byref(prm), out.ctypes.data, motion.ctypes.data, hl.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("the temporal denoise oracle refused the arguments (status %d)" % rc)
    return out, motion, hl


def denoise_temporal(scene, history, colour_a, colour_b, aovs, **params):
    """orc_denoise_temporal over host arrays (the inputs of Scene.denoise_temporal). Returns (rgbw, motion, history_length)."""
    return _call(load().orc_denoise_temporal, (scene._h, history._h), scene.height, scene.width, colour_a, colour_b, aovs, params)


def denoise_temporal_frame(frame, history, colour_a, colour_b, aovs, **params):
    """orc_denoise_temporal_frame: the same over an explicit Frame; the image size is the films' shape"""
    h, w = colour_a.shape[:2]
    return _call(load().orc_denoise_temporal_frame, (w, h, C.byref(frame), history._h), h, w, colour_a, colour_b, aovs, params)

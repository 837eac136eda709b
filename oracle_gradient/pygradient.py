"""Python binding of the temporal gradient oracle (oracle/_build/liboracle_gradient.so, built from oracle_gradient/gradient.cpp) —
TEST INFRASTRUCTURE, like oracle_temporal/pytemporal.py.

``History`` is an oracle history with gradient records. ``denoise_temporal_gradient(scene, history, ...)`` takes an oracle ``Scene``
after ``update_frame``; ``lambda_frame`` and ``denoise_temporal_lambda_frame`` take an explicit ``Frame`` and caller records instead.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from tray_rust_b200 import _ffi as F

_lib = None

# orc_gradient_record: (p_o, inst) (o, time) (d, key) (lum, pad)
RECORD_DTYPE = np.dtype([("p_o", "<f4", 3), ("inst", "<u4"), ("o", "<f4", 3), ("time", "<f4"), ("d", "<f4", 3), ("key", "<u4"),
                         ("lum", "<f4"), ("pad", "<u4", 3)])


class Frame(C.Structure):
    """orc_gradient_frame: oracle_temporal's Frame plus the frame's shutter_open"""
    _fields_ = [("px_to_cam", F.f32 * 16), ("cam_mat", F.f32 * 16), ("cam_inv", F.f32 * 16), ("scaling", F.f32 * 3),
                ("n_instances", F.u32), ("inv", C.c_void_p), ("mat", C.c_void_p), ("shutter_open", F.f32)]


def make_frame(px_to_cam, cam_mat, cam_inv, tan_fov, inv, mat, shutter_open=0.0):
    """A Frame over numpy matrices (inv / mat: (n, 4, 4)); the arrays are kept on the frame"""
    inv, mat = (np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 16) for a in (inv, mat))
    f = Frame()
    for name, m in (("px_to_cam", px_to_cam), ("cam_mat", cam_mat), ("cam_inv", cam_inv)):
        getattr(f, name)[:] = [float(x) for x in np.asarray(m, np.float32).ravel()]
    f.scaling[:] = [float(np.float32(tan_fov)), float(np.float32(tan_fov)), 1.0]
    f.n_instances = len(inv)
    f.inv, f.mat = inv.ctypes.data, mat.ctypes.data
    f.shutter_open = shutter_open
    f._keep = (inv, mat)
    return f


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(O.oracle_path("gradient"))
        vp = C.c_void_p
        lib.orc_gradient_history_create.argtypes = [C.POINTER(vp)]
        lib.orc_gradient_history_destroy.argtypes = [vp]
        lib.orc_gradient_history_reset.argtypes = [vp]
        lib.orc_gradient_lambda_frame.argtypes = [F.u32, F.u32, C.POINTER(Frame), vp, F.u32, vp, vp, F.f32, vp, vp, vp, F.f32, F.f32, F.u32,
                                                  vp, vp, vp, vp]
        lib.orc_denoise_temporal_lambda_frame.argtypes = [F.u32, F.u32, C.POINTER(Frame), vp, C.POINTER(F.DenoiseInput),
                                                          C.POINTER(F.DenoiseGradientParams), vp, vp, vp, vp, vp]
        lib.orc_denoise_temporal_gradient.argtypes = [vp, vp, C.POINTER(F.DenoiseInput), C.POINTER(F.DenoiseGradientParams), F.u32,
                                                      vp, vp, vp, vp]
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
    """An oracle scene in this library (its own copy of oracle.cpp), for orc_denoise_temporal_gradient"""

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


def _inputs(h, w, colour_a, colour_b, aovs):
    ins = [np.ascontiguousarray(a, dtype=np.float32) for a in (colour_a, colour_b, aovs["albedo_w"], aovs["normal_w"])]
    near = np.ascontiguousarray(aovs["nearest"], dtype=np.uint64)
    for a in ins:
        assert a.shape == (h, w, 4)
    assert near.shape == (h, w)
    return ins, near, F.DenoiseInput(*(a.ctypes.data for a in ins), near.ctypes.data)


def denoise_temporal_gradient(scene, history, colour_a, colour_b, aovs, seed, **params):
    """orc_denoise_temporal_gradient over host arrays (the inputs of Scene.denoise_temporal_gradient). Returns (rgbw, motion,
    history_length, lambda)."""
    from tray_rust_b200.api import _gradient_params
    h, w = scene.height, scene.width
    keep = _inputs(h, w, colour_a, colour_b, aovs)
    prm = _gradient_params(params)
    out, motion, hl, lam = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 2), np.float32), np.zeros((h, w), np.uint32), np.zeros((h, w), np.float32)
    rc = load().orc_denoise_temporal_gradient(scene._h, history._h, C.byref(keep[2]), C.byref(prm), seed % (1 << 32), out.ctypes.data,
                                              motion.ctypes.data, hl.ctypes.data, lam.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("the temporal gradient oracle refused the arguments (status %d)" % rc)
    return out, motion, hl, lam


def lambda_frame(w, h, frame, records, n_prev, mat_prev, cam_mat_prev, shutter_open_prev, l_cur, normal_w, nearest, depth_tolerance=0.05,
                 normal_threshold=0.9, iterations=3):
    """orc_gradient_lambda_frame: steps 1-2 over caller records (RECORD_DTYPE, one per stratum) and re-shaded luminances l_cur per
    target stratum. Returns (slot uint64, rays ILLUM_RAY_DTYPE, dm (S, 3), lambda (S,))."""
    S = ((w + 2) // 3) * ((h + 2) // 3)
    records = np.ascontiguousarray(records, RECORD_DTYPE)
    mat_prev = np.ascontiguousarray(mat_prev, np.float32).reshape(-1, 16)
    cam_mat_prev = np.ascontiguousarray(cam_mat_prev, np.float32).reshape(16)
    l_cur = np.ascontiguousarray(l_cur, np.float32)
    normal_w = np.ascontiguousarray(normal_w, np.float32)
    nearest = np.ascontiguousarray(nearest, np.uint64)
    assert records.shape == (S,) and l_cur.shape == (S,) and normal_w.shape == (h, w, 4) and nearest.shape == (h, w)
    slot, rays, dm, lam = np.zeros(S, np.uint64), np.zeros(S, F.ILLUM_RAY_DTYPE), np.zeros((S, 3), np.float32), np.zeros(S, np.float32)
    rc = load().orc_gradient_lambda_frame(w, h, C.byref(frame), records.ctypes.data, n_prev, mat_prev.ctypes.data, cam_mat_prev.ctypes.data,
                                          shutter_open_prev, l_cur.ctypes.data, normal_w.ctypes.data, nearest.ctypes.data, depth_tolerance,
                                          normal_threshold, iterations, slot.ctypes.data, rays.ctypes.data, dm.ctypes.data, lam.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("orc_gradient_lambda_frame refused the arguments (status %d)" % rc)
    return slot, rays, dm, lam


def denoise_temporal_lambda_frame(frame, history, colour_a, colour_b, aovs, lam_s, **params):
    """orc_denoise_temporal_lambda_frame: "Temporal denoising" with a caller lambda per stratum. Returns (rgbw, motion,
    history_length, lambda per pixel)."""
    from tray_rust_b200.api import _gradient_params
    h, w = colour_a.shape[:2]
    keep = _inputs(h, w, colour_a, colour_b, aovs)
    lam_s = np.ascontiguousarray(lam_s, np.float32)
    assert lam_s.shape == (((w + 2) // 3) * ((h + 2) // 3),)
    prm = _gradient_params(params)
    out, motion, hl, lam = np.zeros((h, w, 4), np.float32), np.zeros((h, w, 2), np.float32), np.zeros((h, w), np.uint32), np.zeros((h, w), np.float32)
    rc = load().orc_denoise_temporal_lambda_frame(w, h, C.byref(frame), history._h, C.byref(keep[2]), C.byref(prm), lam_s.ctypes.data,
                                                  out.ctypes.data, motion.ctypes.data, hl.ctypes.data, lam.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("the temporal gradient oracle refused the arguments (status %d)" % rc)
    return out, motion, hl, lam

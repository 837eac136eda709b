"""Python binding of the denoiser oracle (oracle/_build/liboracle_denoise.so, built from oracle_denoise/denoise.cpp) — TEST
INFRASTRUCTURE, like oracle/pyoracle.py.

``denoise`` takes the arguments of ``tray_rust_b200.api.Scene.denoise`` without a scene: the image size is the films' shape.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from tray_rust_b200 import _ffi as F

_lib = None


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(O.oracle_path("denoise"))
        lib.orc_denoise.argtypes = [F.u32, F.u32, C.POINTER(F.DenoiseInput), C.POINTER(F.DenoiseParams), C.c_void_p]
        _lib = lib
    return _lib


def denoise(colour_a, colour_b, aovs, **params):
    """orc_denoise over host arrays: colour_a / colour_b / aovs["albedo_w"] / aovs["normal_w"] of shape (h, w, 4) float32 and
    aovs["nearest"] of shape (h, w) uint64. Returns the (h, w, 4) float32 film; raises ValueError where trb_denoise refuses."""
    h, w = colour_a.shape[:2]
    ins = [np.ascontiguousarray(a, dtype=np.float32) for a in (colour_a, colour_b, aovs["albedo_w"], aovs["normal_w"])]
    near = np.ascontiguousarray(aovs["nearest"], dtype=np.uint64)
    for a in ins:
        assert a.shape == (h, w, 4)
    assert near.shape == (h, w)
    p = dict(F.DENOISE_DEFAULTS, **params)
    prm = F.DenoiseParams(p["iterations"], p["normal_power"], p["sigma_luminance"], p["sigma_depth"])
    out = np.zeros((h, w, 4), np.float32)
    d_in = F.DenoiseInput(*(a.ctypes.data for a in ins), near.ctypes.data)
    rc = load().orc_denoise(w, h, C.byref(d_in), C.byref(prm), out.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("orc_denoise refused the arguments (status %d)" % rc)
    return out

"""Python binding of the sample-variance oracle (oracle/_build/liboracle_variance.so, built from oracle_variance/variance.cpp) —
TEST INFRASTRUCTURE, like oracle/pyoracle.py.

``VarianceOracleScene`` is a ``QueryOracleScene`` backed by that library, with ``lum_film`` (the lum_w film of caller samples and
their AOV records). ``denoise_variance`` takes the arguments of ``tray_rust_b200.api.Scene.denoise_variance`` without a scene: the
image size is the films' shape.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_queries import pyqueries as Q
from tray_rust_b200 import _ffi as F


def load():
    lib = O.load_oracle("variance")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_variance_ready"):
        q = Q.load()
        for name in ("orc_intersect_records", "orc_occluded", "orc_illumination", "orc_bsdf_eval", "orc_bsdf_sample", "orc_light_sample",
                     "orc_light_pdf", "orc_emitted", "orc_scene_lights", "orc_film_write"):  # as pyqueries declares them
            getattr(lib, name).argtypes = getattr(q, name).argtypes
        vp = C.c_void_p
        lib.orc_lum_film.argtypes = [vp, C.c_size_t, vp, vp, vp, vp]
        lib.orc_denoise_variance.argtypes = [F.u32, F.u32, C.POINTER(F.DenoiseFrame), vp, C.POINTER(F.DenoiseParams), vp, vp]
        lib._variance_ready = True
    return lib


class VarianceOracleScene(Q.QueryOracleScene):
    """The ray-query oracle with the lum_w film of caller samples (variance.cpp)."""

    def __init__(self, desc, baseline=False):
        load()
        O.OracleScene.__init__(self, desc, libm="variance", baseline=baseline)

    def lum_film(self, samples, aov, regions, film=None):
        """orc_lum_film: samples (SAMPLE_DTYPE), their AOV records (AOV_SAMPLE_DTYPE) and regions (uint32, as film_write takes them)
        into the (height, width, 4) float32 lum_w film `film` (zeros when None), added into. Returns the film."""
        samples = np.ascontiguousarray(samples, dtype=F.SAMPLE_DTYPE)
        aov = np.ascontiguousarray(aov, dtype=F.AOV_SAMPLE_DTYPE)
        regions = np.ascontiguousarray(regions, dtype=np.uint32)
        assert len(samples) == len(aov) == len(regions)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        self._check(self._lib.orc_lum_film(self._h, len(samples), F.ptr(samples), F.ptr(aov), F.ptr(regions), F.ptr(film)))
        return film


def denoise_variance(colour, aovs, variance=False, **params):
    """orc_denoise_variance over host arrays: colour and aovs["albedo_w"] / ["normal_w"] / ["lum_w"] of shape (h, w, 4) float32,
    aovs["nearest"] of shape (h, w) uint64. Returns the (h, w, 4) float32 film, or (film, variance) with `variance`; raises
    ValueError where trb_denoise_variance refuses the parameters."""
    h, w = colour.shape[:2]
    ins = [np.ascontiguousarray(a, dtype=np.float32) for a in (colour, aovs["albedo_w"], aovs["normal_w"])]
    near = np.ascontiguousarray(aovs["nearest"], dtype=np.uint64)
    lum = np.ascontiguousarray(aovs["lum_w"], dtype=np.float32)
    for a in ins + [lum]:
        assert a.shape == (h, w, 4)
    assert near.shape == (h, w)
    p = dict(F.DENOISE_DEFAULTS, **params)
    prm = F.DenoiseParams(p["iterations"], p["normal_power"], p["sigma_luminance"], p["sigma_depth"])
    out = np.zeros((h, w, 4), np.float32)
    var = np.zeros((h, w), np.float32)
    d_in = F.DenoiseFrame(*(a.ctypes.data for a in ins), near.ctypes.data)
    rc = load().orc_denoise_variance(w, h, C.byref(d_in), lum.ctypes.data, C.byref(prm), out.ctypes.data, var.ctypes.data)
    if rc != F.TRB_OK:
        raise ValueError("orc_denoise_variance refused the arguments (status %d)" % rc)
    return (out, var) if variance else out

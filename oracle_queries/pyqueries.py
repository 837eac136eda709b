"""Python bindings of the ray-query oracle (oracle/_build/liboracle_queries.so, built from oracle_queries/queries.cpp) —
TEST INFRASTRUCTURE, like oracle/pyoracle.py.

``QueryOracleScene`` is an ``OracleScene`` backed by that library (the detmath oracle with the ray queries added), so it has
every oracle method plus ``intersect_records``, ``occluded`` and ``illumination`` with the signatures of ``tray_rust_b200.api.Scene``.
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from tray_rust_b200 import _ffi as F


def load():
    lib = O.load_oracle("queries")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_queries_ready"):
        vp, sz = C.c_void_p, C.c_size_t
        lib.orc_intersect_records.argtypes = [vp, sz, vp, vp, C.POINTER(F.Stats)]
        lib.orc_occluded.argtypes = [vp, sz, vp, vp, C.POINTER(F.Stats)]
        lib.orc_illumination.argtypes = [vp, sz, vp, C.c_uint32, C.c_uint32, vp, C.c_uint32, C.POINTER(F.Stats)]
        lib._queries_ready = True
    return lib


class QueryOracleScene(O.OracleScene):
    """The oracle with Scene::intersect returning the whole Intersection, OcclusionTester::occluded and Integrator::illumination
    along caller rays, per-ray times."""

    def __init__(self, desc, baseline=False):
        load()
        super().__init__(desc, libm="queries", baseline=baseline)

    def intersect_records(self, rays, stats=True):
        """Returns (INTERSECTION_DTYPE records, Stats); the oracle always counts its tests."""
        rays = np.ascontiguousarray(rays, dtype=F.QUERY_RAY_DTYPE)
        out = np.zeros(len(rays), F.INTERSECTION_DTYPE)
        st = F.Stats()
        self._check(self._lib.orc_intersect_records(self._h, len(rays), F.ptr(rays), F.ptr(out), C.byref(st)))
        return out, st

    def occluded(self, rays, reference=True, stats=True):
        """Returns (bool array, Stats). The oracle always walks to the closest hit (light/mod.rs:30-37)."""
        rays = np.ascontiguousarray(rays, dtype=F.QUERY_RAY_DTYPE)
        out = np.zeros(len(rays), np.uint8)
        st = F.Stats()
        self._check(self._lib.orc_occluded(self._h, len(rays), F.ptr(rays), F.ptr(out), C.byref(st)))
        return out.astype(bool), st

    def illumination(self, rays, spp=1, seed=1, clamp=False, stats=None, reference=True):
        """Returns the (n, 3) float32 means; a Stats passed as `stats` receives the counters. The oracle always counts its tests and
        walks shadow rays to the closest hit."""
        rays = np.ascontiguousarray(rays, dtype=F.ILLUM_RAY_DTYPE)
        out = np.zeros((len(rays), 3), np.float32)
        st = stats if stats is not None else F.Stats()
        self._check(self._lib.orc_illumination(self._h, len(rays), F.ptr(rays), spp, seed, F.ptr(out), 1 if clamp else 0, C.byref(st)))
        return out

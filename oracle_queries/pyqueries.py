"""Python bindings of the ray-query oracle (oracle/_build/liboracle_queries.so, built from oracle_queries/queries.cpp) —
TEST INFRASTRUCTURE, like oracle/pyoracle.py.

``QueryOracleScene`` is an ``OracleScene`` backed by that library (the detmath oracle with the ray queries added), so it has
every oracle method plus ``intersect_records``, ``occluded``, ``illumination`` and the shading queries ``bsdf_eval``, ``bsdf_sample``,
``light_sample``, ``light_pdf``, ``emitted`` and ``lights``, and ``film_write``, with the signatures of ``tray_rust_b200.api.Scene``.
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
        for name in ("orc_bsdf_eval", "orc_bsdf_sample"):
            getattr(lib, name).argtypes = [vp, sz, vp, vp, vp]
        for name in ("orc_light_sample", "orc_light_pdf", "orc_emitted"):
            getattr(lib, name).argtypes = [vp, sz, vp, vp]
        lib.orc_scene_lights.argtypes = [vp, vp]
        lib.orc_film_write.argtypes = [vp, sz, vp, vp, vp]
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

    def bsdf_eval(self, records, queries):
        rec = np.ascontiguousarray(records, dtype=F.INTERSECTION_DTYPE)
        q = np.ascontiguousarray(queries, dtype=F.BSDF_EVAL_QUERY_DTYPE)
        out = np.zeros((len(q), 4), np.float32)
        self._check(self._lib.orc_bsdf_eval(self._h, len(q), F.ptr(rec), F.ptr(q), F.ptr(out)))
        return out

    def bsdf_sample(self, records, queries):
        rec = np.ascontiguousarray(records, dtype=F.INTERSECTION_DTYPE)
        q = np.ascontiguousarray(queries, dtype=F.BSDF_SAMPLE_QUERY_DTYPE)
        out = np.zeros(len(q), F.BSDF_SAMPLE_DTYPE)
        self._check(self._lib.orc_bsdf_sample(self._h, len(q), F.ptr(rec), F.ptr(q), F.ptr(out)))
        return out

    def light_sample(self, queries):
        q = np.ascontiguousarray(queries, dtype=F.LIGHT_QUERY_DTYPE)
        out = np.zeros(len(q), F.LIGHT_SAMPLE_DTYPE)
        self._check(self._lib.orc_light_sample(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def light_pdf(self, queries):
        q = np.ascontiguousarray(queries, dtype=F.LIGHT_PDF_QUERY_DTYPE)
        out = np.zeros(len(q), np.float32)
        self._check(self._lib.orc_light_pdf(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def emitted(self, queries):
        q = np.ascontiguousarray(queries, dtype=F.EMIT_QUERY_DTYPE)
        out = np.zeros((len(q), 3), np.float32)
        self._check(self._lib.orc_emitted(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def lights(self):
        """the light list of sample_one_light (instance indices, object order)"""
        n = sum(1 for i in range(self._desc.n_instances) if self._desc.instances[i].kind != F.INST_RECEIVER)
        out = np.zeros(n, np.uint32)
        self._check(self._lib.orc_scene_lights(self._h, F.ptr(out)))
        return out

    def film_write(self, samples, regions, film=None):
        """RenderTarget::write per non-empty region in Morton-list order (see api.Scene.film_write); film is added into in place."""
        samples = np.ascontiguousarray(samples, dtype=F.SAMPLE_DTYPE)
        regions = np.ascontiguousarray(regions, dtype=np.uint32)
        assert len(samples) == len(regions)
        if film is None:
            film = np.zeros((self._desc.film.height, self._desc.film.width, 4), np.float32)
        assert film.dtype == np.float32 and film.flags.c_contiguous and film.size == self._desc.film.height * self._desc.film.width * 4
        self._check(self._lib.orc_film_write(self._h, len(samples), F.ptr(samples), F.ptr(regions), F.ptr(film)))
        return film

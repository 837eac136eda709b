"""Python bindings of the mesh-refit oracle (oracle/_build/liboracle_refit.so, built from oracle_refit/refit.cpp) — TEST
INFRASTRUCTURE, like oracle/pyoracle.py.

``RefitOracleScene`` is a ``QueryOracleScene`` backed by that library (the ray-query oracle with the refit added), so it has every
oracle and ray-query method plus ``refit_mesh`` with the signature of ``tray_rust_b200.api.Scene.refit_mesh``.
``AdaptiveRefitOracleScene`` is the same over the Adaptive-sampler oracle (liboracle_adaptive_refit.so, adaptive_refit.cpp).
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O
from oracle_adaptive import pyadaptive as A
from oracle_queries import pyqueries as Q
from tray_rust_b200 import _ffi as F

_QUERY_FUNCS = ("orc_intersect_records", "orc_occluded", "orc_illumination", "orc_bsdf_eval", "orc_bsdf_sample", "orc_light_sample",
                "orc_light_pdf", "orc_emitted", "orc_scene_lights", "orc_film_write")


def load():
    lib = O.load_oracle("refit")  # the detmath oracle's entry points, set up by pyoracle
    if not hasattr(lib, "_refit_ready"):
        q = Q.load()
        for name in _QUERY_FUNCS:  # the ray-query entry points, declared as pyqueries declares them
            getattr(lib, name).argtypes = getattr(q, name).argtypes
        vp = C.c_void_p
        lib.orc_scene_refit_mesh.argtypes = [vp, F.u32, vp, vp, vp]
        lib._refit_ready = True
    return lib


def load_adaptive():
    lib = O.load_oracle("adaptive_refit")
    if not hasattr(lib, "_refit_ready"):
        a = A.load()
        for name in ("orc_render_adaptive", "orc_render_samples_adaptive", "orc_adaptive_schedule"):  # as pyadaptive declares them
            getattr(lib, name).argtypes = getattr(a, name).argtypes
        lib.orc_scene_refit_mesh.argtypes = [C.c_void_p, F.u32, C.c_void_p, C.c_void_p, C.c_void_p]
        lib._refit_ready = True
    return lib


class _Refit:
    """refit_mesh over an oracle library that has orc_scene_refit_mesh (refit.h). Like the product, a refit re-runs the last
    update_frame, if one has been made."""
    _frame = None

    def update_frame(self, frame=0, start=0.0, end=0.0):
        super().update_frame(frame, start, end)
        self._frame = (frame, start, end)

    def refit_mesh(self, mesh, positions=None, normals=None, texcoords=None):
        arrays = []
        for a, k in ((positions, 3), (normals, 3), (texcoords, 2)):
            if a is not None:
                a = np.ascontiguousarray(a, np.float32)
                assert not 0 <= mesh < self._desc.n_meshes or a.size == self._desc.meshes[mesh].n_verts * k
            arrays.append(a)
        self._check(self._lib.orc_scene_refit_mesh(self._h, mesh, *(None if a is None else F.ptr(a) for a in arrays)))
        if positions is not None and self._frame is not None:
            super().update_frame(*self._frame)


class RefitOracleScene(_Refit, Q.QueryOracleScene):
    """The ray-query oracle with Mesh refits: the kept tree's boxes recomputed over the new positions (refit.cpp)."""

    def __init__(self, desc, baseline=False):
        load()
        O.OracleScene.__init__(self, desc, libm="refit", baseline=baseline)


class AdaptiveRefitOracleScene(_Refit, A.AdaptiveOracleScene):
    """The Adaptive-sampler oracle with Mesh refits (adaptive_refit.cpp)."""

    def __init__(self, desc, baseline=False):
        load_adaptive()
        O.OracleScene.__init__(self, desc, libm="adaptive_refit", baseline=baseline)

"""trb_scene_refit_mesh without a GPU: the exports, the ctypes declarations against the Rust ones in INTEGRATION.md, a plain-C caller's
statuses, Scene.refit_mesh's shape and index checks (which raise before anything reaches the library), and the oracle's refit against
an independent numpy restatement of the contract on C1's meshes, a heightfield and an icosphere, NaN, infinite and signed-zero vertices
included."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB
from oracle_refit import pyrefit as R
from test_mesh_update_cpu import _unopened_scene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_scene_refit_mesh", "trb_scene_refit_mesh_device"]
LEAF = np.uint32(F.BVH_LEAF)


def node_ranges(nodes):
    """each node's ordered_geom range [lo, hi): a leaf's own; an interior node's from its first leaf (first-child chain) to its last
    leaf (second-child chain), followed by pointer jumping"""
    leaf = (nodes["b"] & LEAF) != 0
    idx = np.arange(len(nodes), dtype=np.int64)
    a = nodes["a"].astype(np.int64)
    first, last = np.where(leaf, idx, idx + 1), np.where(leaf, idx, a)
    while True:
        f2, l2 = first[first], last[last]
        if np.array_equal(f2, first) and np.array_equal(l2, last):
            break
        first, last = f2, l2
    cnt = (nodes["b"] & ~LEAF).astype(np.int64)
    return a[first], a[last] + cnt[last]


def restated_tree(nodes, order, positions, indices):
    """the contract in numpy: the same nodes with each box the minimum / maximum (NaN dropped, starting from +-inf) of its
    triangles' boxes over its ordered_geom range"""
    p = np.asarray(positions, np.float32).reshape(-1, 3)
    tri = np.asarray(indices, np.uint32).reshape(-1, 3)[order]
    pa, pb, pc = p[tri[:, 0]], p[tri[:, 1]], p[tri[:, 2]]
    tlo = np.fmin(np.fmin(pa, pb), pc)  # Triangle::bounds: lo = hi = pa, grown with pb and pc
    thi = np.fmax(np.fmax(pa, pb), pc)
    del pa, pb, pc, tri
    lo, hi = node_ranges(nodes)
    cut = np.empty(2 * len(lo), np.int64)
    cut[0::2], cut[1::2] = lo, hi
    out = nodes.copy()
    pad = np.full((1, 3), np.nan, np.float32)  # hi may equal the slot count, which reduceat cannot index
    out["bmin"] = np.fmin(np.float32(np.inf), np.fmin.reduceat(np.concatenate([tlo, pad]), cut)[0::2])
    out["bmax"] = np.fmax(np.float32(-np.inf), np.fmax.reduceat(np.concatenate([thi, pad]), cut)[0::2])
    return out


def assert_tree_equal(got, want):
    """bit for bit but for the sign of a bound tied between -0 and +0 (== compares those equal, and no bound is NaN)"""
    assert len(got) == len(want)
    assert np.array_equal(got["a"], want["a"]) and np.array_equal(got["b"], want["b"])
    for k in ("bmin", "bmax"):
        assert not np.isnan(got[k]).any()
        assert np.array_equal(got[k], want[k]), k
        z = got[k] != 0
        assert np.array_equal(got[k][z].view(np.uint32), want[k][z].view(np.uint32)), k


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name in NEW:
        assert hasattr(trb, name) and name in F.TRB_SYMBOLS, name
        m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
        assert m, name
        rust = [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]
        ct = getattr(trb, name).argtypes
        assert len(ct) == len(rust), name
        for i, (r, c) in enumerate(zip(rust, ct)):
            if r.startswith("*"):
                assert c is C.c_void_p or issubclass(c, C._Pointer), (name, i, r, c)
            else:
                assert c is {"u32": C.c_uint32, "c_int": C.c_int}[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    exe = str(tmp_path / "mesh_refit_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "mesh_refit_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    status = {l.split()[1]: int(l.split()[2]) for l in out if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {k: F.TRB_INVALID_ARG for k in ("trb_scene_refit_mesh:null_scene", "trb_scene_refit_mesh:null_positions", "trb_scene_refit_mesh:null_all",
                                                     "trb_scene_refit_mesh_device:null_scene", "trb_scene_refit_mesh_device:null_all")}


def test_null_scene_needs_no_device(trb):
    v = np.zeros(9, np.float32)
    assert trb.trb_scene_refit_mesh(None, 0, F.ptr(v), None, None) == F.TRB_INVALID_ARG
    assert trb.trb_scene_refit_mesh_device(None, 0, None, None, None, None) == F.TRB_INVALID_ARG


@pytest.mark.parametrize("kw", [dict(positions=np.zeros((15, 3))), dict(positions=np.zeros((16, 2))), dict(positions=np.zeros((16, 3)), normals=np.zeros((16, 4))),
                                dict(positions=np.zeros((16, 3)), texcoords=np.zeros((16, 3))), dict(positions=np.zeros(47)), dict(positions=np.zeros((16, 3)), normals=np.zeros(47))])
def test_refit_mesh_rejects_wrong_shapes_before_the_library(kw):
    s = _unopened_scene()
    assert s._desc.meshes[0].n_verts == 16
    with pytest.raises(ValueError):
        s.refit_mesh(0, **kw)


def test_refit_mesh_rejects_a_mesh_index_out_of_range_before_the_library():
    s = _unopened_scene()
    for k in (1, -1):
        with pytest.raises(ValueError):
            s.refit_mesh(k, np.zeros((16, 3)))
        with pytest.raises(ValueError):
            s.refit_mesh_device(k, 1)
    s._h = None


def mesh_scene(mesh):
    b = SB.SceneBuilder(8, 8, 1)
    mats = SB.cornell_walls(b)
    SB.cornell_light(b, mats["white"])
    m = b.add_mesh(*mesh)
    b.receiver(F.SHAPE_MESH, mats["white"], [SB.trs()], mesh=m)
    b.add_camera([SB.trs(t=(0, 12, -60))])
    return b.finish()


def c1_desc(trb):
    d = C.POINTER(F.SceneDesc)()
    assert trb.trb_desc_load_json(os.path.join(REPO, "tests", "golden", "scenes", "c1_cornell_box.json").encode(), 24, 16, 4, C.byref(d)) == 0
    return d.contents  # left to the process (tiny)


def special(p, seed):
    """a copy of p with NaN, +-inf and +-0 coordinates on a few seeded vertices, and one vertex NaN in every coordinate"""
    q = p.copy()
    rng = np.random.default_rng(seed)
    for v in (np.nan, np.inf, -np.inf, 0.0, -0.0):
        k = rng.integers(0, len(q), size=max(1, len(q) // 50))
        q[k, rng.integers(0, 3, size=len(k))] = v
    q[rng.integers(0, len(q))] = np.nan
    return q


def meshes(trb):
    """(description, mesh index, indices, positions to refit to) on C1's meshes, a heightfield and an icosphere"""
    d = c1_desc(trb)
    for m in range(d.n_meshes):
        me = d.meshes[m]
        p = np.ctypeslib.as_array(me.positions, (me.n_verts * 3,)).reshape(-1, 3).copy()
        idx = np.ctypeslib.as_array(me.indices, (me.n_tris * 3,)).reshape(-1, 3).copy()
        yield d, m, idx, special(p * np.float32(1.5) + np.float32(0.25), m)
    hf = SB.heightfield_mesh(64, 7)
    wave = hf[0].copy()
    wave[:, 1] += np.sin(wave[:, 0]).astype(np.float32)
    yield mesh_scene(hf), 0, hf[3], wave
    yield mesh_scene(hf), 0, hf[3], special(wave, 3)
    ico = SB.icosphere_mesh(3)
    yield mesh_scene(ico), 0, ico[3], special(ico[0][::-1].copy(), 4)  # far from where it was built: boxes grow and overlap


def test_oracle_refit_against_a_numpy_restatement(trb):
    for desc, m, idx, pos in meshes(trb):
        o = R.RefitOracleScene(desc)
        nodes, order = o.bvh(m)
        o.refit_mesh(m, pos)
        got, got_order = o.bvh(m)
        assert np.array_equal(got_order, order)
        assert_tree_equal(got, restated_tree(nodes, order, pos, idx))
        if np.isfinite(pos).all():
            assert not np.array_equal(got["bmin"], nodes["bmin"])


def test_refit_to_the_built_positions_gives_back_the_built_tree(trb):
    for desc, m, idx, _ in meshes(trb):
        me = desc.meshes[m]
        p = np.ctypeslib.as_array(me.positions, (me.n_verts * 3,)).copy()
        o = R.RefitOracleScene(desc)
        nodes, order = o.bvh(m)
        o.refit_mesh(m, p)
        got, got_order = o.bvh(m)
        assert got.tobytes() == nodes.tobytes() and got_order.tobytes() == order.tobytes()


def test_oracle_refit_arguments(trb):
    hf = SB.heightfield_mesh(8, 1)
    o = R.RefitOracleScene(mesh_scene(hf))
    with pytest.raises(Exception):
        o.refit_mesh(1, hf[0])
    nodes, _ = o.bvh(0)
    o.refit_mesh(0, None, normals=hf[1][::-1].copy())  # attributes alone keep the tree
    assert o.bvh(0)[0].tobytes() == nodes.tobytes()

"""The device SAH builder on an H100 (DESIGN.md §4 "Mesh BVH build"): trb_build_bvh and trb_build_bvh_device must return the bytes of
trb_host_build_bvh (nodes in preorder and ordered_geom) on awkward box sets, and every scene's mesh trees, built on the device at
scene creation, must equal the oracle's and the host build's (TRB_BUILD_DEVICE=0), with bit-identical renders."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden  # noqa: E402

f32 = np.float32
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]


def host_build(boxes, max_geom):
    trb = F.load_trb()
    boxes = np.ascontiguousarray(boxes, f32)
    nn = F.u32()
    assert trb.trb_host_build_bvh(F.ptr(boxes), len(boxes), max_geom, C.byref(nn), None, None) == F.TRB_OK
    nodes, order = np.zeros(nn.value, F.NODE_DTYPE), np.zeros(len(boxes), np.uint32)
    assert trb.trb_host_build_bvh(F.ptr(boxes), len(boxes), max_geom, C.byref(nn), F.ptr(nodes), F.ptr(order)) == F.TRB_OK
    return nodes, order


def stream_build(boxes, max_geom):
    import torch
    n = len(boxes)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_boxes = torch.from_numpy(np.ascontiguousarray(boxes, f32)).cuda(non_blocking=False)
        d_nodes = torch.full((2 * n - 1, 8), -1, dtype=torch.int32, device="cuda")
        d_order = torch.zeros(n, dtype=torch.int32, device="cuda")
        d_nn = torch.zeros(1, dtype=torch.int32, device="cuda")
    api.build_bvh_device(d_boxes.data_ptr(), n, max_geom, d_nn.data_ptr(), d_nodes.data_ptr(), d_order.data_ptr(), stream=s.cuda_stream)
    s.synchronize()
    nn = int(d_nn.cpu()[0])
    return d_nodes[:nn].cpu().numpy().view(F.NODE_DTYPE).reshape(-1), d_order.cpu().numpy().view(np.uint32)


def same_tree(a, b, zero_signs=True):
    """byte equality; zero_signs=False lets a bound be +0 in one tree and -0 in the other (DESIGN.md §4: the host builder's
    zero ties depend on how its compiler lowered each fminf / fmaxf)"""
    if zero_signs:
        return a.tobytes() == b.tobytes()
    return (len(a) == len(b) and np.array_equal(a["a"], b["a"]) and np.array_equal(a["b"], b["b"])
            and all(np.array_equal(a[k], b[k], equal_nan=True) for k in ("bmin", "bmax")))


def check(boxes, max_geom, stream=True, zero_signs=True):
    hn, ho = host_build(boxes, max_geom)
    dn, do = api.build_bvh(boxes, max_geom)
    assert same_tree(dn, hn, zero_signs) and do.tobytes() == ho.tobytes(), (len(boxes), max_geom)
    if stream:
        sn, so = stream_build(boxes, max_geom)
        assert sn.tobytes() == dn.tobytes() and so.tobytes() == do.tobytes(), (len(boxes), max_geom)
    return hn


def soup(rng, n, lo=-10.0, hi=10.0, size=0.5):
    c = rng.uniform(lo, hi, (n, 3)).astype(f32)
    e = rng.uniform(0, size, (n, 3)).astype(f32)
    return np.concatenate([c - e, c + e], axis=1).astype(f32)


def box_sets():
    rng = np.random.default_rng(11)
    sets = {"n%d" % n: soup(rng, n) for n in (1, 2, 3, 4, 5, 16, 17, 20000)}
    b = soup(rng, 300)
    b[::3] = b[0]                                                     # coincident centroids among others
    sets["coincident_300"] = b
    for n in (40, 3000):                                              # all centroids coincident, n above and below max_geom
        sets["all_coincident_%d" % n] = np.repeat(soup(rng, 1), n, axis=0) + np.tile(np.array([[-1, -1, -1, 1, 1, 1]], f32), (n, 1)) * rng.uniform(0, 1, (n, 1)).astype(f32)
    k = np.arange(5000, dtype=f32)                                    # centroids on the 12 bucket boundaries
    c = (k % 13) * (12.0 / 12.0)
    sets["bucket_edges"] = np.stack([c, k % 7, k % 5, c, k % 7, k % 5], axis=1).astype(f32)
    e = (2.0 ** (np.arange(6000) % 250 - 125)).astype(f32)            # exponentially spaced centroids: a deep tree
    sets["exponential"] = np.stack([e, 0 * e, 0 * e, e, 0 * e, 0 * e], axis=1).astype(f32)
    fl = soup(rng, 5000)
    fl[:, 4] = fl[:, 1]                                               # flat boxes
    sets["flat"] = fl
    pl = soup(rng, 5000)
    pl[:, 2] = pl[:, 5] = 3.0                                         # one plane: area(bounds) = 0
    sets["plane"] = pl
    z = rng.choice(np.array([-0.0, 0.0, 1e-45, -1e-45, 1e-40, -1e-40], f32), (20000, 6))
    sets["signed_zeros"] = z                                          # zero ties in every fold (lo > hi included)
    z2 = soup(rng, 20000)
    m = rng.random(z2.shape) < 0.5
    z2[m] = rng.choice(np.array([-0.0, 0.0], f32), int(m.sum()))
    sets["signed_zeros_mixed"] = z2
    d = soup(rng, 4000)
    sets["duplicates"] = np.concatenate([d, d, d[::-1]])
    return sets


SETS = box_sets()


@pytest.mark.parametrize("name", sorted(SETS))
@pytest.mark.parametrize("max_geom", [1, 4, 16, 10 ** 6])
def test_device_build_equals_the_host_build(name, max_geom):
    check(SETS[name], max_geom, zero_signs=not name.startswith("signed_zeros"))


def test_nan_and_infinite_coordinates_with_max_geom_above_the_count():
    """NaN and ±inf centroids can put every box of a node in one bucket: the reference builds such a node only as a leaf
    (max_geom >= n); a forced split would leave an empty child, on which the reference's build never finishes."""
    rng = np.random.default_rng(3)
    nf = soup(rng, 20000)
    m = rng.random(nf.shape)
    nf[m < 0.01] = np.inf
    nf[(m >= 0.01) & (m < 0.02)] = -np.inf
    nf[(m >= 0.02) & (m < 0.03)] = np.nan
    nf[:50] = np.nan                                                  # boxes of nothing but NaN
    check(nf, 10 ** 6)


@pytest.mark.parametrize("n", [(1 << 20) + 1, 1 << 22])
def test_large_random_soups(n):
    b = soup(np.random.default_rng(n), n, -100, 100, 0.2)
    nodes = check(b, 16, stream=n < (1 << 22))
    assert len(nodes) > 1000


def mesh_scenes():
    gold = make_golden.golden_scenes()
    out = {name: (mk, make_golden.frame_of(name), kw) for name, (mk, kw) in gold.items()}
    out["c3"] = (lambda: SB.scene_c3(96, 72, 8, subdiv=4), (0, 0.0, 0.0), dict(spp=2, seed=3))

    def signed_zero_mesh():
        desc = gold["c1_cornell"][0]()
        rng = np.random.default_rng(4)
        for i in range(desc.n_meshes):
            m = desc.meshes[i]
            p = np.ctypeslib.as_array(m.positions, shape=(m.n_verts * 3,))
            p[rng.random(len(p)) < 0.3] = 0.0
            z = p == 0
            p[z] = rng.choice(np.array([-0.0, 0.0], f32), int(z.sum()))
        return desc
    out["signed_zero_mesh"] = (signed_zero_mesh, make_golden.frame_of("c1_cornell"), gold["c1_cornell"][1])
    return out


SCENES = mesh_scenes()


def _desc(mk):
    d = mk()
    return d.finish() if hasattr(d, "finish") else d


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scene_mesh_trees_equal_the_oracle_on_both_builds(name, monkeypatch):
    mk, frame, kw = SCENES[name]
    desc = _desc(mk)
    o = O.OracleScene(desc)
    g = api.Scene(desc)
    monkeypatch.setenv("TRB_BUILD_DEVICE", "0")
    h = api.Scene(desc)
    monkeypatch.delenv("TRB_BUILD_DEVICE")
    for i in range(desc.n_meshes):
        (gn, go), (hn, ho), (on, oo) = g.bvh(i), h.bvh(i), o.bvh(i)
        exact = name != "signed_zero_mesh"  # the library's host build and the oracle differ between themselves in tied zero signs
        assert same_tree(gn, on, exact) and go.tobytes() == oo.tobytes(), (name, i)
        assert same_tree(hn, on, exact) and ho.tobytes() == oo.tobytes(), (name, i)
    g.update_frame(*frame); h.update_frame(*frame)
    kw = {k: v for k, v in kw.items() if k in ("spp", "seed", "sample_first", "sample_count", "current_frame")}
    (gs, gst), (hs, hst) = g.render_samples(flags=F.RENDER_STATS, **kw), h.render_samples(flags=F.RENDER_STATS, **kw)
    assert gs.tobytes() == hs.tobytes()
    assert [getattr(gst, k) for k in COUNTERS] == [getattr(hst, k) for k in COUNTERS]

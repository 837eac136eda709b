"""The level-built instance tree without a GPU: the open-node capacity under a small serial-subtree threshold, and
scenebuild.scene_instances' default form."""
import ctypes as C
import hashlib

import numpy as np

from tray_rust_b200 import scenebuild as SB


def test_open_nodes_of_a_level_fit_the_capacity_for_small_thresholds():
    """open_cap(n, small) = n / (small + 1) + 1 against a literal count: whatever the splits, the nodes of more than `small` elements on
    one level are disjoint"""
    rng = np.random.default_rng(5)
    for small in (4, 32, 64, 1024):
        for n in (1, small, small + 1, 2 * small + 1, 1000, 54_321):
            cap = n // (small + 1) + 1
            level = [n] if n > small else []
            while level:
                assert len(level) <= cap, (small, n)
                nxt = []
                for m in level:
                    left = int(rng.integers(1, m)) if rng.random() < 0.8 else (1 if rng.random() < 0.5 else m - 1)
                    nxt += [c for c in (left, m - left) if c > small]
                level = nxt


def description_hash(b):
    d = b.finish()
    m = hashlib.sha256()
    for name in ("keyframes", "splines", "knots", "color_keys", "instances", "cameras", "materials"):
        a = getattr(d, name)
        m.update(C.string_at(a, getattr(d, "n_" + name) * C.sizeof(a._type_)))
    m.update(bytes(d.film))
    m.update(bytes(d.integrator))
    return m.hexdigest(), d


def test_scene_instances_default_form_is_unchanged_and_the_mesh_form_shares_one_mesh():
    h, d = description_hash(SB.scene_instances(37, 11))
    assert h == "e76fc2ed627fa73d03a50dd8b0177e645d3eb321386f4823a6d9c2c95caf9c46" and d.n_meshes == 0  # as before the mesh form existed
    b = SB.scene_instances(37, 11, mesh=True)
    d = b.finish()
    assert d.n_meshes == 1 and d.meshes[0].n_tris == 80 and d.n_instances == 43
    assert all(it[1] == SB.F.SHAPE_MESH and it[4] == 0 for it in b.instances[6:])
    assert [k[0] for k in b.keyframes] == [k[0] for k in SB.scene_instances(37, 11).keyframes]  # the same positions

"""Host side of the wide mesh leaf form (no GPU): the heightfield generator behind the large-mesh scene, and the mesh size limits
that trb_scene_create checks before it touches a device."""
import ctypes as C

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB


@pytest.mark.parametrize("grid", [2, 3, 17])
def test_heightfield_grid(grid):
    p, n, t, idx = SB.heightfield_mesh(grid, seed=7)
    assert p.dtype == n.dtype == t.dtype == np.float32 and idx.dtype == np.uint32
    assert p.shape == n.shape == (grid * grid, 3) and t.shape == (grid * grid, 2)
    assert idx.shape == (2 * (grid - 1) ** 2, 3)
    assert idx.min() == 0 and idx.max() == grid * grid - 1
    assert len(np.unique(idx)) == grid * grid                                  # every vertex is used; shared, not a soup
    assert np.all(np.abs(np.linalg.norm(n.astype(np.float64), axis=1) - 1.0) < 1e-6)
    assert n[:, 1].min() > 0.0                                                  # a heightfield's normals face up
    assert t.min() == 0.0 and t.max() == 1.0
    assert np.array_equal(np.unique(t[:, 0]), np.linspace(0, 1, grid, dtype=np.float32))
    assert p[:, 0].min() == -13 and p[:, 0].max() == 13 and p[:, 2].min() == -8 and p[:, 2].max() == 18
    # no degenerate triangles, and each cell's two triangles share its diagonal
    e = np.cross(p[idx[:, 1]] - p[idx[:, 0]], p[idx[:, 2]] - p[idx[:, 0]])
    assert (np.linalg.norm(e, axis=1) > 0).all()
    assert np.array_equal(idx[0::2, 2], idx[1::2, 1]) and np.array_equal(idx[0::2, 0], idx[1::2, 0])


def test_heightfield_is_seeded():
    a, b, c = SB.heightfield_mesh(9, 1), SB.heightfield_mesh(9, 1), SB.heightfield_mesh(9, 2)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert not np.array_equal(a[0], c[0]) and np.array_equal(a[3], c[3])


def test_heightfield_scene_triangle_count():
    desc = SB.scene_heightfield(33, 64, 64, 1).finish()
    assert desc.n_meshes == 1 and desc.meshes[0].n_tris == 2 * 32 ** 2 and desc.meshes[0].n_verts == 33 ** 2


@pytest.mark.parametrize("field,value,msg", [("n_tris", (1 << 30) + 1, b"2^30 triangles"),
                                             ("n_verts", 0xffffffff // 3 + 1, b"too many vertices")])
def test_mesh_size_limits_are_refused_before_any_device_work(field, value, msg):
    """A mesh above the wide form's 2^30 triangles, or with vertex indices whose 3 * index does not fit 32 bits, is TRB_UNSUPPORTED.
    The check runs before the mesh arrays are read (the sizes here are far larger than the arrays) and before a device is needed."""
    lib = F.load_trb()
    desc = SB.scene_heightfield(3, 64, 64, 1).finish()
    setattr(desc.meshes[0], field, value)
    h = C.c_void_p()
    assert lib.trb_scene_create(C.byref(desc), 0, C.byref(h)) == F.TRB_UNSUPPORTED
    assert msg in lib.trb_last_error()

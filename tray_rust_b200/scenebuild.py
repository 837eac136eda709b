"""Programmatic construction of trb_scene_desc (include/trb.h) for tests and the bench.

The reference builds scenes from JSON (src/scene.rs); JSON scenes go through the C++
loader behind ``trb_desc_load_json``. This module builds the same flattened description
directly for synthetic scenes (SURVEY.md §8d: C3 stand-in, C4 1M-triangle scene, furnace
boxes) where transforms are given as TRS keyframes — exactly what the ABI carries.
"""
import ctypes as C
import math

import numpy as np

from . import _ffi as F


def quat_axis_angle(axis, deg):
    """Quaternion (x, y, z, w) of a rotation of `deg` degrees about `axis`."""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    h = math.radians(deg) / 2.0
    return (a[0] * math.sin(h), a[1] * math.sin(h), a[2] * math.sin(h), math.cos(h))


def trs(t=(0, 0, 0), q=(0, 0, 0, 1), s=(1, 1, 1)):
    if np.isscalar(s):
        s = (s, s, s)
    return (tuple(float(x) for x in t), tuple(float(x) for x in q), tuple(float(x) for x in s))


class Anim:
    """One animated level of a transform stack: B-spline over TRS control points
    (AnimatedTransform::with_keyframes, animated_transform.rs:22-33)."""

    def __init__(self, keys, knots=None, degree=3):
        keys = [list(k) for k in keys]
        for i in range(1, len(keys)):  # with_keyframes keeps successive quaternions in one hemisphere
            a, b = np.asarray(keys[i - 1][1], np.float32), np.asarray(keys[i][1], np.float32)
            if float(np.dot(a, b)) < 0.0:
                keys[i][1] = tuple(-float(x) for x in keys[i][1])
        self.keys = [tuple(k) for k in keys]
        self.degree = degree
        self.knots = list(knots) if knots is not None else clamped_knots(len(keys), degree)


def clamped_knots(n_ctrl, degree, t0=0.0, t1=1.0):
    """Clamped uniform knot vector over [t0, t1] (n_ctrl + degree + 1 knots)."""
    inner = n_ctrl - degree - 1
    assert inner >= 0, "need at least degree + 1 control points"
    mid = [t0 + (t1 - t0) * (i + 1) / (inner + 1) for i in range(inner)]
    return [t0] * (degree + 1) + mid + [t1] * (degree + 1)


class SceneBuilder:
    def __init__(self, width=64, height=64, spp=4, min_depth=4, max_depth=8):
        self.film = dict(width=width, height=height, samples=spp, frames=1, start_frame=0, end_frame=0, scene_time=0.0,
                         filter_type=F.FILTER_MITCHELL_NETRAVALI, filter_w=2.0, filter_h=2.0, filter_b=1.0 / 3.0,
                         filter_c=1.0 / 3.0)
        self.integrator = (0, min_depth, max_depth)
        self.keyframes, self.knots, self.splines = [], [], []
        self.instances, self.color_keys, self.meshes, self.materials, self.merl, self.cameras = [], [], [], [], [], []
        self.fov_floats = []
        self.textures, self.images = [], []
        self._keep = []
        self._given = []  # the mesh list a scene was last given (finish(), meshes_section())

    # -- transforms ---------------------------------------------------------------------
    def _add_xf(self, levels):
        """levels: list of TRS triples, applied first-to-last (animated_transform.rs:42-54)."""
        first = len(self.splines)
        for lv in levels:
            if isinstance(lv, Anim):
                assert len(lv.knots) == len(lv.keys) + lv.degree + 1
                self.splines.append((lv.degree, len(lv.keys), len(self.keyframes), len(lv.knots), len(self.knots)))
                self.keyframes += lv.keys
                self.knots += [float(k) for k in lv.knots]
                continue
            (t, q, s) = lv
            self.splines.append((0, 1, len(self.keyframes), 2, len(self.knots)))
            self.keyframes.append((t, q, s))
            self.knots += [0.0, 1.0]  # AnimatedTransform::unanimated (animated_transform.rs:34-37)
        return first, len(levels)

    def add_texture(self, frames):
        """texture::Image (one frame) or texture::AnimatedImage (>= 2 frames): frames = [(H x W x 4 uint8 array, time), ...] or a single
        array. Returns the value to pass as tex_c0 / tex_c1 / tex_roughness / tex_eta of add_material (index + 1)."""
        if isinstance(frames, np.ndarray):
            frames = [(frames, 0.0)]
        first = len(self.images)
        for px, t in frames:
            px = np.ascontiguousarray(px, np.uint8)
            assert px.ndim == 3 and px.shape[2] == 4
            self.images.append((px, float(t)))
        self.textures.append((first, len(frames)))
        return len(self.textures)

    def add_material(self, mtype, c0=(0, 0, 0), c1=(0, 0, 0), roughness=0.0, eta=1.0, merl=0, tex_c0=0, tex_c1=0, tex_roughness=0, tex_eta=0):
        self.materials.append((mtype, tuple(c0), tuple(c1), float(roughness), float(eta), merl, (tex_c0, tex_c1, tex_roughness, tex_eta)))
        return len(self.materials) - 1

    def add_merl_table(self, table):
        t = np.ascontiguousarray(table, dtype=np.float32).reshape(-1)
        assert t.size == F.MERL_TABLE_FLOATS
        self.merl.append(t)
        return len(self.merl) - 1

    @staticmethod
    def _mesh(positions, normals, texcoords, indices):
        p = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
        n = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
        t = np.ascontiguousarray(texcoords, dtype=np.float32).reshape(-1, 2)
        i = np.ascontiguousarray(indices, dtype=np.uint32).reshape(-1, 3)
        assert len(p) == len(n) == len(t)
        return p, n, t, i

    def add_mesh(self, positions, normals, texcoords, indices):
        self.meshes.append(self._mesh(positions, normals, texcoords, indices))
        return len(self.meshes) - 1

    def set_mesh(self, i, positions, normals, texcoords, indices):
        """Replace mesh i's arrays (any vertex and triangle counts); the next meshes() section builds it anew."""
        self.meshes[i] = self._mesh(positions, normals, texcoords, indices)

    def remove_mesh(self, i):
        """Drop mesh i and renumber the mesh instances above it: the builder is then the one that never added it. Refused (ValueError)
        while an instance still uses mesh i. Returns the removed arrays."""
        users = [k for k, it in enumerate(self.instances) if it[1] == F.SHAPE_MESH and it[4] == i]
        if users:
            raise ValueError("mesh %d is used by instances %s" % (i, users))
        self.instances = [it[:4] + (it[4] - 1,) + it[5:] if it[1] == F.SHAPE_MESH and it[4] > i else it for it in self.instances]
        return self.meshes.pop(i)

    def add_instance(self, kind, shape, material, xf, p0=0.0, p1=0.0, mesh=0, emission=None):
        sf, ns = self._add_xf(xf)
        ef, ne = 0, 0
        if emission is not None:
            # a plain colour, or [(colour, time), ...] for AnimatedColor keyframes (scene.rs:729-747), times ascending
            keyed = isinstance(emission, list) and len(emission) > 0 and isinstance(emission[0], (tuple, list)) and len(emission[0]) == 2 \
                and isinstance(emission[0][0], (tuple, list))
            keys = emission if keyed else [(emission, 0.0)]
            ef, ne = len(self.color_keys), len(keys)
            for col, tm in keys:
                e = list(col)
                if len(e) == 4:  # load_color: rgb scaled by the 4th component (scene.rs:713-716)
                    e = [np.float32(e[0]) * np.float32(e[3]), np.float32(e[1]) * np.float32(e[3]), np.float32(e[2]) * np.float32(e[3]),
                         np.float32(e[3])]
                else:
                    e = e + [1.0]
                self.color_keys.append((tuple(float(x) for x in e), float(tm)))
        self.instances.append((kind, shape, float(p0), float(p1), mesh, material, sf, ns, ef, ne))
        return len(self.instances) - 1

    def receiver(self, shape, material, xf, **kw):
        return self.add_instance(F.INST_RECEIVER, shape, material, xf, **kw)

    def area_light(self, shape, material, xf, emission, **kw):
        return self.add_instance(F.INST_EMITTER_AREA, shape, material, xf, emission=emission, **kw)

    def point_light(self, xf, emission):
        return self.add_instance(F.INST_EMITTER_POINT, F.SHAPE_NONE, 0, xf, emission=emission)

    def add_camera(self, xf, fov=30.0, shutter_size=0.5, active_at=0, fov_knots=None, fov_degree=3):
        """fov: degrees, or a list of B-spline control values with fov_knots / fov_degree (Camera::animated_fov, camera.rs:95-125)."""
        sf, ns = self._add_xf(xf)
        if isinstance(fov, (list, tuple)):
            knots = list(fov_knots) if fov_knots is not None else clamped_knots(len(fov), fov_degree)
            assert len(knots) == len(fov) + fov_degree + 1
            cf = len(self.fov_floats); self.fov_floats += [float(x) for x in fov]
            kf = len(self.fov_floats); self.fov_floats += [float(x) for x in knots]
            self.cameras.append((sf, ns, float(fov[0]), float(shutter_size), active_at, fov_degree, len(fov), cf, len(knots), kf))
        else:
            self.cameras.append((sf, ns, float(fov), float(shutter_size), active_at, 0, 0, 0, 0, 0))

    def remove_instance(self, i):
        """Drop instance i with the splines, keyframes, knots and colour keys it owns, and renumber what the remaining instances, splines
        and cameras reference: the builder is then the one that never added it. Returns the removed instance's tuple."""
        inst = self.instances.pop(i)
        sf, ns, ef, ne = inst[6:10]
        gone = self.splines[sf:sf + ns]

        def cut(items, ranges):
            """delete [first, first + n) for each range; returns the new index of an old one"""
            ranges = sorted(r for r in ranges if r[1])
            for first, n in reversed(ranges):
                del items[first:first + n]
            return lambda idx: idx - sum(n for first, n in ranges if first < idx)
        kf = cut(self.keyframes, [(sp[2], sp[1]) for sp in gone])
        kn = cut(self.knots, [(sp[4], sp[3]) for sp in gone])
        sp_ = cut(self.splines, [(sf, ns)])
        ck = cut(self.color_keys, [(ef, ne)])
        self.splines = [(d, nc, kf(cf), nk, kn(kf0)) for d, nc, cf, nk, kf0 in self.splines]
        self.instances = [it[:6] + (sp_(it[6]), it[7], ck(it[8]), it[9]) for it in self.instances]
        self.cameras = [(sp_(c[0]),) + c[1:] for c in self.cameras]
        return inst

    # -- finish ---------------------------------------------------------------------------
    def _fill_objects(self, d, keep):
        """the object section's seven arrays and counts into d (a SceneDesc or a SceneObjects: same field names)"""
        def arr(ctype, items, conv):
            a = (ctype * max(1, len(items)))()
            for i, it in enumerate(items):
                conv(a[i], it)
            keep.append(a)
            return a

        def kf(o, it):
            o.translation[:] = it[0]; o.rotation[:] = it[1]; o.scaling[:] = it[2]
        d.keyframes = arr(F.Keyframe, self.keyframes, kf); d.n_keyframes = len(self.keyframes)

        def sp(o, it):
            o.degree, o.n_ctrl, o.ctrl_first, o.n_knots, o.knot_first = it
        d.splines = arr(F.Spline, self.splines, sp); d.n_splines = len(self.splines)
        knots = (F.f32 * max(1, len(self.knots)))(*self.knots); keep.append(knots)
        d.knots = knots; d.n_knots = len(self.knots)

        def ck(o, it):
            o.rgba[:] = it[0]; o.time = it[1]
        d.color_keys = arr(F.ColorKey, self.color_keys, ck); d.n_color_keys = len(self.color_keys)

        def inst(o, it):
            (o.kind, o.shape, o.p0, o.p1, o.mesh, o.material, o.spline_first, o.n_splines, o.emission_first, o.n_emission) = it
        d.instances = arr(F.Instance, self.instances, inst); d.n_instances = len(self.instances)

        def cam(o, it):
            (o.spline_first, o.n_splines, o.fov, o.shutter_size, o.active_at, o.fov_degree, o.n_fov_ctrl, o.fov_ctrl_first, o.n_fov_knots,
             o.fov_knot_first) = it
        d.cameras = arr(F.Camera, self.cameras, cam); d.n_cameras = len(self.cameras)
        ff = (F.f32 * max(1, len(self.fov_floats)))(*self.fov_floats); keep.append(ff)
        d.fov_floats = ff; d.n_fov_floats = len(self.fov_floats)

    def objects(self):
        """The builder's object section (trb_scene_objects) for Scene.replace_objects: after b.receiver(...) on the builder a scene was
        created from, scene.replace_objects(b.objects()) adds that receiver to the scene."""
        o = F.SceneObjects()
        o._keep = []
        self._fill_objects(o, o._keep)
        return o

    def _fill_meshes(self, d, keep):
        """the mesh list's count and trb_mesh array into d (a SceneDesc or a SceneMeshes: same field names); the builder remembers the
        list as the one a scene was last given, which meshes() compares against"""
        a = (F.Mesh * max(1, len(self.meshes)))()
        for o, (p, n, t, i) in zip(a, self.meshes):
            o.n_verts, o.n_tris = len(p), len(i)
            o.positions = p.ctypes.data_as(C.POINTER(F.f32)); o.normals = n.ctypes.data_as(C.POINTER(F.f32))
            o.texcoords = t.ctypes.data_as(C.POINTER(F.f32)); o.indices = i.ctypes.data_as(C.POINTER(F.u32))
        keep += [a, list(self.meshes)]
        d.meshes = a; d.n_meshes = len(self.meshes)
        self._given = list(self.meshes)

    def meshes_section(self):
        """The builder's mesh list (trb_scene_meshes) for Scene.replace_meshes: mesh i keeps the scene's mesh j when it is the same
        arrays the scene was last given as mesh j (by finish() or an earlier section; set_mesh makes new ones), otherwise it is new."""
        given = {id(m): j for j, m in enumerate(self._given)}
        keep = []
        for m in self.meshes:
            j = given.pop(id(m), None)
            keep.append(F.MESH_NEW if j is None else j)
        s = F.SceneMeshes()
        s._keep = []
        self._fill_meshes(s, s._keep)
        k = (F.u32 * max(1, len(keep)))(*keep)
        s._keep.append(k)
        s.keep = k
        return s

    def _fill_materials(self, d, keep):
        """the material section's four arrays and counts into d (a SceneDesc or a SceneMaterials: same field names). The MERL tables and
        images are passed as the builder holds them: numpy arrays, or torch CUDA tensors for Scene.replace_materials_device"""
        def arr(ctype, items, conv):
            a = (ctype * max(1, len(items)))()
            for i, it in enumerate(items):
                conv(a[i], it)
            keep.append(a)
            return a

        def addr(t):
            return t.data_ptr() if hasattr(t, "data_ptr") else t.ctypes.data

        def mat(o, it):
            o.type = it[0]; o.c0[:] = it[1]; o.c1[:] = it[2]; o.roughness = it[3]; o.eta = it[4]; o.merl = it[5]
            o.tex[:] = it[6] if len(it) > 6 else (0, 0, 0, 0)
        d.materials = arr(F.Material, self.materials, mat); d.n_materials = len(self.materials)
        mt = (C.POINTER(F.f32) * max(1, len(self.merl)))()
        for i, t in enumerate(self.merl):
            mt[i] = C.cast(addr(t), C.POINTER(F.f32))
        keep.append(mt); keep.append(list(self.merl))
        d.merl_tables = mt; d.n_merl = len(self.merl)

        def tex(o, it):
            o.first_image, o.n_images = it
        d.textures = arr(F.Texture, self.textures, tex); d.n_textures = len(self.textures)

        def image(o, it):
            px, t = it
            o.height, o.width = px.shape[0], px.shape[1]
            o.rgba8 = C.cast(addr(px), C.POINTER(C.c_uint8)); o.time = t
        d.images = arr(F.Image, self.images, image); d.n_images = len(self.images)
        keep.append(list(self.images))

    def materials_section(self):
        """The builder's material section (trb_scene_materials) for Scene.replace_materials: its materials, MERL tables, textures and
        images, as finish() would give them."""
        s = F.SceneMaterials()
        s._keep = []
        self._fill_materials(s, s._keep)
        return s

    def remove_material(self, i):
        """Drop material i and renumber the instances that use the materials above it: the builder is then the one that never added it.
        Refused (ValueError) while an instance other than a point light (which has no material) uses material i. Returns the removed
        material."""
        users = [k for k, it in enumerate(self.instances) if it[0] != F.INST_EMITTER_POINT and it[5] == i]
        if users:
            raise ValueError("material %d is used by instances %s" % (i, users))
        self.instances = [it[:5] + (it[5] - 1,) + it[6:] if it[0] != F.INST_EMITTER_POINT and it[5] > i else it for it in self.instances]
        return self.materials.pop(i)

    def remove_texture(self, i):
        """Drop texture i (the value add_texture returned is i + 1) with its images, and renumber the materials' texture bindings and the
        other textures' image ranges: the builder is then the one that never added it. Refused (ValueError) while a material is bound to
        it. Returns the removed texture's frames [(pixels, time), ...]."""
        users = [k for k, m in enumerate(self.materials) if i + 1 in tuple(m[6])]
        if users:
            raise ValueError("texture %d is used by materials %s" % (i, users))
        first, n = self.textures.pop(i)
        frames = self.images[first:first + n]
        del self.images[first:first + n]
        self.textures = [(f - n if f > first else f, k) for f, k in self.textures]
        self.materials = [m[:6] + (tuple(t - 1 if t > i + 1 else t for t in m[6]),) for m in self.materials]
        return frames

    def remove_merl_table(self, i):
        """Drop MERL table i and renumber the MERL materials that use the tables above it: the builder is then the one that never added
        it. Refused (ValueError) while a MERL material uses table i. Returns the removed table."""
        users = [k for k, m in enumerate(self.materials) if m[0] == F.MAT_MERL and m[5] == i]
        if users:
            raise ValueError("MERL table %d is used by materials %s" % (i, users))
        self.materials = [m[:5] + (m[5] - 1,) + m[6:] if m[0] == F.MAT_MERL and m[5] > i else m for m in self.materials]
        return self.merl.pop(i)

    def finish(self):
        d = F.SceneDesc()
        d.abi_version = F.TRB_ABI_VERSION
        d.film = F.Film(**self.film)
        d.integrator = F.Integrator(*self.integrator)
        keep = self._keep
        self._fill_objects(d, keep)
        self._fill_meshes(d, keep)
        self._fill_materials(d, keep)
        d._keep = keep
        return d


# ---- canned scenes -----------------------------------------------------------------------

CORNELL_MATS = dict(white=(0.740063, 0.742313, 0.733934), red=(0.366046, 0.0371827, 0.0416385),
                    green=(0.162928, 0.408903, 0.0833759))


def cornell_walls(b, group=(0, 12, 0), half=(15, 12, 20), mats=None):
    """The five walls of scenes/cornell_box.json as 'plane' = Rectangle(2,2) instances inside a
    translate group (two spline levels per instance, Q18)."""
    if mats is None:
        mats = dict(white=b.add_material(F.MAT_MATTE, CORNELL_MATS["white"], roughness=1.0),
                    red=b.add_material(F.MAT_MATTE, CORNELL_MATS["red"], roughness=1.0),
                    green=b.add_material(F.MAT_MATTE, CORNELL_MATS["green"], roughness=1.0))
    g = trs(t=group)
    hx, hy, hz = half
    b.receiver(F.SHAPE_RECT, mats["white"], [trs(t=(0, 0, hz), s=(hx, hy, 1)), g], p0=2, p1=2)  # back
    b.receiver(F.SHAPE_RECT, mats["red"], [trs(t=(-hx, 0, 0), q=quat_axis_angle((0, 1, 0), 90), s=(hz, hy, 1)), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, mats["green"], [trs(t=(hx, 0, 0), q=quat_axis_angle((0, 1, 0), -90), s=(hz, hy, 1)), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, mats["white"], [trs(t=(0, hy, 0), q=quat_axis_angle((1, 0, 0), 90), s=(hx, hz, 1)), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, mats["white"], [trs(t=(0, -hy, 0), q=quat_axis_angle((1, 0, 0), 90), s=(hx, hz, 1)), g], p0=2, p1=2)
    return mats


def cornell_light(b, mat, emission=(1, 0.772549, 0.560784, 40)):
    return b.area_light(F.SHAPE_RECT, mat, [trs(t=(0, 23.8, 0), q=quat_axis_angle((1, 0, 0), 90))], emission, p0=6, p1=6)


def random_triangle_mesh(n_tris, seed, lo=(-13, 1, -8), hi=(13, 23, 18), jitter=0.15):
    """SURVEY.md §8d C4 mesh: centre ~U(box), vertices = centre + U([-j, j]^3), per-vertex normal
    = face normal, uvs (0,0),(1,0),(0,1). (numpy PCG64 stream; deterministic for a given seed.)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    c = rng.uniform(lo, hi, size=(n_tris, 1, 3))
    v = (c + rng.uniform(-jitter, jitter, size=(n_tris, 3, 3))).astype(np.float32)
    e0 = v[:, 1] - v[:, 0]
    e1 = v[:, 2] - v[:, 0]
    n = np.cross(e0.astype(np.float64), e1.astype(np.float64))
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    ln[ln == 0] = 1.0
    n = (n / ln).astype(np.float32)
    normals = np.repeat(n[:, None, :], 3, axis=1).reshape(-1, 3)
    uv = np.tile(np.array([[0, 0], [1, 0], [0, 1]], dtype=np.float32), (n_tris, 1))
    idx = np.arange(3 * n_tris, dtype=np.uint32).reshape(-1, 3)
    return v.reshape(-1, 3), normals, uv, idx


def heightfield_mesh(grid, seed, lo=(-13, -8), hi=(13, 18), base=5.0, amplitude=2.5, waves=6):
    """A grid x grid vertex heightfield y(x, z) over [lo, hi] in x and z, with shared vertices: 2 (grid - 1)^2 triangles from grid^2
    vertices, 4200 x 4200 giving 35 263 202 triangles in about 0.6 GB of attributes (a triangle soup of that size would need
    five times as much). The height is a sum of `waves` seeded sinusoids around `base`; normals are the analytic surface
    normals, texcoords (i / (grid - 1), j / (grid - 1)). Vertex j * grid + i sits at (x_i, y, z_j); cell (i, j) is the
    triangles (a, a + 1, a + grid + 1) and (a, a + grid + 1, a + grid) with a = j * grid + i."""
    assert grid >= 2
    rng = np.random.Generator(np.random.PCG64(seed))
    fx, fz = rng.uniform(-1.2, 1.2, size=(2, waves))
    phase = rng.uniform(0.0, 2.0 * math.pi, size=waves)
    amp = amplitude * rng.uniform(0.3, 1.0, size=waves) / math.sqrt(waves)
    xs, zs = np.linspace(lo[0], hi[0], grid), np.linspace(lo[1], hi[1], grid)
    X, Z = np.meshgrid(xs, zs)  # [j, i]
    H = np.full_like(X, base)
    dx, dz = np.zeros_like(X), np.zeros_like(X)
    for k in range(waves):
        s = fx[k] * X + fz[k] * Z + phase[k]
        H += amp[k] * np.sin(s)
        c = amp[k] * np.cos(s)
        dx += fx[k] * c
        dz += fz[k] * c
        del s, c
    positions = np.stack([X, H, Z], axis=-1).astype(np.float32).reshape(-1, 3)
    del X, Z, H
    inv = 1.0 / np.sqrt(dx * dx + dz * dz + 1.0)
    normals = np.stack([-dx * inv, inv, -dz * inv], axis=-1).astype(np.float32).reshape(-1, 3)
    del dx, dz, inv
    t = np.arange(grid, dtype=np.float32) / np.float32(grid - 1)
    texcoords = np.empty((grid, grid, 2), np.float32)
    texcoords[..., 0] = t[None, :]
    texcoords[..., 1] = t[:, None]
    a = (np.arange(grid - 1, dtype=np.uint32)[:, None] * np.uint32(grid) + np.arange(grid - 1, dtype=np.uint32)[None, :]).reshape(-1)
    idx = np.empty((2 * len(a), 3), np.uint32)
    idx[0::2, 0] = a; idx[0::2, 1] = a + 1; idx[0::2, 2] = a + grid + 1
    idx[1::2, 0] = a; idx[1::2, 1] = a + grid + 1; idx[1::2, 2] = a + grid
    return positions, normals, texcoords.reshape(-1, 2), idx


def icosphere_mesh(subdiv, radius=1.0, noise=0.0, seed=0):
    """Closed triangle mesh with smooth vertex normals and spherical uvs (C3 bunny stand-in)."""
    t = (1.0 + math.sqrt(5.0)) / 2.0
    verts = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
             (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    faces = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
             (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
             (9, 8, 1)]
    v = np.array(verts, dtype=np.float64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    f = np.array(faces, dtype=np.int64)
    for _ in range(subdiv):
        edges = {}
        vl = list(v)
        nf = []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in edges:
                m = (vl[a] + vl[b]) / 2.0
                vl.append(m / np.linalg.norm(m))
                edges[k] = len(vl) - 1
            return edges[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        v = np.array(vl)
        f = np.array(nf, dtype=np.int64)
    if noise > 0:
        rng = np.random.Generator(np.random.PCG64(seed))
        v = v * (1.0 + noise * rng.uniform(-1, 1, size=(len(v), 1)))
    # smooth normals from face normals
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    uv = np.stack([np.arctan2(v[:, 1], v[:, 0]) / (2 * math.pi) + 0.5, np.arccos(np.clip(v[:, 2] / np.linalg.norm(v, axis=1), -1, 1)) / math.pi], axis=1)
    return (v * radius).astype(np.float32), n.astype(np.float32), uv.astype(np.float32), f.astype(np.uint32)


def scene_c4(n_tris=1_000_000, width=1920, height=1080, spp=4096, seed=0x5EED1E55):
    """SURVEY.md §8d C4: synthetic random-triangle mesh inside the Cornell walls."""
    b = SceneBuilder(width, height, spp, 4, 8)
    mats = cornell_walls(b)
    cornell_light(b, mats["white"])
    m = b.add_mesh(*random_triangle_mesh(n_tris, seed))
    mat = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0)
    b.receiver(F.SHAPE_MESH, mat, [trs()], mesh=m)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def scene_heightfield(grid=4200, width=1920, height=1080, spp=4, seed=0x4E16F1D):
    """A large shared-vertex mesh inside the Cornell walls: the heightfield_mesh grid (4200: 35 M triangles, more than the 2^25
    a narrow mesh leaf reference can address, so the scene uses wide mesh leaves)."""
    b = SceneBuilder(width, height, spp, 4, 8)
    mats = cornell_walls(b)
    cornell_light(b, mats["white"])
    m = b.add_mesh(*heightfield_mesh(grid, seed))
    mat = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0)
    b.receiver(F.SHAPE_MESH, mat, [trs()], mesh=m)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def scene_instances(k, seed, width=64, height=64, spp=4, radius=0.3, mesh=False):
    """A Cornell box holding k small sphere receivers at seeded positions, each with a one-level static transform: the instance-heavy
    scene of the scene-edit tests and benchmark (every receiver's keyframe is one entry of the description's keyframes). With `mesh`
    the receivers are k instances of one shared 80-triangle icosphere instead, at the same positions."""
    b = SceneBuilder(width, height, spp, 2, 6)
    mats = cornell_walls(b)
    cornell_light(b, mats["white"])
    mat = b.add_material(F.MAT_MATTE, (0.74, 0.74, 0.73), roughness=1.0)
    shared = b.add_mesh(*icosphere_mesh(1)) if mesh else 0
    rng = np.random.Generator(np.random.PCG64(seed))
    for t in rng.uniform((-13, 1, -8), (13, 22, 18), size=(k, 3)):
        if mesh:
            b.receiver(F.SHAPE_MESH, mat, [trs(t=t, s=radius)], mesh=shared)
        else:
            b.receiver(F.SHAPE_SPHERE, mat, [trs(t=t, s=radius)], p0=1.0)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def scene_c3(width=800, height=600, spp=2048, subdiv=6, n_tris=69451):
    """SURVEY.md §8d C3 stand-in: Cornell box + a noisy icosphere cut to the Stanford bunny's 69 451 triangles (the bunny is not
    in the reference repo). The subdivision-6 icosphere has 81 920 faces; the lowest ones (a cap resting towards the floor) are
    dropped so the triangle count is the named one. n_tris=None keeps every face (small test scenes)."""
    b = SceneBuilder(width, height, spp, 4, 8)
    mats = cornell_walls(b)
    cornell_light(b, mats["white"])
    plastic = b.add_material(F.MAT_PLASTIC, (0.8, 0.8, 0.8), (0.6, 0.6, 0.6), roughness=0.5)
    p, n, t, f = icosphere_mesh(subdiv, 1.0, 0.05, 0xB0771E)
    if n_tris is not None and len(f) > n_tris:
        height_of = p[f].mean(axis=1)[:, 1]
        keep = np.sort(np.argsort(-height_of, kind="stable")[:n_tris])   # keep the highest faces, original order
        f = np.ascontiguousarray(f[keep])
    m = b.add_mesh(p, n, t, f)
    b.receiver(F.SHAPE_MESH, plastic, [trs(t=(4, 4.2, -3), q=quat_axis_angle((0, 1, 0), 15), s=4.0)], mesh=m)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def scene_smallpt_like(width=512, height=512, spp=1024):
    """scenes/smallpt.json shape built from TRS: 5 walls scaled 32, metal + glass spheres, sphere light."""
    b = SceneBuilder(width, height, spp, 4, 8)
    white = b.add_material(F.MAT_MATTE, (1, 1, 1), roughness=1.0)
    red = b.add_material(F.MAT_MATTE, (1, 0.2, 0.2), roughness=1.0)
    blue = b.add_material(F.MAT_MATTE, (0.2, 0.2, 1.0), roughness=1.0)
    metal = b.add_material(F.MAT_METAL, (0.155265, 0.116723, 0.138381), (4.82835, 3.12225, 2.14696), roughness=0.2)
    glass = b.add_material(F.MAT_GLASS, (1, 1, 1), (1, 1, 1), eta=1.52)
    g = trs(t=(0, 12, 0))
    b.receiver(F.SHAPE_RECT, white, [trs(t=(0, 0, 20), s=32), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, red, [trs(t=(-15, 0, 0), q=quat_axis_angle((0, 1, 0), 90), s=32), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, blue, [trs(t=(15, 0, 0), q=quat_axis_angle((0, 1, 0), -90), s=32), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, white, [trs(t=(0, 12, 0), q=quat_axis_angle((1, 0, 0), 90), s=32), g], p0=2, p1=2)
    b.receiver(F.SHAPE_RECT, white, [trs(t=(0, -12, 0), q=quat_axis_angle((1, 0, 0), 90), s=32), g], p0=2, p1=2)
    b.receiver(F.SHAPE_SPHERE, metal, [trs(t=(-6, 5, 8), s=5)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, glass, [trs(t=(6, 5, -2), s=5)], p0=1.0)
    b.area_light(F.SHAPE_SPHERE, white, [trs(t=(0, 22, 0))], (0.780131, 0.780409, 0.775833, 60), p0=1.0)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def scene_animated(width=64, height=64, spp=8, frames=4, scene_time=1.0, animated_fov=False):
    """Small keyframed scene (SURVEY 8f N1, the tr15 feature set): B-spline animated receivers (one- and two-level
    stacks), a moving area light with keyframed emission, a moving point light and a keyframed camera."""
    b = SceneBuilder(width, height, spp, 2, 6)
    b.film.update(frames=frames, start_frame=0, end_frame=frames - 1, scene_time=scene_time)
    mats = cornell_walls(b)
    plastic = b.add_material(F.MAT_PLASTIC, (0.2, 0.6, 0.9), (0.7, 0.7, 0.7), roughness=0.2)
    metal = b.add_material(F.MAT_METAL, (0.155265, 0.116723, 0.138381), (4.82835, 3.12225, 2.14696), roughness=0.3)
    glass = b.add_material(F.MAT_GLASS, (1, 1, 1), (1, 1, 1), eta=1.5)
    # a sphere flying along a cubic spline while spinning and pulsing
    fly = Anim([trs(t=(-9, 3, 6), s=2.0), trs(t=(-3, 9, 2), q=quat_axis_angle((0, 1, 0), 80), s=3.0),
                trs(t=(4, 5, -2), q=quat_axis_angle((0, 1, 0), 160), s=2.5), trs(t=(9, 8, 4), q=quat_axis_angle((1, 1, 0), 200), s=2.0),
                trs(t=(6, 3, 8), q=quat_axis_angle((1, 0, 0), 270), s=3.0)], degree=3)
    b.receiver(F.SHAPE_SPHERE, plastic, [fly], p0=1.0)
    # a mesh spinning about its own axis (animated inner level) inside a static placement (two-level stack, Q22: bounds are NOT sampled)
    m = b.add_mesh(*icosphere_mesh(2, 1.0, 0.1, 0x5EED))
    spin = Anim([trs(q=quat_axis_angle((0, 1, 0), a)) for a in (0, 90, 170, 250)], degree=2)
    b.receiver(F.SHAPE_MESH, metal, [spin, trs(t=(0, 4, 0), s=3.0)], mesh=m)
    # a glass sphere on a linear (degree-1) path placed through a static outer level
    b.receiver(F.SHAPE_SPHERE, glass, [trs(s=2.0), Anim([trs(t=(-6, 12, -4)), trs(t=(6, 14, -6))], degree=1)], p0=1.0)
    # moving area light with keyframed emission; static panel light; moving point light
    slide = Anim([trs(t=(-6, 23.5, 0), q=quat_axis_angle((1, 0, 0), 90)), trs(t=(0, 22, 4), q=quat_axis_angle((1, 0, 0), 100)),
                  trs(t=(6, 23.5, 0), q=quat_axis_angle((1, 0, 0), 80))], degree=2)
    b.area_light(F.SHAPE_DISK, mats["white"], [slide], [((1.0, 0.6, 0.3, 30), 0.0), ((0.3, 1.0, 0.4, 60), 0.4), ((0.4, 0.5, 1.0, 20), 0.9)],
                 p0=3.0, p1=0.0)
    b.area_light(F.SHAPE_RECT, mats["white"], [trs(t=(0, 23.9, 8), q=quat_axis_angle((1, 0, 0), 90))], (1, 1, 1, 8), p0=6.0, p1=4.0)
    b.point_light([Anim([trs(t=(-10, 15, -12)), trs(t=(10, 18, -10))], degree=1)], [((1, 1, 1, 120), 0.2), ((1, 0.5, 0.5, 60), 0.8)])
    b.add_camera([Anim([trs(t=(-3, 12, -60)), trs(t=(0, 13, -58), q=quat_axis_angle((0, 1, 0), 3)), trs(t=(4, 12, -60), q=quat_axis_angle((0, 1, 0), -4))],
                       degree=2)], fov=[28.0, 34.0, 30.0, 26.0] if animated_fov else 30.0, fov_degree=2, shutter_size=0.5)
    return b


def scene_materials_zoo(width=64, height=64, spp=16, merl_table=None):
    """Small scene touching every material / shape / light kind, for parity tests."""
    b = SceneBuilder(width, height, spp, 2, 6)
    mats = cornell_walls(b)
    cornell_light(b, mats["white"])
    b.point_light([trs(t=(-8, 18, -10))], (1, 1, 1, 150))
    b.area_light(F.SHAPE_DISK, mats["white"], [trs(t=(9, 20, 5), q=quat_axis_angle((1, 0, 0), 90))], (0.5, 0.8, 1.0, 30), p0=2.0, p1=0.5)
    plastic = b.add_material(F.MAT_PLASTIC, (0.8, 0.2, 0.2), (0.8, 0.8, 0.8), roughness=0.1)
    metal = b.add_material(F.MAT_METAL, (0.155265, 0.116723, 0.138381), (4.82835, 3.12225, 2.14696), roughness=0.2)
    smetal = b.add_material(F.MAT_SPECULAR_METAL, (0.2, 0.9, 1.1), (3.9, 2.4, 2.2))
    glass = b.add_material(F.MAT_GLASS, (1, 1, 1), (1, 1, 1), eta=1.52)
    rglass = b.add_material(F.MAT_ROUGH_GLASS, (1, 1, 1), (0.9, 1, 0.9), roughness=0.3, eta=1.4)
    lamb = b.add_material(F.MAT_MATTE, (0.6, 0.6, 0.2), roughness=0.0)
    b.receiver(F.SHAPE_SPHERE, plastic, [trs(t=(-9, 3, 4), s=3)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, metal, [trs(t=(-3, 3, 8), s=3)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, smetal, [trs(t=(3, 3, 8), s=3)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, glass, [trs(t=(9, 3, 2), s=3)], p0=1.0)
    b.receiver(F.SHAPE_SPHERE, rglass, [trs(t=(0, 3, -4), s=3)], p0=1.0)
    b.receiver(F.SHAPE_DISK, lamb, [trs(t=(0, 9, 12), q=quat_axis_angle((0, 1, 0), 180))], p0=4.0, p1=1.0)
    if merl_table is not None:
        mi = b.add_merl_table(merl_table)
        merl = b.add_material(F.MAT_MERL, merl=mi)
        b.receiver(F.SHAPE_SPHERE, merl, [trs(t=(-6, 10, 10), s=2.5)], p0=1.0)
    m = b.add_mesh(*icosphere_mesh(2, 1.0, 0.1, 7))
    b.receiver(F.SHAPE_MESH, plastic, [trs(t=(6, 10, 8), q=quat_axis_angle((1, 1, 0), 30), s=(2.5, 3.0, 2.5))], mesh=m)
    b.add_camera([trs(t=(0, 12, -60))], fov=30.0)
    return b


def synthetic_merl_table(seed=1):
    """A valid-shaped MERL table (90*90*180 rgb) from an analytic lobe (SURVEY §8d: real MERL files are not in the repo)."""
    th = (np.arange(90, dtype=np.float32) / 90.0) ** 2 * (math.pi / 2)
    td = np.arange(90, dtype=np.float32) / 90.0 * (math.pi / 2)
    lobe = np.exp(-(th[:, None] ** 2) / 0.05) * 4.0 + 0.2
    fres = 0.04 + 0.96 * (1 - np.cos(td)) ** 5
    base = (lobe * (0.3 + fres[None, :])).astype(np.float32)  # (theta_h, theta_d)
    t = np.repeat(base[:, :, None], 180, axis=2)
    rgb = np.stack([t * 0.9, t * 0.7, t * 0.5], axis=-1).astype(np.float32)
    return rgb.reshape(-1)

"""Film writes without a GPU: the exports and their Rust declarations, a plain-C caller, the argument checks that need no device, an
independent float32 restatement of RenderTarget::write (render_target.rs:77-165) against orc_film_write, and orc_film_write over
orc_render_samples against a one-thread orc_render."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from oracle_queries import pyqueries as Q
from test_queries_gpu import json_desc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_film_write", "trb_film_write_device", "trb_camera_rays_device"]
f32 = np.float32


def _c_run(tmp_path):
    exe = str(tmp_path / "film_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "film_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_plain_c_caller_gets_invalid_arg_for_null_arguments(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _c_run(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {n: F.TRB_INVALID_ARG for n in NEW}


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    assert F.SAMPLE_DTYPE.itemsize == C.sizeof(F.Sample) == 20
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
                assert c is {"usize": C.c_size_t, "u32": C.c_uint32}[r], (name, i, r, c)
        assert "`%s(" % name in doc or "`%s`" % name in doc, "no table row for " + name


def test_argument_checks_need_no_device(trb):
    s = np.zeros(1, F.SAMPLE_DTYPE)
    reg = np.zeros(1, np.uint32)
    film = np.zeros(8, np.float32)
    rays = np.zeros(2, F.RAY_DTYPE)
    xy = np.zeros(4, np.float32)
    fake = C.c_void_p(1)  # never dereferenced: every call below fails its argument checks first
    off = lambda a, k: F.ptr(a.view(np.uint8)[k:])  # noqa: E731
    cfg = api._cfg()
    calls = [
        lambda: trb.trb_film_write(None, 0, None, None, None),
        lambda: trb.trb_film_write(fake, 1, None, F.ptr(reg), F.ptr(film)),
        lambda: trb.trb_film_write(fake, 1, F.ptr(s), None, F.ptr(film)),
        lambda: trb.trb_film_write(fake, 1, F.ptr(s), F.ptr(reg), None),
        lambda: trb.trb_film_write(fake, 1 << 32, F.ptr(s), F.ptr(reg), F.ptr(film)),  # n >= 2^32: refused before anything is read
        lambda: trb.trb_film_write_device(fake, (1 << 32) + 5, F.ptr(s), F.ptr(reg), F.ptr(film), None),
        lambda: trb.trb_film_write_device(fake, 1, off(s, 2), F.ptr(reg), F.ptr(film), None),
        lambda: trb.trb_film_write_device(fake, 1, F.ptr(s), off(reg, 1), F.ptr(film), None),
        lambda: trb.trb_film_write_device(fake, 1, F.ptr(s), F.ptr(reg), off(film, 2), None),
        lambda: trb.trb_camera_rays_device(None, C.byref(cfg), 1, F.ptr(rays), F.ptr(xy), None),
        lambda: trb.trb_camera_rays_device(fake, None, 1, F.ptr(rays), F.ptr(xy), None),
        lambda: trb.trb_camera_rays_device(fake, C.byref(cfg), 1, None, F.ptr(xy), None),
        lambda: trb.trb_camera_rays_device(fake, C.byref(cfg), 1, off(rays, 2), F.ptr(xy), None),
        lambda: trb.trb_camera_rays_device(fake, C.byref(cfg), 1, F.ptr(rays), off(xy, 1), None),
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k


# ---- RenderTarget::write restated ---------------------------------------------------------------------------------------------
def restated_write(film, samples, regions, width, height, fw, fh, table):
    """render_target.rs:77-165 in numpy float32 scalars, literal loops: regions in BlockQueue::new's Morton order (morton.rs), each
    region's samples in input order, 2x2 lock blocks, filtered_samples summed then added."""
    fpw = (int(np.floor(f32(fw) / f32(0.5))), int(np.floor(f32(fh) / f32(0.5))))
    inv_w, inv_h = f32(1.0) / f32(fw), f32(1.0) / f32(fh)
    nbx, nby = width // 8, height // 8

    def part(v):
        return sum(((v >> k) & 1) << (2 * k) for k in range(16))

    blocks = sorted(range(nbx * nby), key=lambda i: (part(i // nbx) << 1) + part(i % nbx))
    for r in blocks:
        sel = [s for s, g in zip(samples, regions) if g == r]
        if not sel:
            continue
        sx0, sy0 = (r % nbx) * 8, (r // nbx) * 8
        xr = (max(sx0 - fpw[0], 0), min(sx0 + 8 + fpw[0], width - 1))
        yr = (max(sy0 - fpw[1], 0), min(sy0 + 8 + fpw[1], height - 1))
        for by in range(yr[0] // 2, yr[1] // 2 + 1):
            for bx in range(xr[0] // 2, xr[1] // 2 + 1):
                xw = (max(xr[0], bx * 2), min(xr[1] + 1, bx * 2 + 2))
                yw = (max(yr[0], by * 2), min(yr[1] + 1, by * 2 + 2))
                acc = np.zeros((2, 2, 4), np.float32)
                for s in sel:
                    x, y = f32(s["x"]), f32(s["y"])
                    if not (x >= f32(xw[0] - fpw[0]) and x < f32(xw[1] + fpw[0]) and y >= f32(yw[0] - fpw[1]) and y < f32(yw[1] + fpw[1])):
                        continue
                    img_x, img_y = x - f32(0.5), y - f32(0.5)
                    for iy in range(yw[0], yw[1]):
                        fy = abs(f32(iy) - img_y) * inv_h
                        if fy > f32(fh):
                            continue
                        fyi = min(int(fy * f32(16.0)), 15)
                        for ix in range(xw[0], xw[1]):
                            fx = abs(f32(ix) - img_x) * inv_w
                            if fx > f32(fw):
                                continue
                            wgt = table[fyi, min(int(fx * f32(16.0)), 15)]
                            a = acc[iy - by * 2, ix - bx * 2]
                            a[0] = a[0] + wgt * f32(s["r"]); a[1] = a[1] + wgt * f32(s["g"]); a[2] = a[2] + wgt * f32(s["b"])
                            a[3] = a[3] + wgt
                for iy in range(yw[0], yw[1]):
                    for ix in range(xw[0], xw[1]):
                        film[iy, ix] = film[iy, ix] + acc[iy - by * 2, ix - bx * 2]
    return film


def random_samples(rng, n, width, height, spread=20.0):
    """samples near their region's block and up to `spread` px beyond it, some exactly on pixel and block edges, negative colours"""
    nr = (width // 8) * (height // 8)
    regions = rng.integers(0, nr, n).astype(np.uint32)
    s = np.zeros(n, F.SAMPLE_DTYPE)
    bx, by = (regions % (width // 8)) * 8, (regions // (width // 8)) * 8
    s["x"] = (bx + rng.uniform(-spread, 8 + spread, n)).astype(np.float32)
    s["y"] = (by + rng.uniform(-spread, 8 + spread, n)).astype(np.float32)
    edge = rng.random(n) < 0.2
    s["x"][edge] = (bx[edge] + rng.integers(-2, 11, edge.sum())).astype(np.float32)
    s["y"][edge] = (by[edge] + 8).astype(np.float32)
    for k in ("r", "g", "b"):
        s[k] = rng.uniform(-0.5, 2.0, n).astype(np.float32)
    return s, regions


def test_restated_write_equals_orc_film_write():
    for w, h, ftype, fw, fh, fb, seed in [(24, 16, F.FILTER_MITCHELL_NETRAVALI, 2.0, 2.0, 1 / 3, 1),
                                           (16, 24, F.FILTER_GAUSSIAN, 3.0, 2.5, 0.5, 2),
                                           (24, 24, F.FILTER_GAUSSIAN, 4.0, 4.0, 0.5, 3)]:
        b = SB.scene_smallpt_like(w, h, 1)
        b.film.update(filter_type=ftype, filter_w=fw, filter_h=fh, filter_b=fb, filter_c=1 / 3 if ftype == F.FILTER_MITCHELL_NETRAVALI else 0.0)
        o = Q.QueryOracleScene(b.finish())
        rng = np.random.default_rng(seed)
        s, reg = random_samples(rng, 300, w, h)
        reg[:5] = (w // 8) * (h // 8) + np.arange(5)  # out of range: skipped
        film0 = rng.uniform(-1, 1, (h, w, 4)).astype(np.float32)
        film0[0, 0] = -0.0
        want = restated_write(film0.copy(), s, reg, w, h, fw, fh, o.filter_table())
        got = o.film_write(s, reg, film0.copy())
        assert got.tobytes() == want.tobytes(), (w, h, ftype, fw)
        assert not np.array_equal(got, film0)


def _composition(desc, **kw):
    o = Q.QueryOracleScene(desc)
    o.update_frame(0, 0.0, 0.0)
    samples, _ = o.render_samples(seed=7, **kw)
    film = o.film_write(samples, o.sample_regions(**kw))
    ref, _ = o.render(seed=7, threads=1, flags=F.RENDER_NO_UPDATE, **kw)
    return film, ref


def test_orc_film_write_of_render_samples_is_the_one_thread_render():
    wide = SB.scene_c4(20000, 64, 40, 2)  # the wide-Gaussian film of test_wide_gaussian_filter_film_vs_oracle, smaller
    wide.film.update(filter_type=F.FILTER_GAUSSIAN, filter_w=3.0, filter_h=2.5, filter_b=0.5, filter_c=0.0)
    for name, desc in [("c1", json_desc("c1_cornell_box.json", 32, 24, 2)), ("c2", json_desc("c2_smallpt.json", 32, 32, 2)),
                       ("wide", wide.finish())]:
        film, ref = _composition(desc)
        assert film.tobytes() == ref.tobytes(), name
        assert film[..., 3].min() > 0, name

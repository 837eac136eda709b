"""The shading queries without a GPU: the query and result layouts (plain C, ctypes, numpy and the Rust declarations in INTEGRATION.md),
the exports and the argument checks that need no device, and the oracle's orc_bsdf_* / orc_light_* / orc_emitted against closed forms."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, scenebuild as SB
from oracle_queries import pyqueries as Q

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_bsdf_eval", "trb_bsdf_eval_device", "trb_bsdf_sample", "trb_bsdf_sample_device", "trb_light_sample", "trb_light_sample_device",
       "trb_light_pdf", "trb_light_pdf_device", "trb_emitted", "trb_emitted_device", "trb_scene_lights"]
# C struct -> (ctypes class, numpy dtype, Rust struct name in INTEGRATION.md)
STRUCTS = {
    "trb_bsdf_eval_query": (F.BsdfEvalQuery, F.BSDF_EVAL_QUERY_DTYPE, "TrbBsdfEvalQuery"),
    "trb_bsdf_sample_query": (F.BsdfSampleQuery, F.BSDF_SAMPLE_QUERY_DTYPE, "TrbBsdfSampleQuery"),
    "trb_bsdf_sample_result": (F.BsdfSampleResult, F.BSDF_SAMPLE_DTYPE, "TrbBsdfSampleResult"),
    "trb_light_query": (F.LightQuery, F.LIGHT_QUERY_DTYPE, "TrbLightQuery"),
    "trb_light_sample_result": (F.LightSampleResult, F.LIGHT_SAMPLE_DTYPE, "TrbLightSampleResult"),
    "trb_light_pdf_query": (F.LightPdfQuery, F.LIGHT_PDF_QUERY_DTYPE, "TrbLightPdfQuery"),
    "trb_emit_query": (F.EmitQuery, F.EMIT_QUERY_DTYPE, "TrbEmitQuery"),
}


def _c_run(tmp_path):
    exe = str(tmp_path / "shading_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "shading_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def test_plain_c_layouts_match_ctypes_numpy_and_the_rust_declarations(tmp_path):
    lines = _c_run(tmp_path)
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    rust_size = {"f32": 4, "u32": 4, "TrbQueryRay": 48}
    for cname, (ct, dt, rname) in STRUCTS.items():
        size = [int(l.split()[2]) for l in lines if l.startswith(cname + " sizeof ")][0]
        offsets = [(l.split()[0].split(".")[1], int(l.split()[1])) for l in lines if l.startswith(cname + ".")]
        assert C.sizeof(ct) == size == dt.itemsize and size % 16 == 0, cname
        assert [(f, getattr(ct, f).offset) for f, _ in ct._fields_] == offsets, cname
        assert [(f, dt.fields[f][1]) for f in dt.names] == offsets, cname
        m = re.search(r"pub struct %s \{(.*?)\}" % rname, doc, re.S)
        assert m, rname
        fields = re.findall(r"(\w+)\s*:\s*(\[(\w+);\s*(\d+)\]|\w+)", m.group(1))
        off = 0
        for (name, whole, elem, count), (cf, co) in zip(fields, offsets):
            assert name == cf and off == co, (rname, name)
            off += rust_size[elem] * int(count) if elem else rust_size[whole]
        assert len(fields) == len(offsets) and off == size, rname
    assert F.LIGHT_SAMPLE_DTYPE.fields["shadow"][0] == F.QUERY_RAY_DTYPE


def test_plain_c_caller_gets_invalid_arg_for_null_arguments(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _c_run(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG
    assert status == {n: F.TRB_INVALID_ARG for n in NEW}


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
            want = C.c_void_p if r.startswith("*") else {"usize": C.c_size_t, "u32": C.c_uint32}[r]
            assert c is want, (name, i, r, c)
        assert "`%s(" % name in doc or "`%s`" % name in doc, "no table row for " + name


def test_argument_checks_need_no_device(trb):
    rec = np.zeros(1, F.INTERSECTION_DTYPE)
    eq, sq = np.zeros(1, F.BSDF_EVAL_QUERY_DTYPE), np.zeros(1, F.BSDF_SAMPLE_QUERY_DTYPE)
    lq, pq, mq = np.zeros(1, F.LIGHT_QUERY_DTYPE), np.zeros(1, F.LIGHT_PDF_QUERY_DTYPE), np.zeros(1, F.EMIT_QUERY_DTYPE)
    out = np.zeros(32, np.float32)  # 128 bytes, 16-byte aligned: room for any one result
    fake = C.c_void_p(1)  # never dereferenced: every call below fails its argument checks first
    off = lambda a, k: F.ptr(a.view(np.uint8)[k:])  # noqa: E731
    calls = [
        lambda: trb.trb_bsdf_eval(fake, 1, None, F.ptr(eq), F.ptr(out)),
        lambda: trb.trb_bsdf_eval(fake, 1, F.ptr(rec), None, F.ptr(out)),
        lambda: trb.trb_bsdf_eval(fake, 1, F.ptr(rec), F.ptr(eq), None),
        lambda: trb.trb_bsdf_eval_device(fake, 1, off(rec, 4), F.ptr(eq), F.ptr(out), None),
        lambda: trb.trb_bsdf_eval_device(fake, 1, F.ptr(rec), off(eq, 8), F.ptr(out), None),
        lambda: trb.trb_bsdf_eval_device(fake, 1, F.ptr(rec), F.ptr(eq), off(out, 4), None),  # float4 output: 16-byte
        lambda: trb.trb_bsdf_sample(fake, 1, F.ptr(rec), None, F.ptr(out)),
        lambda: trb.trb_bsdf_sample_device(fake, 1, F.ptr(rec), F.ptr(sq), off(out, 8), None),
        lambda: trb.trb_light_sample(fake, 1, None, F.ptr(out)),
        lambda: trb.trb_light_sample(fake, 1, F.ptr(lq), None),
        lambda: trb.trb_light_sample_device(fake, 1, off(lq, 4), F.ptr(out), None),
        lambda: trb.trb_light_sample_device(fake, 1, F.ptr(lq), off(out, 4), None),
        lambda: trb.trb_light_pdf(fake, 1, None, F.ptr(out)),
        lambda: trb.trb_light_pdf_device(fake, 1, off(pq, 4), F.ptr(out), None),
        lambda: trb.trb_light_pdf_device(fake, 1, F.ptr(pq), off(out, 2), None),  # float output: 4-byte
        lambda: trb.trb_emitted(fake, 1, F.ptr(mq), None),
        lambda: trb.trb_emitted_device(fake, 1, off(mq, 4), F.ptr(out), None),
        lambda: trb.trb_emitted_device(fake, 1, F.ptr(mq), off(out, 2), None),
        lambda: trb.trb_emitted(None, 0, None, None),
        lambda: trb.trb_scene_lights(None, F.ptr(out)),
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k


# ---- the oracle against closed forms ----------------------------------------------------------------------------------------
R = (0.5, 0.25, 0.125)


def closed_form_scene():
    """a Lambertian rectangle at the origin (normal +z), a point light, a sphere light, a rectangle light and a disk light"""
    b = SB.SceneBuilder(8, 8, 1)
    lamb = b.add_material(F.MAT_MATTE, R, roughness=0.0)
    b.receiver(F.SHAPE_RECT, lamb, [SB.trs()], p0=2.0, p1=2.0)                                            # 0
    b.point_light([SB.trs(t=(0, 10, 0))], (1, 1, 1, 100))                                                  # 1
    b.area_light(F.SHAPE_SPHERE, lamb, [SB.trs(t=(0, 0, 10))], (2, 3, 4), p0=1.0)                          # 2
    b.area_light(F.SHAPE_RECT, lamb, [SB.trs(t=(0, 0, 5))], (1, 1, 1), p0=2.0, p1=2.0)                     # 3
    b.area_light(F.SHAPE_DISK, lamb, [SB.trs(t=(20, 0, 5))], (1, 1, 1), p0=2.0, p1=1.0)                    # 4
    b.add_camera([SB.trs(t=(0, 0, -10))])
    return b.finish()


def _oracle(frame=True):
    o = Q.QueryOracleScene(closed_form_scene())
    if frame:
        o.update_frame(0, 0.0, 0.0)
    return o


def _record(material=0, n=(0, 0, 1), dp_du=(1, 0, 0), inst=0):
    r = np.zeros(1, F.INTERSECTION_DTYPE)
    r["inst"], r["material"], r["n"], r["ng"], r["dp_du"] = inst, material, n, n, dp_du
    return r


def test_lambertian_eval_is_r_over_pi_and_pdf_cos_over_pi():
    o = _oracle(frame=False)  # BSDF queries need no frame
    th = np.linspace(0.0, 1.5, 7, dtype=np.float32)
    q = np.zeros(len(th), F.BSDF_EVAL_QUERY_DTYPE)
    q["wo"] = (0.0, 0.6, 0.8)
    q["wi"] = np.stack([np.sin(th), np.zeros_like(th), np.cos(th)], axis=1)
    q["bxdf"] = F.BXDF_ALL
    out = o.bsdf_eval(np.repeat(_record(), len(q)), q)
    assert np.allclose(out[:, :3], np.float32(R) / np.float32(math.pi), rtol=1e-6, atol=0)
    assert np.allclose(out[:, 3], np.cos(th) / math.pi, rtol=1e-5, atol=1e-7)
    q["bxdf"] = F.BXDF_SPECULAR | F.BXDF_REFLECTION  # no such lobe
    assert not o.bsdf_eval(np.repeat(_record(), len(q)), q).any()
    q["wi"][:, 2] *= -1.0  # the other hemisphere: reflection lobes are not evaluated for transmission
    q["bxdf"] = F.BXDF_ALL
    assert not o.bsdf_eval(np.repeat(_record(), len(q)), q)[:, :3].any()
    s = np.zeros(3, F.BSDF_SAMPLE_QUERY_DTYPE)
    s["wo"], s["bxdf"], s["u"], s["u_comp"] = (0, 0, 1), F.BXDF_ALL, [(0.1, 0.2), (0.5, 0.5), (0.9, 0.3)], 0.5
    res = o.bsdf_sample(np.repeat(_record(), 3), s)
    assert (res["sampled"] == F.BXDF_DIFFUSE | F.BXDF_REFLECTION).all()
    assert np.allclose(res["pdf"], res["wi"][:, 2] / math.pi, rtol=1e-5) and np.allclose(res["f"], np.float32(R) / np.float32(math.pi), rtol=1e-6)


def test_point_light_is_i_over_d2_with_pdf_1_and_pdf_query_0():
    o = _oracle()
    q = np.zeros(2, F.LIGHT_QUERY_DTYPE)
    q["p"] = [(0, 0, 0), (0, 5, 0)]
    q["light"] = 1
    q["time"] = 0.0
    s = o.light_sample(q)
    assert np.allclose(s["li"], [[1, 1, 1], [4, 4, 4]], rtol=1e-6)
    assert (s["pdf"] == 1.0).all() and (s["delta"] == 1).all()
    assert np.array_equal(s["wi"], [[0, 1, 0], [0, 1, 0]])
    assert np.array_equal(s["shadow"]["o"], q["p"]) and np.array_equal(s["shadow"]["d"], [[0, 10, 0], [0, 5, 0]])
    assert (s["shadow"]["min_t"] == np.float32(0.001)).all() and (s["shadow"]["max_t"] == np.float32(0.999)).all()
    p = np.zeros(1, F.LIGHT_PDF_QUERY_DTYPE)
    p["wi"], p["light"] = (0, 1, 0), 1
    assert o.light_pdf(p)[0] == 0.0


def test_sphere_light_pdf_is_the_cone_pdf():
    o = _oracle()
    q = np.zeros(3, F.LIGHT_QUERY_DTYPE)
    q["p"], q["u"], q["light"] = (0, 0, 0), [(0.1, 0.2), (0.5, 0.5), (0.9, 0.7)], 2
    s = o.light_sample(q)
    cos_max = math.sqrt(1.0 - 1.0 / 100.0)
    want = 1.0 / (2.0 * math.pi * (1.0 - cos_max))
    assert np.allclose(s["pdf"], want, rtol=1e-3) and (s["delta"] == 0).all()
    assert np.allclose(s["li"], [2, 3, 4]) and (s["wi"][:, 2] >= cos_max - 1e-6).all()
    p = np.zeros(2, F.LIGHT_PDF_QUERY_DTYPE)
    p["wi"], p["light"] = [(0, 0, 1), (1, 0, 0)], 2  # the cone pdf does not depend on the direction
    assert np.allclose(o.light_pdf(p), want, rtol=1e-3)
    inside = np.zeros(1, F.LIGHT_PDF_QUERY_DTYPE)
    inside["p"], inside["wi"], inside["light"] = (0, 0, 10), (0, 0, 1), 2  # inside the sphere: uniform over the area, 4*pi*r (Q3)
    assert np.isclose(o.light_pdf(inside)[0], 1.0 / (4.0 * math.pi))


def test_rectangle_light_pdf_is_d2_over_cos_area():
    o = _oracle()
    wi = np.array([(0, 0, 1), (0.1, 0.05, 1.0), (-0.15, 0.1, 1.0)], np.float32)  # hits inside the 2 x 2 rectangle 5 away
    wi /= np.linalg.norm(wi, axis=1, keepdims=True)
    p = np.zeros(3, F.LIGHT_PDF_QUERY_DTYPE)
    p["wi"], p["light"] = wi, 3
    t = 5.0 / wi[:, 2]
    want = t * t / (wi[:, 2] * 4.0)
    assert np.allclose(o.light_pdf(p), want, rtol=1e-5)
    p["wi"] = (0.9, 0.0, 0.1)  # misses the rectangle
    assert (o.light_pdf(p) == 0).all()
    d = np.zeros(2, F.LIGHT_PDF_QUERY_DTYPE)
    d["p"], d["wi"], d["light"] = (20, 0, 0), [(0, 0, 1), (0.3, 0, 1)], 4  # through the disk's hole, then onto the ring
    got = o.light_pdf(d)
    assert got[0] == 0.0 and got[1] > 0.0


def test_emitted_is_black_from_behind_and_for_receivers():
    o = _oracle(frame=False)  # needs no frame
    q = np.zeros(6, F.EMIT_QUERY_DTYPE)
    q["n"] = (0, 0, 1)
    q["w"] = [(0, 0, 1), (0, 0, -1), (0, 0, 0), (0, 0, 1), (0, 0, 1), (0, 0, 1)]
    q["inst"] = [2, 2, 2, 0, F.MISS, 99]
    rgb = o.emitted(q)
    assert np.array_equal(rgb[0], [2, 3, 4]) and not rgb[1:].any()


def test_out_of_range_indices_give_zeros_and_light_queries_need_a_frame():
    o = _oracle(frame=False)
    lq = np.zeros(1, F.LIGHT_QUERY_DTYPE)
    with pytest.raises(Exception):
        o.light_sample(lq)
    with pytest.raises(Exception):
        o.light_pdf(np.zeros(1, F.LIGHT_PDF_QUERY_DTYPE))
    o.update_frame(0, 0.0, 0.0)
    assert np.array_equal(o.lights(), [1, 2, 3, 4])
    lq = np.zeros(3, F.LIGHT_QUERY_DTYPE)
    lq["light"] = [0, 5, F.MISS]  # a receiver, past the instances
    lq["u"] = 0.5
    assert not o.light_sample(lq).view(np.uint8).any()
    recs = np.concatenate([_record(material=1), _record(inst=F.MISS)])
    q = np.zeros(2, F.BSDF_SAMPLE_QUERY_DTYPE)
    q["wo"], q["bxdf"], q["u"], q["u_comp"] = (0, 0, 1), F.BXDF_ALL, 0.5, 0.5
    assert not o.bsdf_sample(recs, q).view(np.uint8).any()

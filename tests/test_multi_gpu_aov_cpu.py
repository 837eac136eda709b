"""The multi-GPU AOV renders without a GPU: the four entry points are exported, bound with the signatures INTEGRATION.md documents
for Rust callers, callable from plain C, and refuse null and bad arguments before any device is touched; trb_tray and trb_worker
refuse every malformed use of --devices before anything renders."""
import ctypes as C
import os
import re
import subprocess

import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_sharded_aov", "trb_render_sharded_adaptive_aov", "trb_group_render_aov", "trb_group_render_adaptive_aov"]


def test_new_symbols_are_exported_and_listed(trb):
    for name in NEW:
        assert hasattr(trb, name), name
        assert name in F.TRB_SYMBOLS, name


def _rust_params(doc, name):
    m = re.search(r"fn %s\((.*?)\)\s*->\s*c_int;" % name, doc, re.S)
    assert m, name
    return [p.split(":", 1)[1].strip() for p in m.group(1).split(",") if p.strip()]


# what each Rust parameter type may be bound to in ctypes: the struct pointer itself, or an untyped pointer
RUST_TO_CTYPES = {
    "*mut c_void": (C.c_void_p,),
    "*const TrbRenderCfg": (C.POINTER(F.RenderCfg),),
    "*const TrbAdaptive": (C.POINTER(F.Adaptive),),
    "*const TrbAovFilm": (C.POINTER(F.AovFilm),),
    "*mut TrbStats": (C.POINTER(F.Stats), C.c_void_p),
    "*mut f32": (C.c_void_p,),
    "*mut u32": (C.c_void_p,),
    "c_int": (C.c_int,),
}


def test_ctypes_signatures_match_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    for name in NEW:
        rust = _rust_params(doc, name)
        ct = getattr(trb, name).argtypes
        assert ct is not None and len(ct) == len(rust), name
        for i, (r, c) in enumerate(zip(rust, ct)):
            assert c in RUST_TO_CTYPES[r], (name, i, r, c)
        assert "`%s(" % name in doc, "no table row for " + name


def test_plain_c_caller_builds_links_and_gets_invalid_arg(tmp_path):
    exe = str(tmp_path / "multi_gpu_aov_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "multi_gpu_aov_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = dict(line.split() for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["TRB_INVALID_ARG"]) == F.TRB_INVALID_ARG
    assert {k: int(v) for k, v in out.items() if k != "TRB_INVALID_ARG"} == {n: F.TRB_INVALID_ARG for n in NEW}


def test_null_and_bad_arguments_are_rejected_before_any_device_is_touched(trb):
    cfg, ad, st = F.RenderCfg(), F.Adaptive(2, 32), F.Stats()
    film = (C.c_float * 4)()
    aov = F.AovFilm(None, None, None)
    s = c = g = C.c_void_p(1)  # never dereferenced: each call fails on another argument first
    calls = [
        lambda: trb.trb_render_sharded_aov(None, c, C.byref(cfg), 0, film, C.byref(aov), C.byref(st)),
        lambda: trb.trb_render_sharded_aov(s, None, C.byref(cfg), 0, film, C.byref(aov), C.byref(st)),
        lambda: trb.trb_render_sharded_aov(s, c, None, 0, film, C.byref(aov), C.byref(st)),
        lambda: trb.trb_render_sharded_adaptive_aov(s, c, C.byref(cfg), None, 0, film, C.byref(aov), None, C.byref(st)),
        lambda: trb.trb_render_sharded_adaptive_aov(None, c, C.byref(cfg), C.byref(ad), 0, film, C.byref(aov), None, C.byref(st)),
        lambda: trb.trb_group_render_aov(None, C.byref(cfg), film, C.byref(aov), C.byref(st)),
        lambda: trb.trb_group_render_aov(g, None, film, C.byref(aov), C.byref(st)),
        lambda: trb.trb_group_render_aov(g, C.byref(cfg), None, C.byref(aov), C.byref(st)),
        lambda: trb.trb_group_render_aov(g, C.byref(cfg), film, None, C.byref(st)),
        lambda: trb.trb_group_render_adaptive_aov(g, C.byref(cfg), None, film, C.byref(aov), None, C.byref(st)),
        lambda: trb.trb_group_render_adaptive_aov(g, C.byref(cfg), C.byref(ad), film, None, None, C.byref(st)),
        lambda: trb.trb_group_render_adaptive_aov(None, C.byref(cfg), C.byref(ad), film, C.byref(aov), None, C.byref(st)),
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k


# ---- the command line ----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def programs():
    H.build_programs()


def _run(args):
    m = H.Proc(args)
    try:
        return m.finish(timeout=60)
    finally:
        m.kill()


@pytest.mark.parametrize("args,needle", [
    (["--devices", "0", "--device", "0"], "--devices and --device exclude each other"),
    (["--device", "1", "--devices", "0,1"], "--devices and --device exclude each other"),
    (["--master", "localhost:1", "--devices", "0,1"], "--devices is a worker's option with --master"),
    (["--devices"], "--devices needs a comma-separated list"),
    (["--devices", ""], "--devices needs a comma-separated list"),
    (["--devices", "0,,1"], "malformed --devices list"),
    (["--devices", "0,1,"], "malformed --devices list"),
    (["--devices", "a,b"], "malformed --devices list"),
    (["--devices", "-1"], "malformed --devices list"),
    (["--devices", "0;1"], "malformed --devices list"),
    (["--devices", "0,1,0"], "--devices lists device 0 twice"),
    (["--denoise-moments", "--devices", "2,2"], "--devices lists device 2 twice"),
])
def test_tray_refuses_bad_devices_before_the_scene(programs, tmp_path, args, needle):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    rc, out, err = _run([H.TRAY, missing] + args)
    assert rc == 1 and needle in err and "no_such_scene" not in err, err
    assert "Frame" not in out


@pytest.mark.parametrize("prog", ["tray", "worker"])
@pytest.mark.parametrize("args,needle", [
    (["--devices", "0", "--device", "0"], "--devices and --device exclude each other"),
    (["--devices", "1,1"], "--devices lists device 1 twice"),
    (["--devices", "x"], "malformed --devices list"),
    (["--devices"], "--devices needs a comma-separated list"),
])
def test_worker_refuses_bad_devices_before_listening(programs, prog, args, needle):
    exe = [H.TRAY, "--worker"] if prog == "tray" else [H.WORKER]
    rc, out, err = _run(exe + ["--port", str(H.free_port())] + args)
    assert rc == 2 and needle in err, err
    assert "listening" not in out


def test_usage_names_devices(programs):
    rc, out, _ = _run([H.TRAY, "--help"])
    assert rc == 0 and "--devices LIST" in out

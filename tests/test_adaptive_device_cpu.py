"""The Adaptive sampler's stream-ordered and multi-GPU entry points without a GPU: exported, bound with the signatures
INTEGRATION.md documents for Rust callers, callable from plain C, and argument checks that need no device."""
import ctypes as C
import os
import re
import subprocess

from tray_rust_b200 import _ffi as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_render_adaptive_device", "trb_render_sharded_adaptive", "trb_group_render_adaptive"]


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
    exe = str(tmp_path / "adaptive_device_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "adaptive_device_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    out = dict(line.split() for line in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["TRB_INVALID_ARG"]) == F.TRB_INVALID_ARG
    assert {k: int(v) for k, v in out.items() if k != "TRB_INVALID_ARG"} == {n: F.TRB_INVALID_ARG for n in NEW}


def test_null_arguments_are_rejected_before_any_device_is_touched(trb):
    cfg, ad, st = F.RenderCfg(), F.Adaptive(2, 32), F.Stats()
    film = (C.c_float * 4)()
    calls = [
        lambda: trb.trb_render_adaptive_device(None, C.byref(cfg), C.byref(ad), film, None, None, None),
        lambda: trb.trb_render_adaptive_device(C.c_void_p(1), None, C.byref(ad), film, None, None, None),
        lambda: trb.trb_render_adaptive_device(C.c_void_p(1), C.byref(cfg), None, film, None, None, None),
        lambda: trb.trb_render_adaptive_device(C.c_void_p(1), C.byref(cfg), C.byref(ad), None, None, None, None),
        lambda: trb.trb_render_sharded_adaptive(None, None, C.byref(cfg), C.byref(ad), 0, film, None, C.byref(st)),
        lambda: trb.trb_render_sharded_adaptive(C.c_void_p(1), C.c_void_p(1), C.byref(cfg), None, 0, film, None, C.byref(st)),
        lambda: trb.trb_group_render_adaptive(None, C.byref(cfg), C.byref(ad), film, None, C.byref(st)),
        lambda: trb.trb_group_render_adaptive(C.c_void_p(1), C.byref(cfg), None, film, None, C.byref(st)),
    ]
    for k, call in enumerate(calls):
        assert call() == F.TRB_INVALID_ARG, k

"""The device SAH builder without a GPU: the closed form its partition computes, the C ABI and Python bindings of trb_build_bvh and
trb_build_bvh_device, and their argument checks (DESIGN.md §4 "Mesh BVH build")."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["trb_build_bvh", "trb_build_bvh_device"]


def literal_partition(pred):
    """partition.rs:9-38 as the host builder runs it: swap the first false from the front with the first true from the back."""
    a = list(range(len(pred)))
    lo, hi, split = 0, len(a), 0
    while True:
        f = bk = -1
        while lo < hi:
            p = lo
            lo += 1
            if not pred[a[p]]:
                f = p
                break
            split += 1
        while lo < hi:
            hi -= 1
            if pred[a[hi]]:
                bk = hi
                break
        if f < 0 or bk < 0:
            break
        a[f], a[bk] = a[bk], a[f]
        split += 1
    return np.array(a, np.int64), split


def closed_partition(pred):
    """The device form (k_bvh_flags, the scan, k_bvh_ranks, k_bvh_swap): ranks from exclusive prefix sums of the flags."""
    pred = np.asarray(pred, bool)
    n, P = len(pred), int(pred.sum())
    pos = np.arange(n)
    f = np.where(pos < P, ~pred, 0).astype(np.int64) + (np.where(pos >= P, pred, 0).astype(np.int64) << 32)
    pre = np.concatenate([[0], np.cumsum(f)])                # exclusive scan, one entry past the end
    d = pre[1:] - pre[:-1]
    tmp = np.zeros(n, np.int64)
    left = (pos < P) & ((d & 0xffffffff) != 0)
    tmp[(pre[:-1][left] & 0xffffffff) - (pre[0] & 0xffffffff)] = pos[left]
    right = (pos >= P) & ((d >> 32) != 0)
    tmp[P + ((pre[:-1][right] - pre[P]) >> 32)] = pos[right]
    m = int((pre[P] - pre[0]) & 0xffffffff)
    a = np.arange(n)
    k = np.arange(m)
    pl, pr = tmp[k], tmp[P + m - 1 - k]
    a[pl], a[pr] = pr, pl
    return a, P


def test_prefix_sum_partition_equals_the_two_ended_loop():
    rng = np.random.default_rng(7)
    cases = [[], [True], [False], [True] * 9, [False] * 9, [i % 2 == 0 for i in range(11)], [i % 2 == 1 for i in range(11)],
             [False] + [True] * 8, [True] * 8 + [False], [True] + [False] * 8, [False] * 8 + [True]]
    for n in range(1, 40):
        for q in (0.1, 0.5, 0.9):
            cases += [list(rng.random(n) < q) for _ in range(30)]
    cases += [list(rng.random(5000) < 0.3) for _ in range(10)]
    for pred in cases:
        a, s = literal_partition(pred)
        b, t = closed_partition(pred)
        assert s == t and np.array_equal(a, b), pred


def _c_run(tmp_path):
    exe = str(tmp_path / "bvh_build_abi")
    lib = os.path.join(REPO, "tray_rust_b200", "lib")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "bvh_build_abi.c"),
                    "-L" + lib, "-ltrb", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()


def _have_gpu():
    n = C.c_int(0)
    try:
        cudart = C.CDLL("libcudart.so")
    except OSError:
        return None
    return cudart.cudaGetDeviceCount(C.byref(n)) == 0 and n.value > 0


def test_plain_c_caller_gets_the_argument_statuses(tmp_path):
    status = {l.split()[1]: int(l.split()[2]) for l in _c_run(tmp_path) if l.startswith("status ")}
    assert status.pop("TRB_INVALID_ARG") == F.TRB_INVALID_ARG and status.pop("TRB_NO_DEVICE") == F.TRB_NO_DEVICE
    one = status.pop("trb_build_bvh:one")
    assert status == {k: F.TRB_INVALID_ARG for k in ("trb_build_bvh:null", "trb_build_bvh:empty", "trb_build_bvh_device:null",
                                                     "trb_build_bvh_device:empty")}
    assert one in (F.TRB_OK, F.TRB_NO_DEVICE)


def test_new_symbols_are_exported_and_bound_like_the_rust_declarations(trb):
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    assert F.NODE_DTYPE.itemsize == 32
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
        assert "`%s(" % name in doc or "`%s`" % name in doc, "no table row for " + name


def test_argument_checks_need_no_device(trb):
    box = np.zeros(6, np.float32)
    nn = F.u32()
    fake = C.c_void_p(1)  # never dereferenced: every call below fails its argument checks first
    assert trb.trb_build_bvh(0, None, 1, 16, C.byref(nn), None, None) == F.TRB_INVALID_ARG
    assert trb.trb_build_bvh(0, F.ptr(box), 0, 16, C.byref(nn), None, None) == F.TRB_INVALID_ARG
    assert trb.trb_build_bvh(0, F.ptr(box), 1, 16, None, None, None) == F.TRB_INVALID_ARG
    assert trb.trb_build_bvh(0, fake, 1 << 31, 16, C.byref(nn), None, None) == F.TRB_UNSUPPORTED
    assert trb.trb_build_bvh_device(0, fake, 0, 16, fake, fake, fake, None) == F.TRB_INVALID_ARG
    for k in range(4):
        args = [fake] * 4
        args[k] = None
        assert trb.trb_build_bvh_device(0, args[0], 4, 16, args[1], args[2], args[3], None) == F.TRB_INVALID_ARG, k
    assert trb.trb_build_bvh_device(0, fake, 0xffffffff, 16, fake, fake, fake, None) == F.TRB_UNSUPPORTED


def test_without_a_gpu_the_build_is_no_device(trb):
    if _have_gpu() is not False:
        pytest.skip("a GPU is present, or the CUDA runtime could not be asked")
    boxes = np.array([[0, 0, 0, 1, 1, 1], [2, 0, 0, 3, 1, 1]], np.float32)
    nn = F.u32()
    assert trb.trb_build_bvh(0, F.ptr(boxes), 2, 16, C.byref(nn), None, None) == F.TRB_NO_DEVICE
    assert trb.trb_build_bvh_device(0, C.c_void_p(1), 2, 16, C.c_void_p(1), C.c_void_p(1), C.c_void_p(1), None) == F.TRB_NO_DEVICE
    with pytest.raises(api.TrbError) as e:
        api.build_bvh(boxes, 16)
    assert e.value.status == F.TRB_NO_DEVICE

"""The Adaptive sampler (sampler/adaptive.rs) without a GPU: schedule rounding, the shared per-pixel decision against a
literal float32 transcription of needs_supersampling / report_results, and the oracle's literal thread_work."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F
from tray_rust_b200 import scenebuild as SB
from oracle_adaptive.pyadaptive import AdaptiveOracleScene

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def literal_decide(min_in, max_in, lum):
    """adaptive.rs:54-78,82-101,127-141 in numpy float32: returns (samples_taken, avg_luminance)."""
    mn, mx = pow2(min_in), pow2(max_in)
    step = pow2((mx - mn) // 5)
    taken, avg, samples = 0, f32(0.0), []
    with np.errstate(all="ignore"):
        while True:
            n = mn if taken == 0 else step
            taken += n
            assert len(lum) >= len(samples) + n, "sequence too short"
            samples.extend(f32(x) for x in lum[len(samples):len(samples) + n])
            if taken >= mx:
                return taken, avg
            if taken == mn:
                ac = f32(0.0)
                for s in samples:
                    ac = f32(ac + s)
                avg = f32(ac / f32(len(samples)))
            else:
                for i in range(len(samples) - step, len(samples)):
                    avg = f32(f32(samples[i] + f32(f32(i - 1) * avg)) / f32(i))
            if not any(f32(abs(f32(s - avg)) / avg) > f32(0.5) for s in samples):
                return taken, avg


def luminance(r, g, b):
    r, g, b = f32(r), f32(g), f32(b)
    return f32(f32(f32(f32(0.2126) * r) + f32(f32(0.7152) * g)) + f32(f32(0.0722) * b))


def host_decide(trb, min_spp, max_spp, lum):
    lum = np.ascontiguousarray(lum, np.float32)
    taken, avg = F.u32(), F.f32()
    rc = trb.trb_host_adaptive_decide(C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(lum), len(lum), C.byref(taken), C.byref(avg))
    assert rc == F.TRB_OK, trb.trb_last_error()
    return taken.value, avg.value


def schedule(trb, min_spp, max_spp):
    out = [F.u32() for _ in range(4)]
    rc = trb.trb_adaptive_schedule(C.byref(F.Adaptive(min_spp, max_spp)), *(C.byref(x) for x in out))
    return rc, tuple(x.value for x in out)


def test_schedule_rounding(trb, oracle):
    cases = {(3, 100): (4, 128, 32, 132), (4, 64): (4, 64, 16, 68), (4, 4): (4, 4, 1, 4), (0, 8): (1, 8, 1, 8), (16, 16): (16, 16, 1, 16)}
    o = AdaptiveOracleScene(SB.scene_materials_zoo(8, 8, 1).finish())
    for (mn, mx), want in cases.items():
        rc, got = schedule(trb, mn, mx)
        assert rc == F.TRB_OK and got == want, ((mn, mx), got)
        assert o.adaptive_schedule(mn, mx) == want
    rc, _ = schedule(trb, 8, 4)
    assert rc == F.TRB_INVALID_ARG
    with pytest.raises(Exception):
        o.adaptive_schedule(8, 4)
    # (4, 4): one round of 4 samples whatever the samples say
    assert host_decide(trb, 4, 4, [0.0, 1.0, 0.0, 1.0])[0] == 4


def _crafted():
    rng = np.random.default_rng(7)
    seqs = [
        np.zeros(200),                                    # all black: avg 0 -> 0/0 = NaN -> stop at min
        np.r_[np.zeros(3), 0.5, np.zeros(196)],           # one non-black sample after zeros: inf -> go on
        np.r_[0.3, np.nan, 0.3, 0.3, np.full(196, 0.3)],  # NaN luminance: NaN average, every compare false
        np.r_[1.0, 1.0, 1.0, 3.0, np.full(196, 1.5)],     # avg 1.5: |3 - 1.5| / 1.5 = 1 > 0.5 ...
        np.r_[2.0, 2.0, 1.0, 3.0, np.full(196, 2.0)],     # ... |1 - 2| / 2 = 0.5 exactly: not > 0.5, stop
        np.full(200, 0.25),
        rng.uniform(0.0, 1.0, 200),                       # long CMA chains
        rng.uniform(0.45, 0.55, 200),
        np.where(rng.uniform(size=200) < 0.05, 1.0, 0.01),
        np.r_[np.full(4, 0.2), 0.2, 0.2, 0.31, np.full(193, 0.2)],
    ]
    return [np.asarray(s, np.float32) for s in seqs]


@pytest.mark.parametrize("mn,mx", [(4, 64), (1, 8), (2, 16), (4, 4), (3, 100), (8, 32), (1, 2)])
def test_host_decide_matches_literal_transcription(trb, mn, mx):
    for k, seq in enumerate(_crafted()):
        mpp = schedule(trb, mn, mx)[1][3]
        seq = np.resize(seq, max(len(seq), mpp)).astype(np.float32)
        want_taken, want_avg = literal_decide(mn, mx, seq)
        taken, avg = host_decide(trb, mn, mx, seq)
        assert taken == want_taken, (k, mn, mx, taken, want_taken)
        if taken < pow2(mx):  # the reference stops before updating the average once samples_taken >= max_spp
            assert np.float32(avg).tobytes() == want_avg.tobytes(), (k, avg, want_avg)
    # pinned answers of the crafted cases (4, 64)
    seqs = _crafted()
    assert host_decide(trb, 4, 64, seqs[0])[0] == 4
    assert host_decide(trb, 4, 64, seqs[1])[0] == 68
    assert host_decide(trb, 4, 64, seqs[2])[0] == 4
    assert host_decide(trb, 4, 64, seqs[4])[0] == 4
    assert host_decide(trb, 4, 64, seqs[3])[0] > 4


def test_host_decide_rejects_short_sequence(trb):
    lum = np.r_[np.zeros(3), 1.0].astype(np.float32)
    taken, avg = F.u32(), F.f32()
    assert trb.trb_host_adaptive_decide(C.byref(F.Adaptive(4, 64)), F.ptr(lum), 4, C.byref(taken), C.byref(avg)) == F.TRB_INVALID_ARG


def _per_pixel(samples, spp, blocks, width, mpp):
    """(pixel index, its records in slot order) for every pixel of the dump."""
    rec = samples.reshape(len(blocks), 64, mpp)
    for b, (bx, by) in enumerate(blocks):
        for k in range(64):
            px, py = bx * 8 + k % 8, by * 8 + k // 8
            yield py * width + px, rec[b, k]


def test_oracle_counts_follow_the_literal_decision(oracle):
    o = AdaptiveOracleScene(SB.scene_materials_zoo(32, 32, 1, SB.synthetic_merl_table()).finish())
    o.update_frame(0, 0.0, 0.0)
    mn, mx = 2, 16
    mpp = o.adaptive_schedule(mn, mx)[3]
    out, spp, st = o.render_samples_adaptive(mn, mx, seed=3)
    blocks = o.block_list()
    flat = spp.reshape(-1)
    assert st.camera_samples == int(flat.sum())
    refined = 0
    for pixel, rec in _per_pixel(out, spp, blocks, o.width, mpp):
        n = int(flat[pixel])
        lum = [luminance(r["r"], r["g"], r["b"]) for r in rec[:n]]
        assert literal_decide(mn, mx, lum + [0.0] * (mpp - n))[0] == n
        assert not rec[n:].tobytes().strip(b"\0"), "unused slots must be zero"
        refined += n > pow2(mn)
    assert refined > 0 and refined < len(flat)


def test_all_miss_pixel_keeps_min_samples(oracle):
    desc = SB.scene_c4(2000, 64, 32, 1).finish()  # the frame shows the space around the Cornell box
    o = AdaptiveOracleScene(desc)
    o.update_frame(0, 0.0, 0.0)
    mpp = o.adaptive_schedule(4, 64)[3]
    out, spp, _ = o.render_samples_adaptive(4, 64, seed=11)
    black = 0
    for pixel, rec in _per_pixel(out, spp, o.block_list(), o.width, mpp):
        n = int(spp.reshape(-1)[pixel])
        if ((rec["r"][:n] == 0) & (rec["g"][:n] == 0) & (rec["b"][:n] == 0)).all():
            assert n == 4, "a pixel whose samples are all black stops at min_spp"
            black += 1
    assert black > 0, "the scene should have pixels that see nothing"


def test_min_equals_max_converges_to_low_discrepancy(oracle):
    o = AdaptiveOracleScene(SB.scene_materials_zoo(32, 32, 16, SB.synthetic_merl_table()).finish())
    fa, spp, st = o.render_adaptive(16, 16, seed=21)
    assert (spp == 16).all() and st.camera_samples == 32 * 32 * 16
    fb, _ = o.render(seed=22)
    ia = fa[..., :3] / fa[..., 3:]
    ib = fb[..., :3] / fb[..., 3:]
    d = (ia - ib).reshape(-1, 3)
    se = d.std(axis=0) / np.sqrt(len(d))
    assert (np.abs(d.mean(axis=0)) < 3 * se + 1e-7).all(), (d.mean(axis=0), se)
    assert np.abs(ia.mean() - ib.mean()) < 0.05 * ib.mean()


def test_adaptive_abi_layout(tmp_path):
    exe = str(tmp_path / "adaptive_abi")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-I" + os.path.join(REPO, "include"), os.path.join(REPO, "tests", "c", "adaptive_abi.c"),
                    "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["trb_adaptive", str(C.sizeof(F.Adaptive)), str(F.Adaptive.min_spp.offset), str(F.Adaptive.max_spp.offset)]
    assert C.sizeof(F.Adaptive) == 8


def test_integration_doc_declares_the_adaptive_struct():
    import re
    doc = open(os.path.join(REPO, "INTEGRATION.md")).read()
    m = re.search(r"pub struct TrbAdaptive \{(.*?)\}", doc, re.S)
    assert m
    fields = [f.split(":")[0].strip() for f in m.group(1).split(",") if f.strip()]
    assert fields == [f for f, _ in F.Adaptive._fields_]
    assert "fn trb_render_adaptive(" in doc

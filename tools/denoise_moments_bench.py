"""Time the moment denoiser and measure what it buys. The GPU's name and power limit are read in the same call; prints one JSON line.
  - time per call: trb_denoise_moments_device on a 1-spp AOV render of C4 at 1920 x 1080 against trb_denoise_temporal_device on the
    halves of a 2-spp one, CUDA events on one stream, median of --reps after a warm-up (each history holds the previous call's frame);
  - kernel split: k_dn_temporal_moments, k_dn_moments_variance and k_dn_atrous under torch.profiler, in a run of its own;
  - frame time: a 1-spp frame rendered by render_aov_device and denoised by trb_denoise_moments_device, against a 2-spp frame rendered
    as two 1-spp AOV halves and denoised by trb_denoise_temporal_device, device buffers, one stream, median of --reps;
  - quality over --frames frames, frame k rendered with seed 1 + k: per-frame RMSE (colours clamped to [0, 1]) against a --ref-spp
    render of the same frame, moments at 1 spp against max_history 1 (the single-frame filter of the same film) and the noisy 1-spp
    film, beside the half-film temporal call at 2 spp; on C4 with a static camera and with the keyframed camera orbit (update_keyframes
    before every frame); and the flicker, the mean |out_k - out_{k-1}| over the static sequence.

    python tools/denoise_moments_bench.py [--tris 1000000] [--reps 10] [--frames 16] [--ref-spp 256] [--width 1920 --height 1080]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def rmse(film, ref):
    c = np.clip(film[..., :3] / np.maximum(film[..., 3:], 1e-12), 0, 1)
    r = np.clip(ref[..., :3] / ref[..., 3:], 0, 1)
    return float(np.sqrt(((c - r) ** 2).mean()))


def halves(g, seed):
    a, aovs, _ = g.render_aov(spp=2, sample_first=0, sample_count=1, seed=seed, flags=F.RENDER_NO_UPDATE)
    b, _, _ = g.render_aov(albedo=aovs["albedo_w"], normal=aovs["normal_w"], nearest=aovs["nearest"], spp=2, sample_first=1, sample_count=1,
                           seed=seed, flags=F.RENDER_NO_UPDATE)
    return a, b, aovs


def timing(args, out):
    import torch
    s = api.Scene(SB.scene_c4(args.tris, 1920, 1080, 2).finish())
    s.update_frame(0, 0.0, 0.0)
    h, w = s.height, s.width
    a, b, aovs = halves(s, 1)
    film, aovs1, _ = s.render_aov(spp=1, seed=1, flags=F.RENDER_NO_UPDATE)
    t2 = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
    t1 = [torch.from_numpy(x).cuda() for x in (film, aovs1["albedo_w"], aovs1["normal_w"], aovs1["nearest"].view(np.int64))]
    p2, p1 = [x.data_ptr() for x in t2], [x.data_ptr() for x in t1]
    den = torch.zeros_like(t1[0])
    h_t, h_m = api.DenoiseHistory(s), api.DenoiseHistory(s)
    st = torch.cuda.Stream()

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            f()
            e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    calls = dict(moments=lambda: s.denoise_moments_device(h_m, *p1, den.data_ptr(), stream=st.cuda_stream),
                 temporal=lambda: s.denoise_temporal_device(h_t, *p2, den.data_ptr(), stream=st.cuda_stream))
    # whole frames on device buffers: the render (AOVs reset first, as render_aov does) and the denoise
    fa, fb, alb, nrm = (torch.zeros((h, w, 4), device="cuda") for _ in range(4))
    near = torch.full((h, w), -1, dtype=torch.int64, device="cuda")

    def reset():
        for x in (fa, fb, alb, nrm):
            x.zero_()
        near.fill_(-1)

    def frame_moments():
        reset()
        s.render_aov_device(fa.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), stream=st.cuda_stream, spp=1, seed=1,
                            flags=F.RENDER_NO_UPDATE)
        s.denoise_moments_device(h_m, fa.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), den.data_ptr(), stream=st.cuda_stream)

    def frame_temporal():
        reset()
        for f, first in ((fa, 0), (fb, 1)):
            s.render_aov_device(f.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), stream=st.cuda_stream, spp=2,
                                sample_first=first, sample_count=1, seed=1, flags=F.RENDER_NO_UPDATE)
        s.denoise_temporal_device(h_t, fa.data_ptr(), fb.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), den.data_ptr(),
                                  stream=st.cuda_stream)

    def render_1spp():
        reset()
        s.render_aov_device(fa.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), stream=st.cuda_stream, spp=1, seed=1,
                            flags=F.RENDER_NO_UPDATE)

    frames = dict(moments_1spp=frame_moments, temporal_2spp=frame_temporal, render_aov_1spp=render_1spp)
    for f in list(calls.values()) + list(frames.values()):
        for _ in range(3):
            timed(f)
    out["ms_per_call_1080p"] = {k: round(statistics.median(timed(f) for _ in range(args.reps)), 3) for k, f in calls.items()}
    out["ms_per_frame_1080p"] = {k: round(statistics.median(timed(f) for _ in range(args.reps)), 3) for k, f in frames.items()}
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            with torch.cuda.stream(st):
                calls["moments"]()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in ("k_dn_temporal_moments", "k_dn_moments_variance", "k_dn_atrous"):
            if k in e.key:
                per[k] = dict(calls=e.count, mean_ms=round(e.device_time_total / max(e.count, 1) / 1000.0, 4))
    out["kernels"] = per
    h_t.close()
    h_m.close()
    s.close()


def quality(name, g, frames, ref_spp, set_frame, out):
    hm, hs, ht = api.DenoiseHistory(g), api.DenoiseHistory(g), api.DenoiseHistory(g)
    rows, prev, flick = [], None, dict(moments=[], single=[], temporal=[])
    for k in range(frames):
        set_frame(k)
        ref, _ = g.render(spp=ref_spp, seed=1000 + k, flags=F.RENDER_NO_UPDATE)
        film, aovs, _ = g.render_aov(spp=1, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        a, b, aovs2 = halves(g, 1 + k)
        cur = dict(moments=g.denoise_moments(hm, film, aovs), single=g.denoise_moments(hs, film, aovs, max_history=1),
                   temporal=g.denoise_temporal(ht, a, b, aovs2))
        rows.append(dict(frame=k, noisy_1spp=round(rmse(film, ref), 5), **{c: round(rmse(x, ref), 5) for c, x in cur.items()}))
        if prev is not None:
            for c in cur:
                flick[c].append(float(np.abs(cur[c][..., :3] - prev[c][..., :3]).mean()))
        prev = cur
    cols = ["noisy_1spp", "moments", "single", "temporal"]
    out[name] = dict(per_frame=rows, mean_after_first={c: round(statistics.mean(r[c] for r in rows[1:]), 5) for c in cols},
                     last={c: rows[-1][c] for c in cols}, flicker={c: round(statistics.mean(v), 6) for c, v in flick.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    out = dict(gpu=gpu_info())
    timing(args, out)
    if not args.skip_quality:
        b = SB.scene_c4(args.tris, args.width, args.height, 2)
        g = api.Scene(b.finish())
        g.update_frame(0, 0.0, 0.0)
        quality("c4_static", g, args.frames, args.ref_spp, lambda k: None, out)
        cam = len(b.keyframes) - 1
        t0, q0, s0 = b.keyframes[cam]

        def orbit(k):
            ang = 0.01 * k  # radians per frame
            x, z = t0[0], t0[2]
            t = (x * math.cos(ang) - z * math.sin(ang), t0[1], x * math.sin(ang) + z * math.cos(ang))
            g.update_keyframes(cam, np.array([(t, q0, s0)], F.KEYFRAME_DTYPE))
            g.update_frame(0, 0.0, 0.0)
        quality("c4_orbit", g, args.frames, args.ref_spp, orbit, out)
        g.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

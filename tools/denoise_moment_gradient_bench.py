"""Time the moment gradients and measure what they buy. The GPU's name and power limit are read in the same call; prints one JSON line.
  - time per call: trb_denoise_moments_gradient_device against trb_denoise_moments_device on a 1-spp AOV render of C4 at 1920 x 1080,
    CUDA events on one stream, the two alternated, median of --reps after a warm-up (each history holds the previous call's frame);
  - kernel split of the moment gradient call under torch.profiler, in a run of its own;
  - frame time: a 1-spp frame rendered by render_aov_device and denoised by the moment gradient call, against the same frame denoised
    by the plain moment call and a 2-spp frame rendered as two 1-spp AOV halves and denoised by trb_denoise_temporal_gradient_device;
  - quality over --frames frames, frame k rendered with seed 1 + k: per-frame RMSE (colours clamped to [0, 1]) against a --ref-spp
    render of the same frame, moment gradients at 1 spp against plain moments, max_history 1 and the half-film gradient call at 2 spp;
    on the keyframed scene, on a C4 camera orbit, and on a static C4 with the flicker, the mean |out_k - out_{k-1}|.

    python tools/denoise_moment_gradient_bench.py [--tris 1000000] [--reps 10] [--frames 8] [--ref-spp 128] [--width 1024 --height 576]
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402
from denoise_moments_bench import gpu_info, halves, rmse  # noqa: E402


def timing(args, out):
    import torch
    s = api.Scene(SB.scene_c4(args.tris, 1920, 1080, 2).finish())
    s.update_frame(0, 0.0, 0.0)
    h, w = s.height, s.width
    film, aovs, _ = s.render_aov(spp=1, seed=1, flags=F.RENDER_NO_UPDATE)
    t1 = [torch.from_numpy(x).cuda() for x in (film, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
    p1 = [x.data_ptr() for x in t1]
    den = torch.zeros_like(t1[0])
    h_g, h_m, h_t = api.DenoiseHistory(s), api.DenoiseHistory(s), api.DenoiseHistory(s)
    st = torch.cuda.Stream()

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            f()
            e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    seed = [1]

    def moment_gradient():
        seed[0] += 1
        s.denoise_moments_gradient_device(h_g, *p1, seed[0], den.data_ptr(), stream=st.cuda_stream)

    calls = dict(moment_gradient=moment_gradient, moments=lambda: s.denoise_moments_device(h_m, *p1, den.data_ptr(), stream=st.cuda_stream))
    fa, fb, alb, nrm = (torch.zeros((h, w, 4), device="cuda") for _ in range(4))
    near = torch.full((h, w), -1, dtype=torch.int64, device="cuda")

    def render(f, spp, first, count):
        s.render_aov_device(f.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), stream=st.cuda_stream, spp=spp,
                            sample_first=first, sample_count=count, seed=1, flags=F.RENDER_NO_UPDATE)

    def reset():
        for x in (fa, fb, alb, nrm):
            x.zero_()
        near.fill_(-1)

    def frame_moment_gradient():
        reset()
        render(fa, 1, 0, 1)
        seed[0] += 1
        s.denoise_moments_gradient_device(h_g, fa.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), seed[0], den.data_ptr(),
                                          stream=st.cuda_stream)

    def frame_moments():
        reset()
        render(fa, 1, 0, 1)
        s.denoise_moments_device(h_m, fa.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), den.data_ptr(), stream=st.cuda_stream)

    def frame_temporal_gradient():
        reset()
        render(fa, 2, 0, 1)
        render(fb, 2, 1, 1)
        seed[0] += 1
        s.denoise_temporal_gradient_device(h_t, fa.data_ptr(), fb.data_ptr(), alb.data_ptr(), nrm.data_ptr(), near.data_ptr(), seed[0],
                                           den.data_ptr(), stream=st.cuda_stream)

    frames = dict(moment_gradient_1spp=frame_moment_gradient, moments_1spp=frame_moments, temporal_gradient_2spp=frame_temporal_gradient)
    for group, key in ((calls, "ms_per_call_1080p"), (frames, "ms_per_frame_1080p")):
        for f in group.values():
            for _ in range(3):
                timed(f)
        got = {k: [] for k in group}
        for _ in range(args.reps):  # alternated
            for k, f in group.items():
                got[k].append(timed(f))
        out[key] = {k: round(statistics.median(v), 3) for k, v in got.items()}
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            with torch.cuda.stream(st):
                moment_gradient()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            per[e.key[:60]] = dict(calls=e.count, ms_per_call=round(e.device_time_total / args.reps / 1000.0, 4))
    out["kernels_per_moment_gradient_call"] = dict(sorted(per.items(), key=lambda kv: -kv[1]["ms_per_call"])[:16])
    for x in (h_g, h_m, h_t):
        x.close()
    s.close()


def quality(name, g, frames, ref_spp, set_frame, out):
    hg, hm, hs, ht = (api.DenoiseHistory(g) for _ in range(4))
    rows, prev, flick = [], None, dict(moment_gradient=[], moments=[], single=[], temporal_gradient=[])
    for k in range(frames):
        set_frame(k)
        ref, _ = g.render(spp=ref_spp, seed=1000 + k, flags=F.RENDER_NO_UPDATE)
        film, aovs, _ = g.render_aov(spp=1, seed=1 + k, flags=F.RENDER_NO_UPDATE)
        a, b, aovs2 = halves(g, 1 + k)
        cur = dict(moment_gradient=g.denoise_moments_gradient(hg, film, aovs, 1 + k), moments=g.denoise_moments(hm, film, aovs),
                   single=g.denoise_moments(hs, film, aovs, max_history=1), temporal_gradient=g.denoise_temporal_gradient(ht, a, b, aovs2, 1 + k))
        rows.append(dict(frame=k, **{c: round(rmse(x, ref), 5) for c, x in cur.items()}))
        if prev is not None:
            for c in cur:
                flick[c].append(float(np.abs(cur[c][..., :3] - prev[c][..., :3]).mean()))
        prev = cur
    cols = list(flick)
    out[name] = dict(per_frame=rows, mean_after_first={c: round(statistics.mean(r[c] for r in rows[1:]), 5) for c in cols},
                     flicker={c: round(statistics.mean(v), 6) for c, v in flick.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--ref-spp", type=int, default=128)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--height", type=int, default=576)
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    out = dict(gpu=gpu_info())
    timing(args, out)
    if not args.skip_quality:
        g = api.Scene(SB.scene_animated(args.width, args.height, 1).finish())
        quality("scene_animated", g, args.frames, args.ref_spp, lambda k: g.update_frame(k, 0.25 * k, 0.25 * (k + 1)), out)
        g.close()
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

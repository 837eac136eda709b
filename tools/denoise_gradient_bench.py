"""Time the temporal gradients and measure what they buy. The GPU's name and power limit are read in the same call; prints one JSON line.
  - time per call: trb_denoise_temporal_gradient_device against trb_denoise_temporal_device on the halves of a 2-spp AOV render of C4
    at 1920 x 1080, alternating, CUDA events on one stream, median of --reps after a warm-up (each history holds the previous call's
    frame, so every gradient call re-shades the records of the one before);
  - kernel split: the gradient kernels, the ray queries and illumination passes they launch, and k_dn_temporal_grad, under
    torch.profiler in a run of its own;
  - quality over --frames frames at 2 spp, each frame rendered with seed 1 + frame: per-frame RMSE (colours clamped to [0, 1]) against
    a --ref-spp render of the same frame and the flicker (mean |out_k - out_{k-1}|), spatial, plain temporal and gradient temporal at
    gradient_iterations 1, 3 and 5, on scenebuild.scene_animated, C4 with a keyframed camera orbit, and frames of c5_tr15_like (colour
    keyed emitters), at --width x --height.

    python tools/denoise_gradient_bench.py [--tris 1000000] [--reps 5] [--frames 16] [--ref-spp 256] [--width 1920 --height 1080]
                                           [--skip-quality]
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
from denoise_temporal_bench import gpu_info, halves, rmse  # noqa: E402

ITERATIONS = (1, 3, 5)


def timing(args, out):
    import torch
    s = api.Scene(SB.scene_c4(args.tris, 1920, 1080, 2).finish())
    s.update_frame(0, 0.0, 0.0)
    a, b, aovs = halves(s, 1)
    t = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
    ptrs = [x.data_ptr() for x in t]
    den = torch.zeros_like(t[0])
    hp, hg = api.DenoiseHistory(s), api.DenoiseHistory(s)
    st = torch.cuda.Stream()

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            f()
            e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    calls = dict(temporal=lambda: s.denoise_temporal_device(hp, *ptrs, den.data_ptr(), stream=st.cuda_stream),
                 gradient=lambda: s.denoise_temporal_gradient_device(hg, *ptrs, 1, den.data_ptr(), stream=st.cuda_stream))
    for f in calls.values():
        for _ in range(3):
            timed(f)
    times = {k: [] for k in calls}
    for _ in range(args.reps):  # alternating
        for k, f in calls.items():
            times[k].append(timed(f))
    out["ms_per_call_1080p"] = {k: round(statistics.median(v), 3) for k, v in times.items()}
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            with torch.cuda.stream(st):
                calls["gradient"]()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            per[e.key[:60]] = dict(calls=e.count, ms_per_call=round(e.device_time_total / args.reps / 1000.0, 4))
    out["kernels_per_gradient_call"] = dict(sorted(per.items(), key=lambda kv: -kv[1]["ms_per_call"])[:16])
    hp.close()
    hg.close()
    s.close()


def quality(name, g, frames, ref_spp, set_frame, out):
    hp = api.DenoiseHistory(g)
    hg = {it: api.DenoiseHistory(g) for it in ITERATIONS}
    rows, prev, flick = [], None, {}
    for k in range(frames):
        set_frame(k)
        ref, _ = g.render(spp=ref_spp, seed=1000 + k, flags=F.RENDER_NO_UPDATE)
        a, b, aovs = halves(g, 1 + k)
        cur = dict(spatial=g.denoise(a, b, aovs), temporal=g.denoise_temporal(hp, a, b, aovs))
        for it, h in hg.items():
            cur["g%d" % it] = g.denoise_temporal_gradient(h, a, b, aovs, 1 + k, gradient_iterations=it)
        rows.append(dict(frame=k, **{c: round(rmse(v, ref), 5) for c, v in cur.items()}))
        if prev is not None:
            for c in cur:
                flick.setdefault(c, []).append(float(np.abs(cur[c][..., :3] - prev[c][..., :3]).mean()))
        prev = cur
    cols = list(cur)
    out[name] = dict(per_frame=rows, mean_rmse_after_first={c: round(statistics.mean(r[c] for r in rows[1:]), 5) for c in cols},
                     flicker={c: round(statistics.mean(v), 6) for c, v in flick.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--c5-first", type=int, default=6)
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    out = dict(gpu=gpu_info())
    timing(args, out)
    if not args.skip_quality:
        a = api.Scene(SB.scene_animated(args.width, args.height, 2, frames=args.frames).finish())
        quality("scene_animated", a, args.frames, args.ref_spp, lambda k: a.update_frame(k, k / args.frames, (k + 1) / args.frames), out)
        a.close()
        b = SB.scene_c4(args.tris, args.width, args.height, 2)
        g = api.Scene(b.finish())
        cam = len(b.keyframes) - 1
        t0, q0, s0 = b.keyframes[cam]

        def orbit(k):
            ang = 0.01 * k
            x, z = t0[0], t0[2]
            t = (x * math.cos(ang) - z * math.sin(ang), t0[1], x * math.sin(ang) + z * math.cos(ang))
            g.update_keyframes(cam, np.array([(t, q0, s0)], F.KEYFRAME_DTYPE))
            g.update_frame(0, 0.0, 0.0)
        quality("c4_orbit", g, args.frames, args.ref_spp, orbit, out)
        g.close()
        sys.path.insert(0, os.path.join(REPO, "tests"))
        import cli_helpers as H
        sys.path.insert(0, os.path.join(REPO, "tests", "golden"))
        import make_scenes
        merl = os.path.join(H.SCENES, "merl", "synthetic.binary")
        if not os.path.exists(merl):
            make_scenes.write_synthetic_merl(merl)
        c = api.Scene(H.load_desc(H.C5, args.width, args.height, 2).contents)
        first, step = args.c5_first, 0.5  # 50 frames over a scene_time of 25; the emitters' colour keys change from t = 3.5 to 7
        quality("c5_tr15_like", c, args.frames, args.ref_spp, lambda k: c.update_frame(first + k, (first + k) * step, (first + k + 1) * step), out)
        c.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Time the temporal denoiser and measure what it buys. The GPU's name and power limit are read in the same call; prints one JSON line.
  - time per call: trb_denoise_temporal_device against trb_denoise_device on the halves of a 2-spp AOV render of C4 at 1920 x 1080,
    CUDA events on one stream, median of --reps after a warm-up (the temporal history holds the previous call's frame);
  - kernel split: k_dn_temporal against k_dn_prepare (and the a-trous iterations), under torch.profiler in a run of its own;
  - quality over --frames frames at 2 spp, each frame rendered with seed 1 + frame: per-frame RMSE (colours clamped to [0, 1]) against
    a --ref-spp render of the same frame, temporal at max_history 1, 4, 8 and 16 against spatial, on C4 with a keyframed camera orbit
    (update_keyframes before every frame) and on scenebuild.scene_animated, both at --width x --height; and the flicker, the mean
    |out_k - out_{k-1}| over a static-camera C4 sequence.

    python tools/denoise_temporal_bench.py [--tris 1000000] [--reps 5] [--frames 16] [--ref-spp 256] [--width 1920 --height 1080]
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

HISTORIES = (1, 4, 8, 16)


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
    a, b, aovs = halves(s, 1)
    t = [torch.from_numpy(x).cuda() for x in (a, b, aovs["albedo_w"], aovs["normal_w"], aovs["nearest"].view(np.int64))]
    ptrs = [x.data_ptr() for x in t]
    den = torch.zeros_like(t[0])
    motion = torch.zeros((s.height, s.width, 2), dtype=torch.float32, device="cuda")
    hl = torch.zeros((s.height, s.width), dtype=torch.int32, device="cuda")
    hist = api.DenoiseHistory(s)
    st = torch.cuda.Stream()

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            f()
            e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    calls = dict(spatial=lambda: s.denoise_device(*ptrs, den.data_ptr(), stream=st.cuda_stream),
                 temporal=lambda: s.denoise_temporal_device(hist, *ptrs, den.data_ptr(), stream=st.cuda_stream),
                 temporal_motion=lambda: s.denoise_temporal_device(hist, *ptrs, den.data_ptr(), motion.data_ptr(), hl.data_ptr(), stream=st.cuda_stream))
    for f in calls.values():
        for _ in range(3):
            timed(f)
    out["ms_per_call_1080p"] = {k: round(statistics.median(timed(f) for _ in range(args.reps)), 3) for k, f in calls.items()}
    # kernel split, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f in (calls["spatial"], calls["temporal"]):
            for _ in range(args.reps):
                with torch.cuda.stream(st):
                    f()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for k in ("k_dn_prepare", "k_dn_temporal", "k_dn_atrous"):
            if k in e.key:
                per[k] = dict(calls=e.count, mean_ms=round(e.device_time_total / max(e.count, 1) / 1000.0, 4))
    out["kernels"] = per
    hist.close()
    s.close()


def quality(name, g, frames, ref_spp, set_frame, out):
    hists = {m: api.DenoiseHistory(g) for m in HISTORIES}
    rows = []
    for k in range(frames):
        set_frame(k)
        ref, _ = g.render(spp=ref_spp, seed=1000 + k, flags=F.RENDER_NO_UPDATE)
        a, b, aovs = halves(g, 1 + k)
        row = dict(frame=k, spatial=round(rmse(g.denoise(a, b, aovs), ref), 5), noisy=round(rmse(a + b, ref), 5))
        for m, hst in hists.items():
            row["t%d" % m] = round(rmse(g.denoise_temporal(hst, a, b, aovs, max_history=m), ref), 5)
        rows.append(row)
    out[name] = dict(per_frame=rows, mean_after_first={c: round(statistics.mean(r[c] for r in rows[1:]), 5)
                                                       for c in ["noisy", "spatial"] + ["t%d" % m for m in HISTORIES]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--skip-quality", action="store_true")
    args = ap.parse_args()
    out = dict(gpu=gpu_info())
    timing(args, out)
    if not args.skip_quality:
        # C4 with a keyframed camera orbit: the camera's keyframe moved along a circle about the scene before every frame
        b = SB.scene_c4(args.tris, args.width, args.height, 2)
        g = api.Scene(b.finish())
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
        a = api.Scene(SB.scene_animated(args.width, args.height, 2, frames=args.frames).finish())
        quality("scene_animated", a, args.frames, args.ref_spp, lambda k: a.update_frame(k, k / args.frames, (k + 1) / args.frames), out)
        a.close()
        # flicker on a static camera
        g = api.Scene(SB.scene_c4(args.tris, args.width, args.height, 2).finish())
        g.update_frame(0, 0.0, 0.0)
        hst = api.DenoiseHistory(g)
        prev, flick = None, dict(spatial=[], temporal=[])
        for k in range(args.frames):
            a_, b_, aovs = halves(g, 1 + k)
            cur = dict(spatial=g.denoise(a_, b_, aovs), temporal=g.denoise_temporal(hst, a_, b_, aovs))
            if prev is not None:
                for c in cur:
                    flick[c].append(float(np.abs(cur[c][..., :3] - prev[c][..., :3]).mean()))
            prev = cur
        out["flicker_c4_static"] = {c: round(statistics.mean(v), 6) for c, v in flick.items()}
        g.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

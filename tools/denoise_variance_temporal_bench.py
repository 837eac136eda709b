"""The variance temporal denoiser on C4 at 1920x1080: what trb_denoise_variance_temporal costs against trb_denoise_variance and
trb_denoise_moments, and what carrying the sample variance through the history buys against the moment call, the half-film temporal
call, the single-frame variance call and the noisy film. Measures and reports; gates nothing.

    python tools/denoise_variance_temporal_bench.py [--reps 7] [--ref-spp 256] [--frames 16] [--out results/denoise_variance_temporal_bench.json]

1. Time per call on the 2-spp films of one render (device forms, default parameters, one torch stream, CUDA events, median of
   --reps after a warm-up, the three calls alternated): trb_denoise_variance_temporal_device (a warm history), trb_denoise_variance_device
   and trb_denoise_moments_device. Then one call of each under torch.profiler (its own run): the time of each kernel. And the
   whole frame: render_aov_device with the lum_w film plus the variance temporal call.
2. Quality over --frames frames (seed 1 + k): RMSE of colours clamped to [0, 1] against a --ref-spp render of the same frame, mean
   over frames 1 .. frames-1, and flicker, the mean over those frames of mean |out_k - out_(k-1)|. Methods: "vt" (this call, one
   render), "moments" (trb_denoise_moments on the same render; Adaptive: render_denoised_adaptive's call), "halves"
   (trb_denoise_temporal on two half renders, LowDiscrepancy only), "variance1" (trb_denoise_variance, single frame), "noisy" (the
   film); on scene_animated also "vt_grad", "moments_grad" and "halves_grad", the gradient forms. Cases: C4 at 2 and 4 spp with a
   static camera and on a camera arc set with update_keyframes; C4 Adaptive (2, 32) with a static camera, over the whole image and
   over the pixels that took at least 16 samples; scene_animated at 1920x1080 and 2 spp.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return q.stdout.strip().splitlines()[0]


def clamped(x):
    return np.clip(x[..., :3] / np.maximum(x[..., 3:], 1e-12), 0, 1)


def rmse(x, ref, mask=None):
    d = (clamped(x) - clamped(ref)) ** 2
    if mask is not None:
        d = d[mask]
    return float(np.sqrt(d.mean()))


def c4():
    return SB.scene_c4(1_000_000, 1920, 1080, 4096).finish()


def timing(out, reps):
    import torch
    g = api.Scene(c4())
    g.update_frame()
    h, w, dev = g.height, g.width, "cuda:%d" % g.device
    st = torch.cuda.Stream()
    film, alb, nor, lum, den = (torch.zeros((h, w, 4), dtype=torch.float32, device=dev) for _ in range(5))
    near = torch.full((h, w), -1, dtype=torch.int64, device=dev)
    st.wait_stream(torch.cuda.current_stream())
    P = lambda t: t.data_ptr()  # noqa: E731
    hv, hm = api.DenoiseHistory(g), api.DenoiseHistory(g)

    def render():
        with torch.cuda.stream(st):
            for t in (film, alb, nor, lum):
                t.zero_()
            near.fill_(-1)
        g.render_aov_device(P(film), P(alb), P(nor), P(near), None, st.cuda_stream, d_lum=P(lum), spp=2, seed=1, flags=F.RENDER_NO_UPDATE)

    calls = dict(
        variance_temporal=lambda: g.denoise_variance_temporal_device(hv, P(film), P(alb), P(nor), P(near), P(lum), P(den), stream=st.cuda_stream),
        variance=lambda: g.denoise_variance_device(P(film), P(alb), P(nor), P(near), P(lum), P(den), stream=st.cuda_stream),
        moments=lambda: g.denoise_moments_device(hm, P(film), P(alb), P(nor), P(near), P(den), stream=st.cuda_stream))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(*fns):
        e0.record(st)
        for fn in fns:
            fn()
        e1.record(st)
        st.synchronize()
        return e0.elapsed_time(e1)

    render()
    for fn in calls.values():
        for _ in range(3):
            timed(fn)  # warm-up, and a history of 3 frames
    t = {k: [] for k in calls}
    for _ in range(reps):
        for k, fn in calls.items():
            t[k].append(timed(fn))
    out["call_ms"] = {k: round(statistics.median(v), 4) for k, v in t.items()}
    timed(render, calls["variance_temporal"])
    out["frame_ms_render_aov_lum_2spp_plus_variance_temporal"] = round(statistics.median(timed(render, calls["variance_temporal"])
                                                                                          for _ in range(reps)), 3)
    out["render_aov_lum_2spp_ms"] = round(statistics.median(timed(render) for _ in range(reps)), 3)
    from torch.profiler import ProfilerActivity, profile
    split = {}
    for k, fn in calls.items():
        st.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            st.synchronize()
        rows = {}
        for e in prof.key_averages():
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us > 0:
                name = e.key.split("(")[0].replace("void trb::", "")
                rows[name] = round(rows.get(name, 0.0) + us / 1e3, 4)
        split[k] = rows
    out["kernel_ms"] = split
    g.close()


def quality(name, desc, frames, ref_spp, spp=2, adaptive=None, arc=False, animated=False):
    g = api.Scene(desc)
    cam_idx = desc.splines[desc.cameras[0].spline_first].ctrl_first  # the camera's keyframe
    cam = desc.keyframes[cam_idx]
    base_t = np.array(cam.translation, np.float64)
    base = (tuple(cam.rotation), tuple(cam.scaling))
    methods = ["vt", "moments", "variance1", "noisy"] + ([] if adaptive else ["halves"])
    if animated:
        methods += ["vt_grad", "moments_grad", "halves_grad"]
    hist = {m: api.DenoiseHistory(g) for m in methods}
    outs = {m: [] for m in methods}
    refs, many = [], None
    ref = None
    for k in range(frames):
        if arc:
            ang = np.radians(0.5 * k)
            t = base_t + np.array([200 * np.sin(ang), 0.0, 200 * (1 - np.cos(ang))])
            g.update_keyframes(cam_idx, np.array([(tuple(t), base[0], base[1])], F.KEYFRAME_DTYPE))
        if animated:
            g.update_frame(k, 0.25 * k, 0.25 * (k + 1))
        else:
            g.update_frame()
        seed = 1 + k
        nf = F.RENDER_NO_UPDATE
        if adaptive:
            film, aovs, pspp, _ = g.render_adaptive_aov(adaptive[0], adaptive[1], lum=True, seed=seed, flags=nf)
            many = pspp >= 16
        else:
            film, aovs, _ = g.render_aov(spp=spp, lum=True, seed=seed, flags=nf)
        o = outs
        o["noisy"].append(film)
        o["vt"].append(g.denoise_variance_temporal(hist["vt"], film, aovs))
        o["moments"].append(g.denoise_moments(hist["moments"], film, aovs))
        o["variance1"].append(g.denoise_variance(film, aovs))
        if animated:
            o["vt_grad"].append(g.denoise_variance_temporal_gradient(hist["vt_grad"], film, aovs, seed))
            o["moments_grad"].append(g.denoise_moments_gradient(hist["moments_grad"], film, aovs, seed))
        if not adaptive:
            a, aovs_h, _ = g.render_aov(spp=spp, sample_first=0, sample_count=spp // 2, seed=seed, flags=nf)
            b, _, _ = g.render_aov(albedo=aovs_h["albedo_w"], normal=aovs_h["normal_w"], nearest=aovs_h["nearest"], spp=spp,
                                   sample_first=spp // 2, sample_count=spp // 2, seed=seed, flags=nf)
            o["halves"].append(g.denoise_temporal(hist["halves"], a, b, aovs_h))
            if animated:
                o["halves_grad"].append(g.denoise_temporal_gradient(hist["halves_grad"], a, b, aovs_h, seed))
        if ref is None or arc or animated:
            ref, _ = g.render(spp=ref_spp, seed=99, flags=nf)
        refs.append(ref)
    r = {}
    for m in methods:
        seq = outs[m]
        row = dict(rmse=round(float(np.mean([rmse(seq[k], refs[k]) for k in range(1, frames)])), 5),
                   flicker=round(float(np.mean([np.abs(clamped(seq[k]) - clamped(seq[k - 1])).mean() for k in range(1, frames)])), 5))
        if many is not None:
            row["rmse_ge16_last"] = round(rmse(seq[-1], refs[-1], many), 5)
        r[m] = row
    if many is not None:
        r["share_ge16_last"] = round(float(many.mean()), 4)
    g.close()
    print(name, json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--skip-quality", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("denoise_variance_temporal_bench needs a CUDA device")
    out = dict(gpu=gpu_info(), scene="C4 1920x1080")
    timing(out, args.reps)
    print(json.dumps(out), flush=True)
    if not args.skip_quality:
        q = {}
        for spp in (2, 4):
            q["c4_static_%dspp" % spp] = quality("c4 static %d spp" % spp, c4(), args.frames, args.ref_spp, spp=spp)
            q["c4_arc_%dspp" % spp] = quality("c4 arc %d spp" % spp, c4(), args.frames, args.ref_spp, spp=spp, arc=True)
        q["c4_adaptive_2_32"] = quality("c4 adaptive (2, 32)", c4(), args.frames, args.ref_spp, adaptive=(2, 32))
        q["animated_2spp"] = quality("scene_animated 2 spp", SB.scene_animated(1920, 1080, 2, frames=args.frames,
                                                                                scene_time=0.25 * args.frames).finish(),
                                     args.frames, args.ref_spp, animated=True)
        out["quality"] = q
        out["ref_spp"] = args.ref_spp
        out["frames"] = args.frames
    out["gpu_after"] = gpu_info()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""The sample-variance denoiser on C4 at 1920x1080: what the lum_w film costs a render, what trb_denoise_variance costs against
trb_denoise, and what the per-pixel sample variance buys against the half films and the moment call's spatial estimate. Measures and
reports; gates nothing.

    python tools/denoise_variance_bench.py [--reps 5] [--ref-spp 256] [--out results/denoise_variance_bench.json]

1. render_aov_device (albedo, normal, nearest) against the same call with the lum_w film (trb_render_aov_lum_device) at 1 and 8
   spp, alternating, on one torch stream into device buffers: CUDA events around each call, median of --reps after a warm-up.
   Then a run of its own under torch.profiler: the LUM film kernel's time in one lum render.
2. trb_denoise_variance_device against trb_denoise_device (default parameters) on the 8-spp films, alternating.
3. RMSE of colours clamped to [0, 1] against a --ref-spp render at k = 2, 4, 8, 16 spp for four methods: the variance call on one
   k-spp render ("variance"), render_denoised's two halves ("halves"), the moment call at max_history 1 on one k-spp render
   ("moments1") and the noisy k-spp film ("noisy"); each method's render + denoise time (device forms, CUDA events, median of
   --reps). Equal time: for each k, every other method's RMSE at the largest power-of-two spp whose time fits in the variance
   method's time at k.
4. Adaptive (2, 32): the variance call against the moment call at max_history 1, over the whole image and over the pixels that
   took at least 16 samples.
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

KS = (2, 4, 8, 16)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return q.stdout.strip().splitlines()[0]


def rmse(x, ref, mask=None):
    c = np.clip(x[..., :3] / np.maximum(x[..., 3:], 1e-12), 0, 1)
    r = np.clip(ref[..., :3] / np.maximum(ref[..., 3:], 1e-12), 0, 1)
    d = (c - r) ** 2
    if mask is not None:
        d = d[mask]
    return round(float(np.sqrt(d.mean())), 5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("denoise_variance_bench needs a CUDA device")
    out = dict(gpu=gpu_info(), scene="C4 1920x1080")
    g = api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 4096).finish())
    g.update_frame()
    h, w, dev = g.height, g.width, "cuda:%d" % g.device
    st = torch.cuda.Stream()
    film, fb, alb, nor, lum, den = (torch.zeros((h, w, 4), dtype=torch.float32, device=dev) for _ in range(6))
    near = torch.full((h, w), -1, dtype=torch.int64, device=dev)
    st.wait_stream(torch.cuda.current_stream())
    nf = F.RENDER_NO_UPDATE
    P = lambda t: t.data_ptr()  # noqa: E731

    def reset():
        with torch.cuda.stream(st):
            for t in (film, fb, alb, nor, lum):
                t.zero_()
            near.fill_(-1)

    def timed(*fns):
        reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for fn in fns:
            fn()
        e1.record(st)
        st.synchronize()
        return e0.elapsed_time(e1)

    def aov(spp, first=0, count=0, dst=film, with_lum=False):
        return lambda: g.render_aov_device(P(dst), P(alb), P(nor), P(near), None, st.cuda_stream, d_lum=P(lum) if with_lum else None, spp=spp,
                                           sample_first=first, sample_count=count, seed=1, flags=nf)

    def plain(spp):
        return lambda: g.render_device(P(film), None, st.cuda_stream, spp=spp, seed=1, flags=nf)

    def var_dn():
        g.denoise_variance_device(P(film), P(alb), P(nor), P(near), P(lum), P(den), stream=st.cuda_stream)

    def halves_dn():
        g.denoise_device(P(film), P(fb), P(alb), P(nor), P(near), P(den), stream=st.cuda_stream)

    hist = api.DenoiseHistory(g)  # max_history 1: a single-frame filter, whatever the history holds

    def mom_dn():
        g.denoise_moments_device(hist, P(film), P(alb), P(nor), P(near), P(den), stream=st.cuda_stream, max_history=1)

    def med(*fns):
        timed(*fns)  # warm-up
        return statistics.median(timed(*fns) for _ in range(args.reps))

    # 1. the lum_w film's cost, alternating
    for spp in (1, 8):
        timed(aov(spp)); timed(aov(spp, with_lum=True))
        t0, t1 = [], []
        for _ in range(args.reps):
            t0.append(timed(aov(spp)))
            t1.append(timed(aov(spp, with_lum=True)))
        out["render_aov_device_ms_%dspp" % spp] = round(statistics.median(t0), 3)
        out["render_aov_lum_device_ms_%dspp" % spp] = round(statistics.median(t1), 3)
        out["lum_overhead_%dspp" % spp] = round(statistics.median(t1) / statistics.median(t0) - 1.0, 4)
    from torch.profiler import ProfilerActivity, profile
    for spp in (1, 8):
        reset()
        st.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            aov(spp, with_lum=True)()
            st.synchronize()
        total, lum_us, film_us = 0.0, 0.0, 0.0
        for e in prof.key_averages():
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us <= 0:
                continue
            total += us
            if "k_wf_film" in e.key:
                if "true>" in e.key or ", true" in e.key:
                    lum_us += us
                else:
                    film_us += us
        out["profile_%dspp" % spp] = dict(kernel_ms=round(total / 1e3, 3), lum_film_ms=round(lum_us / 1e3, 4), other_film_ms=round(film_us / 1e3, 4),
                                          lum_film_share=round(lum_us / max(total, 1e-9), 4))

    # 2. the denoise calls on the 8-spp films, alternating
    timed(aov(8, 0, 4), aov(8, 4, 4, dst=fb))
    reset()
    aov(8, with_lum=True)()
    aov(8, 4, 4, dst=fb)()
    st.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def time_only(fn):
        e0.record(st)
        fn()
        e1.record(st)
        st.synchronize()
        return e0.elapsed_time(e1)

    time_only(var_dn); time_only(halves_dn)
    tv, th = [], []
    for _ in range(args.reps):
        tv.append(time_only(var_dn))
        th.append(time_only(halves_dn))
    out["denoise_variance_device_ms"] = round(statistics.median(tv), 3)
    out["denoise_device_ms"] = round(statistics.median(th), 3)

    # 3. quality at equal spp and equal time
    times = {m: {} for m in ("variance", "halves", "moments1", "noisy")}
    for k in (1, 2, 4, 8, 16, 32, 64):
        times["noisy"][k] = round(med(plain(k)), 3)
        times["moments1"][k] = round(med(aov(k), mom_dn), 3)
        if k >= 2:
            times["variance"][k] = round(med(aov(k, with_lum=True), var_dn), 3)
            times["halves"][k] = round(med(aov(k, 0, k // 2), aov(k, k // 2, k // 2, dst=fb), halves_dn), 3)
    ref, _ = g.render(spp=args.ref_spp, seed=99, flags=nf)
    err = {m: {} for m in times}
    for k in (1, 2, 4, 8, 16, 32, 64):
        f, _ = g.render(spp=k, seed=1, flags=nf)
        err["noisy"][k] = rmse(f, ref)
        fm, am, _ = g.render_aov(spp=k, seed=1, flags=nf)
        err["moments1"][k] = rmse(g.denoise_moments(api.DenoiseHistory(g), fm, am, max_history=1), ref)
        if k >= 2:
            err["variance"][k] = rmse(g.render_denoised_variance(spp=k, seed=1, flags=nf)[0], ref)
            err["halves"][k] = rmse(g.render_denoised(spp=k, seed=1, flags=nf)[0], ref)
    out["ms"] = times
    out["rmse"] = err
    out["equal_spp"] = {k: {m: err[m][k] for m in err} for k in KS}
    eq = {}
    for k in KS:
        budget = times["variance"][k]
        row = dict(variance=dict(spp=k, ms=budget, rmse=err["variance"][k]))
        for m in ("halves", "moments1", "noisy"):
            fits = [s for s, t in times[m].items() if t <= budget]
            s = max(fits) if fits else min(times[m])
            row[m] = dict(spp=s, ms=times[m][s], rmse=err[m][s])
        eq[k] = row
    out["equal_time"] = eq

    # 4. Adaptive (2, 32): the sample variance against the spatial estimate
    afilm, aaovs, aspp, _ = g.render_adaptive_aov(2, 32, lum=True, seed=1, flags=nf)
    vden = g.denoise_variance(afilm, aaovs)
    mden = g.denoise_moments(api.DenoiseHistory(g), afilm, aaovs, max_history=1)
    many = aspp >= 16
    out["adaptive"] = dict(mean_spp=round(float(aspp.mean()), 3), share_ge16=round(float(many.mean()), 4),
                           rmse_all=dict(variance=rmse(vden, ref), moments1=rmse(mden, ref), noisy=rmse(afilm, ref)),
                           rmse_ge16=dict(variance=rmse(vden, ref, many), moments1=rmse(mden, ref, many), noisy=rmse(afilm, ref, many)))
    out["ref_spp"] = args.ref_spp
    out["gpu_after"] = gpu_info()
    g.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""AOVs of Adaptive renders on C4 at 1920x1080: what the AOVs cost the Adaptive sampler, and what Adaptive + the moment denoiser
buys at equal time. Measures and reports; gates nothing.

    python tools/adaptive_aov_bench.py [--min 2] [--max 32] [--reps 5] [--ref-spp 256] [--out results/adaptive_aov_bench.json]

1. render_adaptive_device against render_adaptive_aov_device (albedo, normal, nearest), alternating, on one torch stream into device
   buffers: CUDA events around each call, median of --reps after one warm-up of each.
2. A run of its own under torch.profiler: the kernel times of one render_adaptive_aov_device call; the new kernels' share.
3. Equal-time quality, RMSE of colours clamped to [0, 1] against a --ref-spp LowDiscrepancy render: Adaptive (min, max) denoised by
   the moment call as a single-frame filter (max_history 1) and noisy, and LowDiscrepancy at the largest power-of-two spp whose
   render_aov + moment call fits in the Adaptive render + moment call's time, denoised and noisy. Times are device-form calls
   between CUDA events, median of --reps.
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

NEW_KERNELS = ("k_wf_aov_ad", "k_wf_nearest_ad", "k_ad_aov_slots")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return q.stdout.strip().splitlines()[0]


def rmse(x, ref):
    c = np.clip(x[..., :3] / np.maximum(x[..., 3:], 1e-12), 0, 1)
    r = np.clip(ref[..., :3] / np.maximum(ref[..., 3:], 1e-12), 0, 1)
    return float(np.sqrt(np.mean((c - r) ** 2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min", type=int, default=2)
    ap.add_argument("--max", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("adaptive_aov_bench needs a CUDA device")
    out = dict(gpu=gpu_info(), scene="C4 1920x1080", adaptive=[args.min, args.max])
    g = api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 4096).finish())
    g.update_frame()
    h, w, dev = g.height, g.width, "cuda:%d" % g.device
    st = torch.cuda.Stream()
    film, alb, nor, den = (torch.zeros((h, w, 4), dtype=torch.float32, device=dev) for _ in range(4))
    near = torch.full((h, w), -1, dtype=torch.int64, device=dev)
    st.wait_stream(torch.cuda.current_stream())
    nf = F.RENDER_NO_UPDATE

    def reset():
        with torch.cuda.stream(st):
            for t in (film, alb, nor):
                t.zero_()
            near.fill_(-1)

    def plain():
        g.render_adaptive_device(args.min, args.max, film.data_ptr(), None, None, st.cuda_stream, seed=1, flags=nf)

    def with_aov():
        g.render_adaptive_aov_device(args.min, args.max, film.data_ptr(), alb.data_ptr(), nor.data_ptr(), near.data_ptr(), None, None, st.cuda_stream,
                                     seed=1, flags=nf)

    def ld_aov(spp):
        return lambda: g.render_aov_device(film.data_ptr(), alb.data_ptr(), nor.data_ptr(), near.data_ptr(), None, st.cuda_stream, spp=spp, seed=1,
                                           flags=nf)

    hist = api.DenoiseHistory(g)  # max_history 1: a single-frame filter, whatever the history holds

    def denoise():
        g.denoise_moments_device(hist, film.data_ptr(), alb.data_ptr(), nor.data_ptr(), near.data_ptr(), den.data_ptr(),
                                 stream=st.cuda_stream, max_history=1)

    def timed(*fns):
        reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for fn in fns:
            fn()
        e1.record(st)
        st.synchronize()
        return e0.elapsed_time(e1)

    # 1. the AOVs' cost, alternating
    timed(plain); timed(with_aov)  # warm-up: allocations, first launches
    t_plain, t_aov = [], []
    for _ in range(args.reps):
        t_plain.append(timed(plain))
        t_aov.append(timed(with_aov))
    out["render_adaptive_device_ms"] = round(statistics.median(t_plain), 3)
    out["render_adaptive_aov_device_ms"] = round(statistics.median(t_aov), 3)
    out["aov_overhead"] = round(statistics.median(t_aov) / statistics.median(t_plain) - 1.0, 4)

    # 2. kernel split under the profiler (a run of its own: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    reset()
    st.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with_aov()
        st.synchronize()
    total, new, split = 0.0, 0.0, {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
        if us <= 0:
            continue
        total += us
        if any(k in e.key for k in NEW_KERNELS) or "k_wf_film" in e.key:
            split[e.key[:60]] = dict(ms=round(us / 1e3, 4), launches=e.count)
        if any(k in e.key for k in NEW_KERNELS):
            new += us
    out["profiled_kernel_ms"] = round(total / 1e3, 3)
    out["new_kernels_ms"] = round(new / 1e3, 4)
    out["new_kernels_share"] = round(new / max(total, 1e-9), 4)
    out["kernels"] = split

    # 3. equal-time quality
    t_ad = statistics.median(timed(with_aov, denoise) for _ in range(args.reps))
    ld = {}
    spp = 1
    while True:
        t = statistics.median(timed(ld_aov(spp), denoise) for _ in range(args.reps))
        ld[spp] = round(t, 3)
        if t > t_ad or spp >= 1024:
            break
        spp *= 2
    fits = [s for s, t in ld.items() if t <= t_ad]
    ld_spp = max(fits) if fits else 1
    out["adaptive_denoised_ms"] = round(t_ad, 3)
    out["ld_aov_denoised_ms_by_spp"] = ld
    out["ld_equal_time_spp"] = ld_spp
    ref, _ = g.render(spp=args.ref_spp, seed=99, flags=nf)
    afilm, aaovs, aspp, _ = g.render_adaptive_aov(args.min, args.max, seed=1, flags=nf)
    aden = g.denoise_moments(api.DenoiseHistory(g), afilm, aaovs, max_history=1)
    lfilm, laovs, _ = g.render_aov(spp=ld_spp, seed=1, flags=nf)
    lden = g.denoise_moments(api.DenoiseHistory(g), lfilm, laovs, max_history=1)
    out["adaptive_mean_spp"] = round(float(aspp.mean()), 3)
    out["rmse"] = dict(adaptive_denoised=rmse(aden, ref), adaptive_noisy=rmse(afilm, ref), ld_denoised=rmse(lden, ref), ld_noisy=rmse(lfilm, ref))
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

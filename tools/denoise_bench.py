"""Time the denoiser on C4 at 1920 x 1080 and measure what it buys. On one stream, CUDA events around each call, median of --reps after
a warm-up:
  - trb_denoise_device at 0 to 5 and 10 iterations on the halves of a 2-spp AOV render, and from the differences the time of the
    iteration at each step 1 .. 16;
  - a 2-spp frame as two 1-spp trb_render_aov_device halves plus the denoise, against a plain 2-spp trb_render_device;
  - equal-time quality: for k = 2, 4, 8 the RMSE (colours clamped to [0, 1]) of the denoised k-spp frame and of a noisy frame of the
    sample count whose plain render takes the same time (sample_count need not be a power of two), both against a --ref-spp render.
Then, in a run of its own under torch.profiler, the per-kernel split of one 5-iteration denoise (k_dn_prepare, k_dn_atrous). The
GPU's name and power limit are read in the same call. Prints one JSON line.

    python tools/denoise_bench.py [--tris 1000000] [--reps 5] [--ref-spp 256]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def rmse(film, ref):
    c = np.clip(film[..., :3] / np.maximum(film[..., 3:], 1e-12), 0, 1)
    r = np.clip(ref[..., :3] / ref[..., 3:], 0, 1)
    return float(np.sqrt(((c - r) ** 2).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-spp", type=int, default=256)
    args = ap.parse_args()
    import torch
    out = dict(gpu=gpu_info())
    s = api.Scene(SB.scene_c4(args.tris, 1920, 1080, 2).finish())
    s.update_frame(0, 0.0, 0.0)
    h, w = s.height, s.width
    st = torch.cuda.Stream()
    film = lambda: torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")  # noqa: E731
    a, b, albedo, normal, den = film(), film(), film(), film(), film()
    nearest = torch.full((h, w), -1, dtype=torch.int64, device="cuda")

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record(st)
            f()
            e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1)

    def halves(spp):
        for t in (a, b, albedo, normal):
            t.zero_()
        nearest.fill_(-1)
        for first, t in ((0, a), (spp // 2, b)):
            s.render_aov_device(t.data_ptr(), albedo.data_ptr(), normal.data_ptr(), nearest.data_ptr(), stream=st.cuda_stream, spp=spp,
                                sample_first=first, sample_count=spp // 2, seed=5)

    ptrs = lambda: (a.data_ptr(), b.data_ptr(), albedo.data_ptr(), normal.data_ptr(), nearest.data_ptr(), den.data_ptr())  # noqa: E731
    denoise = lambda **p: s.denoise_device(*ptrs(), stream=st.cuda_stream, **p)  # noqa: E731
    med = lambda xs: round(statistics.median(xs[1:]), 4)  # noqa: E731

    with torch.cuda.stream(st):
        halves(2)
    st.synchronize()
    out["denoise_ms"] = {str(it): med([timed(lambda: denoise(iterations=it)) for _ in range(args.reps + 1)]) for it in (0, 1, 2, 3, 4, 5, 10)}
    # the cost of the iteration at step 2^(i-1): does the wider, less cache-friendly step cost more?
    out["iteration_ms_by_step"] = {str(1 << (i - 1)): round(out["denoise_ms"][str(i)] - out["denoise_ms"][str(i - 1)], 4) for i in range(1, 6)}
    out["denoise_ms_all_5"] = [round(timed(lambda: denoise(iterations=5)), 4) for _ in range(args.reps)]

    plain_film = film()

    def plain(spp, count=0):
        plain_film.zero_()
        s.render_device(plain_film.data_ptr(), stream=st.cuda_stream, spp=spp, sample_count=count, seed=5)

    rows = {"render_2spp_ms": [], "aov_halves_2spp_ms": [], "aov_halves_plus_denoise_2spp_ms": []}
    for _ in range(args.reps + 1):
        rows["render_2spp_ms"].append(timed(lambda: plain(2)))
        rows["aov_halves_2spp_ms"].append(timed(lambda: halves(2)))
        rows["aov_halves_plus_denoise_2spp_ms"].append(timed(lambda: (halves(2), denoise())))
    out.update({k: med(v) for k, v in rows.items()})

    # equal-time quality against a high-spp reference
    ref = film()
    step = 16
    for first in range(0, args.ref_spp, step):
        s.render_device(ref.data_ptr(), stream=st.cuda_stream, spp=args.ref_spp, sample_first=first, sample_count=step, seed=99)
    st.synchronize()
    ref_h = ref.cpu().numpy()
    per_sample = med([timed(lambda: plain(16)) for _ in range(args.reps + 1)]) / 16
    out["plain_ms_per_spp"] = round(per_sample, 4)
    eq = {}
    for k in (2, 4, 8):
        t_den = med([timed(lambda: (halves(k), denoise())) for _ in range(args.reps + 1)])
        den_rmse = rmse(den.cpu().numpy(), ref_h)
        m = max(1, int(t_den / per_sample))
        pow2 = 1 << (m - 1).bit_length()
        t_noisy = med([timed(lambda: plain(pow2, m)) for _ in range(args.reps + 1)])
        eq["k%d" % k] = dict(denoised_ms=t_den, denoised_rmse=round(den_rmse, 5), noisy_spp=m, noisy_ms=t_noisy,
                             noisy_rmse=round(rmse(plain_film.cpu().numpy(), ref_h), 5),
                             noisy_same_spp_rmse=round(rmse((a + b).cpu().numpy(), ref_h), 5))
    out["equal_time"] = eq
    out["ref_spp"] = args.ref_spp

    # kernel split under the profiler (a run of its own: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    with torch.cuda.stream(st):
        halves(2)
        denoise()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with torch.cuda.stream(st):
            denoise(iterations=5)
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
        if us > 0 and "k_dn_" in e.key:
            split[e.key[:40]] = dict(ms=round(us / 1e3, 4), launches=e.count)
    out["kernel_ms_5_iterations"] = split
    out["gpu_after"] = gpu_info()
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

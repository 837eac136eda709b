"""Time AOV renders on C4 at 1920 x 1080: trb_render_device and trb_render_aov_device (albedo, normal and nearest) alternate on one stream
at 1 and 8 spp, median of 5 after a warm-up, CUDA events around each call. Then, in a run of its own under torch.profiler, the times of
k_wf_aov, k_wf_nearest and the film kernel, which an AOV render launches once for the colour and once per AOV film. For comparison,
the composed query route for the normal film and depth only: trb_camera_rays_device -> trb_intersect_records_device (96-byte records)
-> trb_film_write_device of the records' normals (the rays' conversion to query rays and the samples' assembly are torch copies, timed
with it). The GPU's name and power limit are read in the same call. Prints one JSON line.

    python tools/aov_bench.py [--tris 1000000] [--reps 5]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    out = dict(gpu=gpu_info())
    s = api.Scene(SB.scene_c4(args.tris, 1920, 1080, 8).finish())
    s.update_frame(0, 0.0, 0.0)
    h, w = s.height, s.width
    st = torch.cuda.Stream()
    film = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    albedo, normal = torch.zeros_like(film), torch.zeros_like(film)
    nearest = torch.full((h, w), -1, dtype=torch.int64, device="cuda")

    def timed(f):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            a.record(st)
            f()
            b.record(st)
        b.synchronize()
        return a.elapsed_time(b)

    plain = lambda spp: s.render_device(film.data_ptr(), stream=st.cuda_stream, spp=spp, seed=3)  # noqa: E731
    aov = lambda spp: s.render_aov_device(film.data_ptr(), albedo.data_ptr(), normal.data_ptr(), nearest.data_ptr(), stream=st.cuda_stream,  # noqa: E731
                                          spp=spp, seed=3)
    for spp in (1, 8):
        rows = {"render_ms": [], "render_aov_ms": []}
        for r in range(args.reps + 1):
            rows["render_ms"].append(timed(lambda: plain(spp)))
            rows["render_aov_ms"].append(timed(lambda: aov(spp)))
        res = {k: round(statistics.median(v[1:]), 3) for k, v in rows.items()}
        res.update({k + "_all": [round(x, 3) for x in v[1:]] for k, v in rows.items()})
        res["overhead_ms"] = round(res["render_aov_ms"] - res["render_ms"], 3)

        # the composed query route: normal film and per-sample depth from a second primary trace
        n = s._n_samples(api._cfg(spp=spp))
        rays = torch.empty((n, 8), dtype=torch.float32, device="cuda")
        xy = torch.empty((n, 2), dtype=torch.float32, device="cuda")
        q = torch.zeros((n, 12), dtype=torch.float32, device="cuda")
        rec = torch.empty((n, 24), dtype=torch.float32, device="cuda")
        smp = torch.empty((n, 5), dtype=torch.float32, device="cuda")
        regions = torch.from_numpy(s.sample_regions(spp=spp).view(np.int32)).cuda()
        nfilm = torch.zeros_like(film)

        def composed():
            s.camera_rays_device(rays.data_ptr(), xy.data_ptr(), stream=st.cuda_stream, spp=spp, seed=3)
            q[:, :8] = rays
            s.intersect_records_device(n, q.data_ptr(), rec.data_ptr(), stream=st.cuda_stream)
            smp[:, :2] = xy
            smp[:, 2:] = rec[:, 7:10]  # trb_intersection.n
            s.film_write_device(n, smp.data_ptr(), regions.data_ptr(), nfilm.data_ptr(), stream=st.cuda_stream)
        res["composed_normal_depth_ms"] = round(statistics.median([timed(composed) for _ in range(args.reps + 1)][1:]), 3)
        del rays, xy, q, rec, smp, regions
        out["spp%d" % spp] = res
        torch.cuda.empty_cache()

    # kernel times under the profiler (a run of its own: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    for spp in (1, 8):
        aov(spp)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with torch.cuda.stream(st):
                aov(spp)
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us > 0 and any(k in e.key for k in ("k_wf_aov", "k_wf_nearest", "k_wf_film")):
                split[e.key[:60]] = dict(ms=round(us / 1e3, 4), launches=e.count)
        out["spp%d" % spp]["kernel_ms"] = split
    out["gpu_after"] = gpu_info()
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

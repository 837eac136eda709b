"""What the motion_w film costs an AOV render: C4 (1M triangles) and the keyframed scene at 1920x1080. Measures and reports; gates nothing.

    python tools/motion_bench.py [--reps 7] [--out results/motion_bench.json]

1. render_aov_lum_device (albedo, normal, nearest, lum_w) against the same call with the motion_w film (trb_render_aov_motion_device,
   dt one frame back) at 1 and 8 spp, alternating, on one torch stream into device buffers: CUDA events around each call, median of
   --reps after a warm-up.
2. A run of its own under torch.profiler per scene and spp: the motion kernel's time (k_wf_motion) and the film launches (k_wf_film
   or k_wf_film_v2 without the LUM flag: colour, albedo, normal and, with motion, motion_w), so the extra film launch is their
   difference.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return q.stdout.strip().splitlines()[0]


def scenes():
    yield "C4 1920x1080", SB.scene_c4(1_000_000, 1920, 1080, 4096).finish(), (0, 0.0, 0.0)
    yield "keyframed 1920x1080", SB.scene_animated(1920, 1080, 8).finish(), (1, 0.25, 0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        sys.exit("motion_bench needs a CUDA device")
    out = dict(gpu=gpu_info(), results=[])
    for name, desc, frame in scenes():
        g = api.Scene(desc)
        g.update_frame(*frame)
        h, w, dev = g.height, g.width, "cuda:%d" % g.device
        st = torch.cuda.Stream()
        film, alb, nor, lum, mo = (torch.zeros((h, w, 4), dtype=torch.float32, device=dev) for _ in range(5))
        near = torch.full((h, w), -1, dtype=torch.int64, device=dev)
        st.wait_stream(torch.cuda.current_stream())
        P = lambda t: t.data_ptr()  # noqa: E731

        def call(spp, motion):
            g.render_aov_device(P(film), P(alb), P(nor), P(near), None, st.cuda_stream, d_lum=P(lum), d_motion=P(mo) if motion else None,
                                spp=spp, seed=1, flags=F.RENDER_NO_UPDATE)

        def timed(spp, motion):
            with torch.cuda.stream(st):
                for t in (film, alb, nor, lum, mo):
                    t.zero_()
                near.fill_(-1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            call(spp, motion)
            e1.record(st)
            st.synchronize()
            return e0.elapsed_time(e1)

        for spp in (1, 8):
            timed(spp, False), timed(spp, True)  # warm-up, including the first motion render's record allocation
            t0, t1 = [], []
            for _ in range(args.reps):
                t0.append(timed(spp, False))
                t1.append(timed(spp, True))
            row = dict(scene=name, spp=spp, lum_ms=round(statistics.median(t0), 3), lum_motion_ms=round(statistics.median(t1), 3))
            row["motion_overhead"] = round(row["lum_motion_ms"] / row["lum_ms"] - 1.0, 4)
            for motion in (False, True):
                st.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(spp, motion)
                    st.synchronize()
                motion_us, film_us, n_film = 0.0, 0.0, 0
                for e in prof.key_averages():
                    us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
                    if "k_wf_motion" in e.key:
                        motion_us += us
                    elif "k_wf_film" in e.key and "true>" not in e.key and ", true" not in e.key:
                        film_us += us
                        n_film += e.count
                key = "with_motion" if motion else "without_motion"
                row[key] = dict(k_wf_motion_ms=round(motion_us / 1e3, 4), film_ms=round(film_us / 1e3, 4), film_launches=n_film)
            row["extra_film_launch_ms"] = round(row["with_motion"]["film_ms"] - row["without_motion"]["film_ms"], 4)
            out["results"].append(row)
            print(json.dumps(row), flush=True)
        g.close()
    print(json.dumps(dict(gpu=out["gpu"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

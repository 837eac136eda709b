"""AOV renders and denoised frames on a trb_group against one GPU, on C4 at 1920x1080. Measures and reports; gates nothing.

    python tools/multi_gpu_aov_bench.py [--devices 0,1,2,3] [--spp 4] [--reps 5] [--out results/multi_gpu_aov_bench.json]

1. Group(devices).render_aov against Scene.render_aov on device 0 (colour, albedo, normal and nearest into host buffers), alternating,
   with a second Scene on device 0 as the control for run-to-run spread: CUDA events on device 0's default stream around each
   blocking call, median, min and max of --reps after one warm-up of each.
2. The per-frame NCCL group of the group's AOV render, timed separately: one render_aov under torch.profiler, the sum of the NCCL
   kernels' device time per GPU (the colour film, albedo + normal and nearest reduces). A group of one device performs no reduce.
3. A 1-spp moment-denoised frame (render_denoised_moments with a fresh history, so a single-frame filter) on the group against one
   GPU, timed as in 1.
With one device in --devices the tool measures what the group costs over the scene on one GPU; scaling needs two or more.
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
from tray_rust_b200 import api, scenebuild as SB  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30, check=True)
    return q.stdout.strip().splitlines()


def timed(torch, call, reps):
    """median device-0 milliseconds of a blocking call between CUDA events on the default stream"""
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms)


def alternate(torch, calls, reps):
    """the calls' medians and ranges, measured in alternation, in forward and reverse order by turns, so that clock and thermal
    drift and the position in the sequence fall on all of them alike"""
    for c in calls.values():
        c()  # warm-up: first-use allocations, block lists
    ms = {k: [] for k in calls}
    order = list(calls)
    for i in range(reps):
        for k in (order if i % 2 == 0 else order[::-1]):
            ms[k].append(timed(torch, calls[k], 1))
    return {k: dict(median=round(statistics.median(v), 3), min=round(min(v), 3), max=round(max(v), 3)) for k, v in ms.items()}


def nccl_ms(torch, call):
    """device time of the NCCL kernels in one call, per CUDA device"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if "nccl" in e.name.lower() and e.device_type.name == "CUDA":
            per[e.device_index] = per.get(e.device_index, 0.0) + e.device_time / 1e3
    return {str(k): round(v, 3) for k, v in sorted(per.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default=None, help="comma-separated device list (default: every visible GPU)")
    ap.add_argument("--spp", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("multi_gpu_aov_bench needs a CUDA device")
    devices = [int(d) for d in args.devices.split(",")] if args.devices else list(range(torch.cuda.device_count()))
    torch.cuda.set_device(devices[0])
    out = dict(gpus=gpu_info(), devices=devices, scene="C4 1920x1080, 1 M triangles", spp=args.spp, reps=args.reps)

    def desc():
        return SB.scene_c4(1_000_000, 1920, 1080, 4096).finish()

    # a second scene on device 0 is the control: what two identical one-GPU calls differ by in this run
    s, s2, grp = api.Scene(desc(), devices[0]), api.Scene(desc(), devices[0]), api.Group(desc(), devices)
    kw = dict(spp=args.spp, seed=3)
    ms = alternate(torch, {"scene_render_aov": lambda: s.render_aov(**kw), "group_render_aov": lambda: grp.render_aov(**kw),
                           "control_scene_render_aov": lambda: s2.render_aov(**kw)}, args.reps)
    out["render_aov_ms"] = ms
    out["render_aov_speedup"] = round(ms["scene_render_aov"]["median"] / ms["group_render_aov"]["median"], 3)
    out["nccl_group_ms_per_device"] = nccl_ms(torch, lambda: grp.render_aov(**kw)) if len(devices) > 1 else "no reduce: one device"

    def moments(r, scene):
        def call():
            h = api.DenoiseHistory(scene)
            r.render_denoised_moments(h, 1, seed=3)
            h.close()
        return call

    ms = alternate(torch, {"scene_denoised_moments_1spp": moments(s, s), "group_denoised_moments_1spp": moments(grp, grp.scene(0)),
                           "control_scene_denoised_moments_1spp": moments(s2, s2)}, args.reps)
    out["denoised_moments_1spp_ms"] = ms
    out["denoised_moments_1spp_speedup"] = round(ms["scene_denoised_moments_1spp"]["median"] / ms["group_denoised_moments_1spp"]["median"], 3)
    grp.close()
    s.close()
    s2.close()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()

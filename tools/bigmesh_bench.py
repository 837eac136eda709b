"""Developer tool: the wide mesh leaf form on one GPU (needs CUDA; prints one JSON object, also written to --out if given).

  * the GPU's name and power limit (read in the same run as the numbers);
  * trb_scene_create wall time for the scenebuild.scene_heightfield mesh (host SAH build + upload; 4200 x 4200 vertices =
    35 263 202 triangles, more than a narrow mesh leaf reference can address);
  * whole-path Mrays/s (primary + shadow + MIS + continuation rays over device time) on that scene at 1920x1080;
  * C4 (bench.py's 1 M-triangle scene, 1920x1080) with trace.wide_leaf 0 and 1 on one scene in the same process, alternating
    runs, so the two forms' difference can be held against the run-to-run spread.

  python tools/bigmesh_bench.py [--grid 4200] [--spp-per-run 4] [--runs 5] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tray_rust_b200 import api, scenebuild as SB  # noqa: E402


def gpu_info():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def timed_runs(g, spp_per_run, first_run, n_runs, seed=1):
    """n_runs passes of spp_per_run samples per pixel over the whole frame; Mrays/s per pass from CUDA events and the ray counters"""
    import torch
    dev = torch.device("cuda:0")
    film = torch.zeros((g.height, g.width, 4), dtype=torch.float32, device=dev)
    stats = torch.zeros(10, dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    out = []
    for k in range(n_runs):
        i = first_run + k
        stats.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.render_device(film.data_ptr(), stats.data_ptr(), stream, spp=g.spp, sample_first=i * spp_per_run, sample_count=spp_per_run, seed=seed)
        e1.record()
        torch.cuda.synchronize()
        st = stats.cpu().numpy()
        ms = e0.elapsed_time(e1)
        out.append({"ms": ms, "rays": int(st[1:5].sum()), "mrays_s": float(st[1:5].sum()) / ms / 1e3})
    return out


def spread(vals):
    v = np.array(vals)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max()), "runs": [float(x) for x in v]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--spp-per-run", type=int, default=4)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    a = ap.parse_args()
    res = {"gpu": gpu_info()}

    t0 = time.perf_counter()
    desc = SB.scene_heightfield(a.grid, 1920, 1080, 4096).finish()
    res["bigmesh_generate_s"] = time.perf_counter() - t0
    res["bigmesh_tris"] = int(desc.meshes[0].n_tris)
    t0 = time.perf_counter()
    g = api.Scene(desc)
    res["bigmesh_create_s"] = time.perf_counter() - t0
    g.update_frame(0, 0.0, 0.0)
    timed_runs(g, a.spp_per_run, 0, 1)                                         # warm-up
    runs = timed_runs(g, a.spp_per_run, 1, a.runs)
    res["bigmesh_mrays_s"] = spread([r["mrays_s"] for r in runs])
    res["bigmesh_rays_per_run"] = runs[0]["rays"]
    g.close(); del g, desc

    c4 = api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 4096).finish())
    c4.update_frame(0, 0.0, 0.0)
    vals = {0: [], 1: []}
    for form in (0, 1):                                                        # warm both forms
        c4.set_option("trace.wide_leaf", form)
        timed_runs(c4, a.spp_per_run, 0, 1)
    run = 1
    for _ in range(a.runs):
        for form in (0, 1):
            c4.set_option("trace.wide_leaf", form)
            vals[form] += [r["mrays_s"] for r in timed_runs(c4, a.spp_per_run, run, 1)]
            run += 1
    res["c4_narrow_mrays_s"] = spread(vals[0])
    res["c4_wide_mrays_s"] = spread(vals[1])
    res["c4_wide_over_narrow_median"] = res["c4_wide_mrays_s"]["median"] / res["c4_narrow_mrays_s"]["median"]
    res["config"] = {"grid": a.grid, "spp_per_run": a.spp_per_run, "runs": a.runs, "resolution": "1920x1080"}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

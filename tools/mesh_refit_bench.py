"""Time trb_scene_refit_mesh_device against trb_scene_update_mesh_device on C4's 1 M-triangle mesh and the 35 M-triangle heightfield
(grid 4200), alternately in one process, the vertices moving between two deformed states; median of 5 after a warm-up, host clock around
each blocking call. Per round: update_mesh (a rebuild), then the first refit of the rebuilt tree (which computes its parent links),
then a second refit (the steady state of a mesh refit every frame), then that refit followed by a 1-spp 1920 x 1080 trb_render_device.
Then the kernel split of the steady refit under torch.profiler, and what the refit costs in traversal: a travelling wave run for
--steps refits, then a 1-spp render with counters and the trace kernel timed (RENDER_TIME_TRACE), on the refit tree and, after
update_mesh to the same positions, on a rebuilt tree. The GPU's name and power limit are read in the same call. Prints one JSON line.

    python tools/mesh_refit_bench.py [--grid 4200] [--c4 1000000] [--reps 5] [--steps 64]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def desc_of(kind, n, seed):
    return (SB.scene_c4(n, 1920, 1080, 1, seed) if kind == "c4" else SB.scene_heightfield(n, 1920, 1080, 1, seed)).finish()


def deformed(p, t):
    """a travelling wave in y (heights of the heightfield; the random triangles of C4 ride the same field)"""
    q = p.copy()
    q[:, 1] += (1.5 * np.sin(0.7 * p[:, 0] - 2.0 * t) * np.cos(0.3 * p[:, 2] + t)).astype(np.float32)
    return q


def bench(kind, n, reps, steps, seed):
    import torch
    desc = desc_of(kind, n, seed)
    me = desc.meshes[0]
    p0 = np.ctypeslib.as_array(me.positions, (me.n_verts * 3,)).reshape(-1, 3).copy()
    states = [torch.from_numpy(deformed(p0, t)).cuda() for t in (0.5, 1.0)]
    s = api.Scene(desc)
    s.update_frame(0, 0.0, 0.0)
    stream = torch.cuda.current_stream().cuda_stream
    film = torch.zeros((1080, 1920, 4), dtype=torch.float32, device="cuda")

    def timed(f):
        torch.cuda.synchronize()
        t = time.perf_counter()
        f()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3

    refit = lambda k: s.refit_mesh_device(0, states[k].data_ptr(), None, None, stream=stream)  # noqa: E731
    rows = {"update_ms": [], "refit_first_ms": [], "refit_ms": [], "refit_render_ms": [], "render_ms": []}
    for r in range(reps + 1):
        k = r % 2
        rows["update_ms"].append(timed(lambda: s.update_mesh_device(0, states[k].data_ptr(), None, None, stream=stream)))
        rows["refit_first_ms"].append(timed(lambda: refit(1 - k)))
        rows["refit_ms"].append(timed(lambda: refit(k)))
        rows["refit_render_ms"].append(timed(lambda: (refit(1 - k), s.render_device(film.data_ptr(), stream=stream, spp=1, seed=3))))
        rows["render_ms"].append(timed(lambda: s.render_device(film.data_ptr(), stream=stream, spp=1, seed=3)))
    out = dict(triangles=int(me.n_tris), **{key: statistics.median(v[1:]) for key, v in rows.items()})
    out["refit_ms_all"] = [round(x, 3) for x in rows["refit_ms"][1:]]
    out["update_ms_all"] = [round(x, 3) for x in rows["update_ms"][1:]]

    # kernel split of the steady refit (a run of its own: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    refit(0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in (1, 0, 1, 0):
            refit(k)
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us > 0:
                split[e.key[:60]] = round(us / 4 / 1e3, 4)  # ms per refit
    out["refit_kernel_split_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1]))

    # traversal after a long deformation: refit tree against a rebuilt tree on the same positions
    for t in range(steps):
        step = torch.from_numpy(deformed(p0, 0.1 * t)).cuda()
        s.refit_mesh_device(0, step.data_ptr(), None, None, stream=stream)
    final = step

    def traversal():
        s.render_samples(spp=1, seed=3, flags=F.RENDER_TIME_TRACE)  # warm-up of this tree
        s.trace_time()
        _, st = s.render_samples(spp=1, seed=3, flags=F.RENDER_STATS | F.RENDER_TIME_TRACE)
        ms, launches = s.trace_time()
        return dict(trace_ms=round(ms, 3), node_tests_per_ray=round(st.node_tests / st.rays_total(), 3),
                    tri_tests_per_ray=round(st.tri_tests / st.rays_total(), 3))
    out["after_%d_steps_refit" % steps] = traversal()
    s.update_mesh_device(0, final.data_ptr(), None, None, stream=stream)
    out["after_%d_steps_rebuilt" % steps] = traversal()
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--c4", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    if args.child:  # one workload per process, so that the two scenes never share the device memory
        kind, n = args.child.split(":")
        print(json.dumps(bench(kind, int(n), args.reps, args.steps, 0x5EED1E55 if kind == "c4" else 0x4E16F1D)))
        return
    out = dict(gpu=gpu_info())
    for kind, n in (("c4", args.c4), ("heightfield", args.grid)):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "%s:%d" % (kind, n), "--reps", str(args.reps),
                            "--steps", str(args.steps)], capture_output=True, text=True, cwd=tempfile.gettempdir())
        out[kind] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else dict(error=r.stderr[-2000:])
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Time trb_scene_update_mesh_device: C4's 1 M-triangle mesh and the 35 M-triangle heightfield (grid 4200), each updated between two
seeds of the same topology, median of 5 after a warm-up; beside it trb_build_bvh_device on the same triangle boxes and
trb_scene_create of the same scene in a fresh process whose CUDA context exists before the timer starts. The phase split (build /
read-back of the tree / triangle records / node-record packing / frame refresh) is the library's own report (TRB_MESH_UPDATE_TIME=1:
CUDA events on the default stream), median over the timed updates (the warm-up excluded). Prints one JSON line.

    python tools/mesh_update_bench.py [--grid 4200] [--c4 1000000] [--reps 5]
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


def meshes(kind, n, seed):
    if kind == "c4":
        return SB.random_triangle_mesh(n, seed)
    return SB.heightfield_mesh(n, seed)


def desc_of(kind, n, seed):
    return (SB.scene_c4(n, 64, 64, 1, seed) if kind == "c4" else SB.scene_heightfield(n, 64, 64, 1, seed)).finish()


def create_time(kind, n, seed):
    """trb_scene_create of the scene in a fresh process (description built and CUDA context created first, neither timed)"""
    code = ("import sys, time; sys.path.insert(0, %r)\n"
            "from tools.mesh_update_bench import desc_of\nfrom tray_rust_b200 import api\nimport torch\n"
            "d = desc_of(%r, %d, %d)\ntorch.zeros(1, device='cuda'); torch.cuda.synchronize()\n"
            "t = time.perf_counter(); s = api.Scene(d); print(time.perf_counter() - t)\n") % (REPO, kind, n, seed)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=tempfile.gettempdir())
    return float(r.stdout.strip().splitlines()[-1]) * 1e3 if r.returncode == 0 else None


def phases_of(text):
    out = {}
    for line in text.splitlines():
        if line.startswith("trb_scene_update_mesh "):
            name, ms = line[len("trb_scene_update_mesh "):].rsplit(" ", 2)[0], float(line.split()[-2])
            out.setdefault(name, []).append(ms)
    return {k: statistics.median(v[1:]) for k, v in out.items() if len(v) > 1}  # v[0]: the warm-up


def bench(kind, n, reps, seed_a, seed_b):
    import torch
    a, b = meshes(kind, n, seed_a), meshes(kind, n, seed_b)
    d_a = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a[:3]]
    d_b = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in b[:3]]
    s = api.Scene(desc_of(kind, n, seed_a))
    s.update_frame(0, 0.0, 0.0)
    stream = torch.cuda.current_stream().cuda_stream
    times = []
    for r in range(reps + 1):
        src = d_b if r % 2 == 0 else d_a
        torch.cuda.synchronize()
        t = time.perf_counter()
        s.update_mesh_device(0, src[0].data_ptr(), None, None, stream=stream)
        times.append((time.perf_counter() - t) * 1e3)
    s.close()
    # trb_build_bvh_device over the same triangle boxes (Triangle::bounds of the seed-B positions)
    p, i = b[0], b[3]
    tri = p[i.astype(np.int64)]
    boxes = np.concatenate([tri.min(axis=1), tri.max(axis=1)], axis=1).astype(np.float32)
    nt = len(boxes)
    d_boxes = torch.from_numpy(boxes).cuda()
    d_nodes = torch.empty((2 * nt - 1, 8), dtype=torch.int32, device="cuda")
    d_order = torch.empty(nt, dtype=torch.int32, device="cuda")
    d_nn = torch.zeros(1, dtype=torch.int32, device="cuda")
    bt = []
    for r in range(reps + 1):
        torch.cuda.synchronize()
        t = time.perf_counter()
        api.build_bvh_device(d_boxes.data_ptr(), nt, 16, d_nn.data_ptr(), d_nodes.data_ptr(), d_order.data_ptr(), stream=stream)
        torch.cuda.synchronize()
        bt.append((time.perf_counter() - t) * 1e3)
    del d_boxes, d_nodes, d_order, d_a, d_b
    torch.cuda.empty_cache()
    return dict(triangles=nt, update_ms=statistics.median(times[1:]), build_bvh_device_ms=statistics.median(bt[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--c4", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    if args.child:  # one workload, phases reported by the library on stderr
        kind, n = args.child.split(":")
        seeds = (0x5EED1E55, 0x5EED1E56) if kind == "c4" else (0x4E16F1D, 0x1234567)
        print(json.dumps(bench(kind, int(n), args.reps, *seeds)))
        return
    out = dict(gpu=gpu_info())
    for kind, n in (("c4", args.c4), ("heightfield", args.grid)):
        env = dict(os.environ, TRB_MESH_UPDATE_TIME="1")
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "%s:%d" % (kind, n), "--reps", str(args.reps)],
                           capture_output=True, text=True, env=env, cwd=tempfile.gettempdir())
        if r.returncode != 0:
            out[kind] = dict(error=r.stderr[-2000:])
            continue
        res = json.loads(r.stdout.strip().splitlines()[-1])
        res["phases_ms"] = phases_of(r.stderr)
        res["create_ms"] = create_time(kind, n, 0x5EED1E56 if kind == "c4" else 0x1234567)
        out[kind] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

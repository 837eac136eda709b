"""Developer tool: the mesh BVH build on one GPU (needs CUDA; prints one JSON object, also written to --out if given).

  * the GPU's name and power limit (read in the same run as the numbers);
  * trb_scene_create wall time for the scenebuild.scene_heightfield mesh (4200 x 4200 vertices = 35 263 202 triangles), C4
    (1 M triangles) and the tr15-shaped scene, with TRB_BUILD_DEVICE 1 (device build) and 0 (host build) alternating; each
    creation runs in a fresh process, which also reports its peak host RSS and the device memory in use after creation;
  * trb_build_bvh_device time and Mboxes/s on 1 M and 16 M random boxes and on the heightfield's 35 M triangle boxes, median
    of 5 after a warm-up (CUDA events around the call; the call synchronises its stream once per level).

  python tools/build_bench.py [--grid 4200] [--rounds 2] [--out results.json]
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests", "golden"))
from tray_rust_b200 import api, scenebuild as SB  # noqa: E402


def gpu_info():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def scene_desc(name, grid):
    if name == "heightfield":
        return SB.scene_heightfield(grid, 1920, 1080, 4).finish()
    if name == "c4":
        return SB.scene_c4(1000000, 1920, 1080, 4).finish()
    import make_golden
    return make_golden.golden_scenes()["c5_tr15_like_f12"][0]()


def create_once(name, grid):
    """child process: one trb_scene_create of the named scene under the environment's TRB_BUILD_DEVICE"""
    import torch
    desc = scene_desc(name, grid)
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info(0)
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    t0 = time.perf_counter()
    g = api.Scene(desc)
    t1 = time.perf_counter()
    free1, _ = torch.cuda.mem_get_info(0)
    rss1 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    nodes, order = g.bvh(0)
    h = np.frombuffer(nodes.tobytes() + order.tobytes(), np.uint8)
    digest = int(np.bitwise_xor.reduce(h[: len(h) // 8 * 8].view(np.uint64))) if len(h) >= 8 else 0
    return {"create_s": t1 - t0, "peak_rss_before_gb": rss0 / 1e6, "peak_rss_after_gb": rss1 / 1e6,
            "device_gb_after_create": (free0 - free1) / 1e9, "mesh0_digest": digest}


def build_timings(grid):
    import torch
    out = {}
    rng = np.random.default_rng(1)
    sets = {}
    for n in (1 << 20, 1 << 24):
        c = rng.uniform(-100, 100, (n, 3)).astype(np.float32)
        e = rng.uniform(0, 0.2, (n, 3)).astype(np.float32)
        sets["random_%d" % n] = np.concatenate([c - e, c + e], axis=1)
    desc = SB.scene_heightfield(grid, 64, 64, 1).finish()
    m = desc.meshes[0]
    p = np.ctypeslib.as_array(m.positions, shape=(m.n_verts * 3,)).reshape(-1, 3)
    ix = np.ctypeslib.as_array(m.indices, shape=(m.n_tris * 3,)).reshape(-1, 3)
    tri = p[ix]
    sets["heightfield_%d" % m.n_tris] = np.concatenate([tri.min(axis=1), tri.max(axis=1)], axis=1).astype(np.float32)
    del tri
    for name, boxes in sets.items():
        n = len(boxes)
        d_boxes = torch.from_numpy(boxes).cuda()
        d_nodes = torch.empty((2 * n - 1) * 8, dtype=torch.int32, device="cuda")
        d_order = torch.empty(n, dtype=torch.int32, device="cuda")
        d_nn = torch.zeros(1, dtype=torch.int32, device="cuda")
        stream = torch.cuda.current_stream()
        ms = []
        for k in range(6):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            api.build_bvh_device(d_boxes.data_ptr(), n, 16, d_nn.data_ptr(), d_nodes.data_ptr(), d_order.data_ptr(), stream=stream.cuda_stream)
            e1.record()
            torch.cuda.synchronize()
            if k:
                ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        out[name] = {"n": n, "nodes": int(d_nn.cpu()[0]), "ms_runs": ms, "median_ms": med, "mboxes_s": n / med / 1e3}
        del d_boxes, d_nodes, d_order
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out")
    ap.add_argument("--create", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.create:
        print(json.dumps(create_once(a.create, a.grid)))
        return
    res = {"gpu": gpu_info(), "create": {}, "build_device": build_timings(a.grid)}
    for name in ("heightfield", "c4", "tr15_like"):
        runs = []
        for r in range(a.rounds):
            for dev in ((1, 0) if r % 2 == 0 else (0, 1)):
                env = dict(os.environ, TRB_BUILD_DEVICE=str(dev))
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--create", name, "--grid", str(a.grid)],
                                   capture_output=True, text=True, env=env, check=True)
                runs.append(dict(json.loads(p.stdout.strip().splitlines()[-1]), build_device=dev))
        res["create"][name] = runs
        assert len({r["mesh0_digest"] for r in runs}) == 1, "device and host builds differ on " + name
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()

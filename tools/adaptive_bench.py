"""Adaptive sampler vs LowDiscrepancy on one GPU: wall time, camera samples, Mrays/s, rounds and the RMSE of each image
against a high-spp LowDiscrepancy render of the same scene. Measures and reports; gates nothing.

    python tools/adaptive_bench.py [--n 8] [--ref-spp 256] [--scenes c2,c4] [--out results/adaptive_bench.json]

LD runs at N spp, Adaptive at (N/4, 4N); both one trb_render / trb_render_adaptive call each, after one warm-up call. The
"adaptive_device" row is the same Adaptive render through trb_render_adaptive_device on a torch stream into a device film:
GPU time between CUDA events on that stream, and the host time the call took to enqueue every round.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def img(film):
    return film[..., :3] / np.maximum(film[..., 3:], 1e-6)


def rmse(a, b):
    return float(np.sqrt(np.mean((img(a) - img(b)) ** 2)))


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def scene(name):
    if name == "c2":
        import ctypes as C
        lib = F.load_trb()
        d = C.POINTER(F.SceneDesc)()
        path = os.path.join(REPO, "tests", "golden", "scenes", "c2_smallpt.json")
        assert lib.trb_desc_load_json(path.encode(), 512, 512, 1024, C.byref(d)) == F.TRB_OK
        g = api.Scene(d.contents)
        g._desc = None
        lib.trb_desc_free(d)
        return g
    return api.Scene(SB.scene_c4(1_000_000, 1920, 1080, 4096).finish())


def rounds_of(spp, mn, mx):
    mn2, _, step, _ = api.adaptive_schedule(mn, mx)
    return int(1 + np.max((spp.astype(np.int64) - mn2 + step - 1) // step))


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def device_timed(g, mn, mx, seed):
    """trb_render_adaptive_device on a non-default stream: (GPU ms between events, enqueue ms, camera samples)"""
    import torch
    s = torch.cuda.Stream(device=g.device)
    film = torch.zeros((g.height, g.width, 4), dtype=torch.float32, device="cuda:%d" % g.device)
    stats = torch.zeros(9, dtype=torch.int64, device=film.device)
    s.wait_stream(torch.cuda.current_stream(film.device))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.render_adaptive_device(mn, mx, film.data_ptr(), None, stats.data_ptr(), s.cuda_stream, seed=seed, flags=F.RENDER_NO_UPDATE)  # warm-up
    s.synchronize()
    film.zero_()
    stats.zero_()
    torch.cuda.synchronize(film.device)
    e0.record(s)
    t0 = time.perf_counter()
    g.render_adaptive_device(mn, mx, film.data_ptr(), None, stats.data_ptr(), s.cuda_stream, seed=seed, flags=F.RENDER_NO_UPDATE)
    enqueue = time.perf_counter() - t0
    e1.record(s)
    e1.synchronize()
    st = F.Stats.from_buffer_copy(stats.cpu().numpy().tobytes())
    return e0.elapsed_time(e1), enqueue * 1e3, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8)
    ap.add_argument("--ref-spp", type=int, default=256)
    ap.add_argument("--scenes", default="c2,c4")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"device": device_info(), "n": a.n, "adaptive": [a.n // 4, 4 * a.n], "ref_spp": a.ref_spp, "scenes": {}}
    for name in a.scenes.split(","):
        g = scene(name)
        ref, _ = g.render(spp=a.ref_spp, seed=99)
        g.render(spp=a.n, seed=1)                      # warm-up of both paths
        g.render_adaptive(a.n // 4, 4 * a.n, seed=1)
        (ld, st_ld), t_ld = timed(lambda: g.render(spp=a.n, seed=2))
        (ad, spp, st_ad), t_ad = timed(lambda: g.render_adaptive(a.n // 4, 4 * a.n, seed=2))
        row = {
            "ld": {"wall_s": t_ld, "camera_samples": st_ld.camera_samples, "mrays_s": st_ld.rays_total() / t_ld / 1e6, "rmse": rmse(ld, ref)},
            "adaptive": {"wall_s": t_ad, "camera_samples": st_ad.camera_samples, "mrays_s": st_ad.rays_total() / t_ad / 1e6, "rmse": rmse(ad, ref),
                         "rounds": rounds_of(spp, a.n // 4, 4 * a.n), "mean_spp": float(spp.mean()), "pixels_at_min": float((spp == spp.min()).mean())},
        }
        gpu_ms, enqueue_ms, st_dev = device_timed(g, a.n // 4, 4 * a.n, 2)
        row["adaptive_device"] = {"gpu_ms": gpu_ms, "enqueue_ms": enqueue_ms, "camera_samples": st_dev.camera_samples,
                                  "mrays_s": st_dev.rays_total() / gpu_ms / 1e3}
        res["scenes"][name] = row
        print(name, json.dumps(row), flush=True)
        g.close()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

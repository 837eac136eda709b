"""Adaptive sampler vs LowDiscrepancy on one GPU: wall time, camera samples, Mrays/s, rounds and the RMSE of each image
against a high-spp LowDiscrepancy render of the same scene. Measures and reports; gates nothing.

    python tools/adaptive_bench.py [--n 8] [--ref-spp 256] [--scenes c2,c4] [--out results/adaptive_bench.json]

LD runs at N spp, Adaptive at (N/4, 4N); both one trb_render / trb_render_adaptive call each, after one warm-up call.
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

"""Time trb_scene_replace_settings and trb_scene_replace_materials on C4 (1920 x 1080, 1 M triangles), median of 5 after a warm-up,
host clock around each blocking call. Prints one JSON line with the card's name and power limit.

- settings: the film switched 1920 x 1080 -> 480 x 272 (270 rounded up to whole 8 x 8 blocks) and back, the integrator switched Path -> NormalsDebug and back, and each of
  these followed by a 1-spp trb_render at the size it leaves (each timed call follows the untimed one that undoes it);
- materials, with a 4096 x 4096 texture bound to the mesh's colour: the material section replaced from host memory, and through
  the _device form from a torch tensor holding the texture;
- for comparison: trb_scene_create + update_frame of C4 with the texture, in a fresh process.

    python tools/settings_bench.py [--reps 5]
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
from tools.scene_edit_bench import gpu_info  # noqa: E402

MESH_MAT = 3  # three wall materials, then the mesh's
TEX = 4096


def timed(reps, call, undo=lambda: None):
    """median ms of call(): each timed call follows the untimed undo(); one warm-up"""
    times = []
    for _ in range(reps + 1):
        undo()
        t = time.perf_counter()
        call()
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times[1:])


def textured_c4():
    """C4 with a seeded 4096 x 4096 RGBA8 texture on the mesh's colour"""
    b = SB.scene_c4(1_000_000, 1920, 1080, 1)
    px = np.random.default_rng(4).integers(0, 256, (TEX, TEX, 4), dtype=np.uint8)
    t = b.add_texture(px)
    b.materials[MESH_MAT] = b.materials[MESH_MAT][:6] + ((t, 0, 0, 0),)
    return b


def bench_settings(reps):
    b = SB.scene_c4(1_000_000, 1920, 1080, 1)
    s = api.Scene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    full, small = dict(b.film), dict(b.film, width=480, height=272)  # 480 x 270 rounded up to whole 8 x 8 blocks
    path, normals = tuple(b.integrator), (F.INTEGRATOR_NORMALS_DEBUG, 0, 1)
    render = lambda: s.render(spp=1)  # noqa: E731
    out = dict(small_film=[small["width"], small["height"]])
    out["to_small_ms"] = timed(reps, lambda: s.replace_settings(small), lambda: s.replace_settings(full))
    out["to_full_ms"] = timed(reps, lambda: s.replace_settings(full), lambda: s.replace_settings(small))
    out["to_small_render_ms"] = timed(reps, lambda: (s.replace_settings(small), render()), lambda: s.replace_settings(full))
    out["to_full_render_ms"] = timed(reps, lambda: (s.replace_settings(full), render()), lambda: s.replace_settings(small))
    out["to_normals_debug_ms"] = timed(reps, lambda: s.replace_settings(integrator=normals), lambda: s.replace_settings(integrator=path))
    out["to_path_ms"] = timed(reps, lambda: s.replace_settings(integrator=path), lambda: s.replace_settings(integrator=normals))
    out["to_normals_debug_render_ms"] = timed(reps, lambda: (s.replace_settings(integrator=normals), render()),
                                              lambda: s.replace_settings(integrator=path))
    out["to_path_render_ms"] = timed(reps, lambda: (s.replace_settings(integrator=path), render()),
                                     lambda: s.replace_settings(integrator=normals))
    out["render_ms"] = timed(reps, render)
    s.close()
    return out


def bench_materials(reps):
    import torch
    b = textured_c4()
    s = api.Scene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    host = b.materials_section()
    px = b.images[0][0]
    d_px = torch.from_numpy(px).cuda()
    b.images[0] = (d_px, b.images[0][1])
    dev = b.materials_section()
    b.images[0] = (px, b.images[0][1])
    out = dict(texture=[TEX, TEX])
    out["host_ms"] = timed(reps, lambda: s.replace_materials(host))
    out["device_ms"] = timed(reps, lambda: s.replace_materials_device(dev))
    s.close()
    return out


def create_time():
    """trb_scene_create + update_frame of the textured C4, in a fresh process"""
    code = ("import sys, time; sys.path.insert(0, %r)\n"
            "from tools.settings_bench import textured_c4\nfrom tray_rust_b200 import api\nimport torch\n"
            "d = textured_c4().finish()\ntorch.zeros(1, device='cuda'); torch.cuda.synchronize()\n"
            "t = time.perf_counter(); s = api.Scene(d); s.update_frame(0, 0.0, 0.0); print(time.perf_counter() - t)\n") % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=tempfile.gettempdir())
    return float(r.stdout.strip().splitlines()[-1]) * 1e3 if r.returncode == 0 else r.stderr[-2000:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info(), settings=bench_settings(args.reps), materials=bench_materials(args.reps),
                          create_frame_ms=create_time())))


if __name__ == "__main__":
    main()

"""Time trb_scene_replace_objects, median of 5 after a warm-up, host clock around each blocking call. Prints one JSON line with the
card's name and power limit.

- C4 (1920 x 1080, 1 M triangles): the object section replaced to add one sphere, to remove it again and to bind the mesh instance to
  another material (each alternating with the section it undoes); the add followed by a 1-spp trb_render; for comparison
  trb_scene_create + trb_scene_update_frame + the same render in a fresh process (scene_edit_bench.c4_create_time).
- the heightfield (grid 4200: 35 M triangles): trb_scene_create, then the same add.
- scenebuild.scene_instances(k), k = 10^3, 10^4, 10^5: the section replaced by that of 2k instances and back; then, in a separate
  process under torch.profiler, the kernel times of k_frame_instances and k_tlas_build (mean per replacement), the two kernels of the
  frame rebuild that a replacement runs.

    python tools/scene_objects_bench.py [--instances 1000,10000,100000] [--grid 4200] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402
from tools.scene_edit_bench import c4_create_time, gpu_info, timed  # noqa: E402

MESH_INST, MESH_MAT = 6, 3  # five walls and the light, then the mesh instance; three wall materials, then the mesh's


def replace_ms(s, new, old, reps):
    """median ms of replacing the section `old` by `new`: each timed call follows the untimed one that undoes it; one warm-up"""
    times = []
    for _ in range(reps + 1):
        s.replace_objects(old)
        t = time.perf_counter()
        s.replace_objects(new)
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times[1:])


def with_sphere(b):
    """the sections of builder b as it is and with one more sphere"""
    plain = b.objects()
    b.receiver(F.SHAPE_SPHERE, MESH_MAT, [SB.trs(t=(0, 15, 5), s=2)], p0=1.0)
    return plain, b.objects()


def bench_c4(reps):
    import numpy as np
    b = SB.scene_c4(1_000_000, 1920, 1080, 1)
    s = api.Scene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    plain, more = with_sphere(b)
    b.remove_instance(len(b.instances) - 1)
    b.instances[MESH_INST] = b.instances[MESH_INST][:5] + (0,) + b.instances[MESH_INST][6:]  # the white walls' material
    rebound = b.objects()
    film = np.zeros((s.height, s.width, 4), np.float32)

    def add_render(r):
        s.replace_objects(more if r % 2 == 0 else plain)
        s.render(film, spp=1)
    out = dict(add_sphere_ms=replace_ms(s, more, plain, reps), remove_sphere_ms=replace_ms(s, plain, more, reps),
               rebind_material_ms=replace_ms(s, rebound, plain, reps),
               replace_render_ms=timed(add_render, reps))
    s.close()
    out["create_frame_render_ms"] = c4_create_time()
    return out


def bench_heightfield(grid, reps):
    b = SB.scene_heightfield(grid)
    d = b.finish()
    t = time.perf_counter()
    s = api.Scene(d)
    create = (time.perf_counter() - t) * 1e3
    s.update_frame(0, 0.0, 0.0)
    plain, more = with_sphere(b)
    out = dict(triangles=int(d.meshes[0].n_tris), create_ms=create, add_sphere_ms=replace_ms(s, more, plain, reps))
    s.close()
    return out


def instance_sections(k, seed=9):
    """scene_instances(k) with its frame set, and the sections of 2k and of k instances"""
    s = api.Scene(SB.scene_instances(k, seed).finish())
    s.update_frame(0, 0.0, 0.0)
    return s, SB.scene_instances(2 * k, seed).objects(), SB.scene_instances(k, seed).objects()


def profile_instances(k, reps):
    """mean device time per replacement of k_frame_instances and k_tlas_build, from torch.profiler (half the replacements build the
    frame of 2k instances, half that of k)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    s, double, single = instance_sections(k)
    s.replace_objects(double)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(2 * reps):
            s.replace_objects(single if r % 2 == 0 else double)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("k_frame_instances", "k_tlas_build"):
            if name in ev.key:
                total = getattr(ev, "device_time_total", None)
                if total is None:
                    total = ev.cuda_time_total
                out[name + "_ms"] = total / 1e3 / (2 * reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", default="1000,10000,100000")
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", type=int, default=None)
    args = ap.parse_args()
    if args.profile:  # a separate process: tracing slows the host
        print(json.dumps(profile_instances(args.profile, args.reps)))
        return
    out = dict(gpu=gpu_info(), c4=bench_c4(args.reps), heightfield=bench_heightfield(args.grid, args.reps))
    for k in (int(x) for x in args.instances.split(",")):
        s, double, single = instance_sections(k)
        res = dict(to_2k_ms=replace_ms(s, double, single, args.reps), to_k_ms=replace_ms(s, single, double, args.reps))
        s.close()
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile", str(k), "--reps", str(args.reps)], capture_output=True,
                           text=True, cwd=tempfile.gettempdir())
        res["kernels"] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else r.stderr[-2000:]
        out["instances_%d" % k] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

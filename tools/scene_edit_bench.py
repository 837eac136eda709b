"""Time the scene edits (trb_scene_update_keyframes / _device / _color_keys / _materials), median of 5 after a warm-up, host clock around
each blocking call. Prints one JSON line with the card's name and power limit.

- C4 (1920 x 1080, 1 M triangles): a camera keyframe edit alone and followed by a 1-spp trb_render; for comparison
  trb_scene_create + trb_scene_update_frame + the same render in a fresh process (description built and CUDA context created before
  the timer); a material edit and a colour-key edit alone.
- scenebuild.scene_instances(k), k = 10^3, 10^4, 10^5: trb_scene_update_keyframes_device moving every instance; then, in a separate
  process under torch.profiler, the kernel times of k_frame_instances and k_tlas_build (mean per edit), the two kernels of the frame
  rebuild that such an edit runs.

    python tools/scene_edit_bench.py [--instances 1000,10000,100000] [--reps 5]
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

C4_CAMERA_KF, C4_MESH_MAT = 12, 3  # five walls (two levels each), the light, the mesh instance, then the camera; three wall materials


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps):
    """median ms of reps calls after one warm-up call; fn(r) gets the call's index"""
    times = []
    for r in range(reps + 1):
        t = time.perf_counter()
        fn(r)
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times[1:])


def c4_desc():
    return SB.scene_c4(1_000_000, 1920, 1080, 1).finish()


def c4_create_time():
    """trb_scene_create + update_frame + a 1-spp render of C4 in a fresh process"""
    code = ("import sys, time; sys.path.insert(0, %r)\n"
            "from tools.scene_edit_bench import c4_desc\nfrom tray_rust_b200 import api\nimport torch\n"
            "d = c4_desc()\ntorch.zeros(1, device='cuda'); torch.cuda.synchronize()\n"
            "t = time.perf_counter(); s = api.Scene(d); s.update_frame(0, 0.0, 0.0); s.render(spp=1); print(time.perf_counter() - t)\n") % REPO
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=tempfile.gettempdir())
    return float(r.stdout.strip().splitlines()[-1]) * 1e3 if r.returncode == 0 else r.stderr[-2000:]


def bench_c4(reps):
    s = api.Scene(c4_desc())
    s.update_frame(0, 0.0, 0.0)
    cams = [np.array([SB.trs(t=(x, 12, -60), q=SB.quat_axis_angle((0, 1, 0), x / 4))], F.KEYFRAME_DTYPE) for x in (-2.0, 2.0)]
    film = np.zeros((s.height, s.width, 4), np.float32)

    def edit_render(r):
        s.update_keyframes(C4_CAMERA_KF, cams[r % 2])
        s.render(film, spp=1)
    mats = [np.array([(F.MAT_MATTE, c, (0, 0, 0), 1.0, 1.0, 0, (0, 0, 0, 0))], F.MATERIAL_DTYPE) for c in ((0.7, 0.7, 0.7), (0.5, 0.6, 0.7))]
    keys = [np.array([((x, x, x, 1.0), 0.0)], F.COLOR_KEY_DTYPE) for x in (30.0, 40.0)]
    out = dict(camera_edit_ms=timed(lambda r: s.update_keyframes(C4_CAMERA_KF, cams[r % 2]), reps),
               camera_edit_render_ms=timed(edit_render, reps),
               material_edit_ms=timed(lambda r: s.update_materials(C4_MESH_MAT, mats[r % 2]), reps),
               color_key_edit_ms=timed(lambda r: s.update_color_keys(0, keys[r % 2]), reps))
    s.close()
    out["create_frame_render_ms"] = c4_create_time()
    return out


def instance_edits(k, seed=9):
    """scene_instances(k) with its frame set, and two device arrays that move every instance"""
    import torch
    s = api.Scene(SB.scene_instances(k, seed).finish())
    s.update_frame(0, 0.0, 0.0)
    rng = np.random.default_rng(seed)
    moves = [torch.from_numpy(np.array([SB.trs(t=t, s=0.3) for t in rng.uniform((-13, 1, -8), (13, 22, 18), size=(k, 3))], F.KEYFRAME_DTYPE)
                              .view(np.float32).reshape(k, 10).copy()).cuda() for _ in range(2)]
    torch.cuda.synchronize()
    return s, moves, lambda r: s.update_keyframes_device(11, k, moves[r % 2].data_ptr())  # five walls (two levels each), the light


def profile_instances(k, reps):
    """mean device time per edit of k_frame_instances and k_tlas_build, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    s, moves, edit = instance_edits(k)
    edit(0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(reps):
            edit(r + 1)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("k_frame_instances", "k_tlas_build"):
            if name in ev.key:
                total = getattr(ev, "device_time_total", None)
                if total is None:
                    total = ev.cuda_time_total
                out[name + "_ms"] = total / 1e3 / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", default="1000,10000,100000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", type=int, default=None)
    args = ap.parse_args()
    if args.profile:  # a separate process: tracing slows the host
        print(json.dumps(profile_instances(args.profile, args.reps)))
        return
    out = dict(gpu=gpu_info(), c4=bench_c4(args.reps))
    for k in (int(x) for x in args.instances.split(",")):
        s, moves, edit = instance_edits(k)
        res = dict(update_keyframes_device_ms=timed(edit, args.reps))
        s.close()
        del moves
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile", str(k), "--reps", str(args.reps)], capture_output=True,
                           text=True, cwd=tempfile.gettempdir())
        res["kernels"] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else r.stderr[-2000:]
        out["instances_%d" % k] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

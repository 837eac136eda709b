"""Time trb_scene_update_frame with each builder of the instance tree (option frame.tlas_min): scenebuild.scene_instances(k) for
k = 10 ... 10^6, the one-thread kernel and the level builder alternating in one process, median of --reps calls after a warm-up, host
clock around the blocking call; the phase report (TRB_FRAME_TIME) of one further call of each; at 10^5 a keyframe edit of every instance,
alone and followed by a 1-spp trb_render at 1920 x 1080. Before any timing the two builders' trb_scene_get_bvh(-1) bytes are compared at
each k, and nothing is printed for a k where they differ. The one-thread arm is skipped at 10^6 (over ten seconds of one CUDA thread
per call). first_frame_host_ms is the host time before the first launch of the scene's first frame, which fills and uploads the static
instance records; the phases' "host before the first launch" is that of a later frame, which does not. TRB_FRAME_TLAS_SMALL=<n> in the
environment runs the level builder with another serial-subtree threshold (the sweep behind the default). Prints one JSON line with
the card's name and power limit.

    python tools/tlas_bench.py [--instances 10,100,1000,10000,100000,1000000] [--reps 5] [--mesh]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

os.environ["TRB_FRAME_TIME"] = "1"  # read when a scene is created
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402

LEVEL, ONE_THREAD = 0, 1 << 40
ONE_THREAD_MAX = 100_000
FIRST_KF = 11  # five walls (two levels each) and the light come first


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


class Stderr:
    """the C library's stderr (the phase report) captured into a file for the duration"""

    def __enter__(self):
        sys.stderr.flush()
        self.tmp = tempfile.TemporaryFile()
        self.saved = os.dup(2)
        os.dup2(self.tmp.fileno(), 2)
        return self

    def __exit__(self, *exc):
        ctypes.CDLL(None).fflush(None)
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.tmp.seek(0)
        self.text = self.tmp.read().decode()
        self.tmp.close()


def phases(text):
    """the last report in `text` as {phase: ms or count}"""
    out = {}
    for line in text.splitlines():
        w = line.split()
        if not line.startswith("trb_scene_update_frame "):
            continue
        if w[1] == "instances":
            out = {"builder": w[4]}
        elif w[1] == "levels":
            out["levels"], out["launches"] = int(w[2]), int(w[4])
        else:
            out[" ".join(w[1:-2])] = float(w[-2])
    return out


def bench(k, reps, mesh):
    s = api.Scene(SB.scene_instances(k, 9, mesh=mesh).finish())
    arms = [("level", LEVEL)] + ([("one_thread", ONE_THREAD)] if k <= ONE_THREAD_MAX else [])
    res, trees, times = {}, {}, {name: [] for name, _ in arms}
    with Stderr() as first:  # the scene's first frame also fills and uploads the static instance records
        s.set_option("frame.tlas_min", arms[0][1])
        s.update_frame(0, 0.0, 0.0)
    res["first_frame_host_ms"] = phases(first.text).get("host before the first launch")
    with Stderr():
        for name, v in arms:
            s.set_option("frame.tlas_min", v)
            s.update_frame(0, 0.0, 0.0)
            trees[name] = [a.tobytes() for a in s.bvh(-1)]
    if len(arms) == 2 and trees["level"] != trees["one_thread"]:
        return dict(error="the two builders' trees differ: not timed")
    with Stderr():
        for r in range(reps + 1):  # alternating; the first round is the warm-up
            for name, v in arms:
                s.set_option("frame.tlas_min", v)  # untimed: a change of the option rebuilds the frame by itself
                t = time.perf_counter()
                s.update_frame(0, 0.0, 0.0)
                if r:
                    times[name].append((time.perf_counter() - t) * 1e3)
    for name, v in arms:
        s.set_option("frame.tlas_min", v)
        with Stderr() as err:
            s.update_frame(0, 0.0, 0.0)
        res[name] = dict(median_ms=statistics.median(times[name]), min_ms=min(times[name]), max_ms=max(times[name]), phases=phases(err.text))
    if len(arms) == 1:
        res["one_thread"] = "skipped: more than ten seconds of one CUDA thread per call"
    s.close()
    return res


def bench_edit(k, reps, mesh):
    """a keyframe edit of every instance (default builder choice), alone and with a 1-spp 1920 x 1080 render"""
    import torch
    s = api.Scene(SB.scene_instances(k, 9, 1920, 1080, 1, mesh=mesh).finish())
    s.update_frame(0, 0.0, 0.0)
    rng = np.random.default_rng(9)
    moves = [torch.from_numpy(np.array([SB.trs(t=t, s=0.3) for t in rng.uniform((-13, 1, -8), (13, 22, 18), size=(k, 3))], F.KEYFRAME_DTYPE)
                              .view(np.float32).reshape(k, 10).copy()).cuda() for _ in range(2)]
    torch.cuda.synchronize()
    film = np.zeros((s.height, s.width, 4), np.float32)
    out = {}
    with Stderr():
        for name in ("edit_ms", "edit_render_ms", "render_ms"):
            times = []
            for r in range(reps + 1):
                t = time.perf_counter()
                if name != "render_ms":
                    s.update_keyframes_device(FIRST_KF, k, moves[r % 2].data_ptr())
                if name != "edit_ms":
                    s.render(film, spp=1, flags=F.RENDER_NO_UPDATE)
                times.append((time.perf_counter() - t) * 1e3)
            out[name] = statistics.median(times[1:])
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", default="10,100,1000,10000,100000,1000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mesh", action="store_true", help="instances of one shared mesh instead of spheres")
    ap.add_argument("--edit", type=int, default=100_000, help="instance count of the edit-plus-render timing (0: none)")
    args = ap.parse_args()
    out = dict(gpu=gpu_info(), mesh=args.mesh)
    for k in (int(x) for x in args.instances.split(",")):
        out["instances_%d" % k] = bench(k, args.reps, args.mesh)
        print("instances_%d" % k, json.dumps(out["instances_%d" % k]), file=sys.stderr, flush=True)
    if args.edit:
        out["edit_%d" % args.edit] = bench_edit(args.edit, args.reps, args.mesh)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

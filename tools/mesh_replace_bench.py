"""Time trb_scene_replace_meshes, median of 5 after a warm-up, host clock around each blocking call. Prints one JSON line with the
card's name and power limit.

- the heightfield (grid 4200: 35 M triangles): trb_scene_create, then C4's 1 M-triangle random mesh added with an instance of it and
  removed again (each timed call follows the untimed one that undoes it); the add followed by a 1-spp 1920 x 1080 trb_render; for
  comparison trb_scene_create + update_frame of the combined scene in a fresh process.
- C4 (1920 x 1080, 1 M triangles): a 20 480-triangle icosphere added with an instance and removed again, its topology swapped
  (subdivision 5 <-> 4, no object section), and the add followed by a 1-spp trb_render.

    python tools/mesh_replace_bench.py [--grid 4200] [--reps 5]
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
from tools.scene_edit_bench import gpu_info  # noqa: E402

C4_SEED = 0x5EED1E55
MESH_MAT = 3  # three wall materials, then the mesh's


def mesh_section(meshes, keep):
    """a trb_scene_meshes of the given arrays with an explicit keep list"""
    t = SB.SceneBuilder()
    t.meshes = list(meshes)
    s = t.meshes_section()
    for i, k in enumerate(keep):
        s.keep[i] = k
    return s


def with_mesh(b, mesh, xf):
    """(mesh list, object section) of builder b as it is, and with `mesh` and an instance of it added; each applies to a scene that
    holds the other"""
    n = len(b.meshes)
    plain = (mesh_section(b.meshes, list(range(n))), b.objects())
    m = b.add_mesh(*mesh)
    b.receiver(F.SHAPE_MESH, MESH_MAT, [xf], mesh=m)
    more = (mesh_section(b.meshes, list(range(n)) + [F.MESH_NEW]), b.objects())
    return plain, more


def replace_ms(s, new, old, reps, then=lambda: None):
    """median ms of replacing `old` by `new` (and then()): each timed call follows the untimed one that undoes it; one warm-up"""
    times = []
    for _ in range(reps + 1):
        s.replace_meshes(*old)
        t = time.perf_counter()
        s.replace_meshes(*new)
        then()
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times[1:])


def add_render_ms(s, plain, more, reps):
    """the add followed by a 1-spp trb_render"""
    import numpy as np
    film = np.zeros((s.height, s.width, 4), np.float32)
    return replace_ms(s, more, plain, reps, lambda: s.render(film, spp=1))


def combined_create_time(grid):
    """trb_scene_create + update_frame of the heightfield scene with C4's mesh and its instance, in a fresh process"""
    code = ("import sys, time; sys.path.insert(0, %r)\n"
            "from tray_rust_b200 import _ffi as F, api, scenebuild as SB\nimport torch\n"
            "b = SB.scene_heightfield(%d)\nm = b.add_mesh(*SB.random_triangle_mesh(1_000_000, %d))\n"
            "b.receiver(F.SHAPE_MESH, %d, [SB.trs(t=(0, 4, 0), s=0.5)], mesh=m)\nd = b.finish()\n"
            "torch.zeros(1, device='cuda'); torch.cuda.synchronize()\n"
            "t = time.perf_counter(); s = api.Scene(d); s.update_frame(0, 0.0, 0.0); print(time.perf_counter() - t)\n") % (
        REPO, grid, C4_SEED, MESH_MAT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=tempfile.gettempdir())
    return float(r.stdout.strip().splitlines()[-1]) * 1e3 if r.returncode == 0 else r.stderr[-2000:]


def bench_heightfield(grid, reps):
    b = SB.scene_heightfield(grid)
    d = b.finish()
    t = time.perf_counter()
    s = api.Scene(d)
    create = (time.perf_counter() - t) * 1e3
    s.update_frame(0, 0.0, 0.0)
    plain, more = with_mesh(b, SB.random_triangle_mesh(1_000_000, C4_SEED), SB.trs(t=(0, 4, 0), s=0.5))
    out = dict(triangles=int(d.meshes[0].n_tris), create_ms=create, add_1m_mesh_ms=replace_ms(s, more, plain, reps),
               remove_1m_mesh_ms=replace_ms(s, plain, more, reps), add_render_ms=add_render_ms(s, plain, more, reps))
    s.close()
    out["combined_create_frame_ms"] = combined_create_time(grid)
    return out


def bench_c4(reps):
    b = SB.scene_c4(1_000_000, 1920, 1080, 1)
    s = api.Scene(b.finish())
    s.update_frame(0, 0.0, 0.0)
    ball = SB.icosphere_mesh(5, 3.0, 0.05, 1)
    plain, more = with_mesh(b, ball, SB.trs(t=(-6, 16, 2)))
    out = dict(icosphere_triangles=len(ball[3]), add_icosphere_ms=replace_ms(s, more, plain, reps),
               remove_icosphere_ms=replace_ms(s, plain, more, reps))
    fine, coarse = (mesh_section([b.meshes[0], SB.icosphere_mesh(k, 3.0, 0.05, 1)], [0, F.MESH_NEW]) for k in (5, 4))
    s.replace_meshes(*more)
    out["swap_topology_ms"] = replace_ms(s, (coarse, None), (fine, None), reps)
    out["add_render_ms"] = add_render_ms(s, plain, more, reps)
    s.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=4200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps(dict(gpu=gpu_info(), c4=bench_c4(args.reps), heightfield=bench_heightfield(args.grid, args.reps))))


if __name__ == "__main__":
    main()

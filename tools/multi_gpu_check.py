"""Multi-GPU paths of the library on a real box (N >= 2 GPUs):
   torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/multi_gpu_check.py   # one process per GPU
   python tools/multi_gpu_check.py --group 2                                                                       # one process, 2 GPUs
Checks trb_render_sharded (interleaved and reference-style contiguous sharding, ONE ncclReduce per frame issued by libtrb) and
trb_group_render against the single-GPU render of the same frame: same ray counts, film equal up to float addition order. The
Adaptive cases (trb_render_sharded_adaptive, trb_group_render_adaptive) check the same against trb_render_adaptive on one GPU,
and that every pixel's sample count is equal. The AOV cases (trb_render_sharded_aov, trb_render_sharded_adaptive_aov,
trb_group_render_aov, trb_group_render_adaptive_aov) check the albedo and normal films the same way and nearest exactly, and the
denoise cases check a group's render_denoised and render_denoised_moments (denoised on replica 0) against one GPU's, within the
tolerance tests/test_multi_gpu_aov_gpu.py states."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402

W, H, SPP = 640, 360, 4
AD = (2, 16)  # Adaptive (min_spp, max_spp)
RAYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation"]


def desc():
    return SB.scene_c4(100_000, W, H, 64).finish()


def img(f):
    return f[..., :3] / np.maximum(f[..., 3:], 1e-6)


def aovs_close(a, b):
    """the AOV films up to float addition order, nearest exactly"""
    return (np.allclose(a["albedo_w"], b["albedo_w"], rtol=2e-4, atol=2e-5) and np.allclose(a["normal_w"], b["normal_w"], rtol=2e-4, atol=2e-5)
            and a["nearest"].tobytes() == b["nearest"].tobytes())


def group_aov_cases(g1, grp, n):
    ok = True
    ref, aref, st1 = g1.render_aov(spp=SPP, seed=3)
    film, aovs, st = grp.render_aov(spp=SPP, seed=3)
    good = st.rays_total() == st1.rays_total() and np.allclose(film, ref, rtol=2e-4, atol=2e-5) and aovs_close(aovs, aref)
    print(json.dumps({"mode": "trb_group_render_aov", "devices": n, "rays": st.rays_total(), "rays_single": st1.rays_total(),
                      "nearest_differs": int((aovs["nearest"] != aref["nearest"]).sum()), "ok": bool(good)}))
    ok = ok and good
    ref, aref, spp1, st1 = g1.render_adaptive_aov(*AD, seed=3)
    film, aovs, spp, st = grp.render_adaptive_aov(*AD, seed=3)
    good = (st.rays_total() == st1.rays_total() and bool((spp == spp1).all()) and np.allclose(film, ref, rtol=2e-4, atol=2e-5)
            and aovs_close(aovs, aref))
    print(json.dumps({"mode": "trb_group_render_adaptive_aov", "devices": n, "adaptive": AD, "pixels_with_other_count": int((spp != spp1).sum()),
                      "nearest_differs": int((aovs["nearest"] != aref["nearest"]).sum()), "ok": bool(good)}))
    ok = ok and good
    for name, call in (("render_denoised", lambda r, h: r.render_denoised(SPP, seed=3)),
                       ("render_denoised_moments", lambda r, h: r.render_denoised_moments(h, 1, seed=3))):
        want = call(g1, api.DenoiseHistory(g1))[0]
        got = call(grp, api.DenoiseHistory(grp.scene(0)))[0]
        good = bool(np.allclose(got, want, rtol=1e-4, atol=1e-5))
        print(json.dumps({"mode": "Group." + name, "devices": n, "max_abs_diff": float(np.abs(got - want).max()), "ok": good}))
        ok = ok and good
    return ok


def group_mode(n):
    g1 = api.Scene(desc(), 0)
    ref, st1 = g1.render(spp=SPP, seed=3)
    grp = api.Group(desc(), list(range(n)))
    film, st = grp.render(spp=SPP, seed=3)
    film2, _ = grp.render(spp=SPP, seed=3)            # a second frame through the same communicators
    ok = st.rays_total() == st1.rays_total() and st.camera_samples == st1.camera_samples and np.allclose(film, ref, rtol=2e-4, atol=2e-5) and np.allclose(film2, film, rtol=2e-4, atol=2e-5)
    print(json.dumps({"mode": "trb_group_render", "devices": n, "rays": st.rays_total(), "rays_single": st1.rays_total(),
                      "rmse": float(np.sqrt(np.mean((img(film) - img(ref)) ** 2))), "kernel_ms": st.kernel_ms, "kernel_ms_single": st1.kernel_ms, "ok": bool(ok)}))
    aref, aspp1, ast1 = g1.render_adaptive(*AD, seed=3)
    afilm, aspp, ast = grp.render_adaptive(*AD, seed=3)
    aok = bool((aspp == aspp1).all()) and [getattr(ast, k) for k in RAYS] == [getattr(ast1, k) for k in RAYS] and np.allclose(afilm, aref, rtol=2e-4, atol=2e-5)
    print(json.dumps({"mode": "trb_group_render_adaptive", "devices": n, "adaptive": AD, "rays": ast.rays_total(), "rays_single": ast1.rays_total(),
                      "pixels_with_other_count": int((aspp != aspp1).sum()), "rmse": float(np.sqrt(np.mean((img(afilm) - img(aref)) ** 2))),
                      "kernel_ms": ast.kernel_ms, "kernel_ms_single": ast1.kernel_ms, "ok": bool(aok)}))
    return ok and aok and group_aov_cases(g1, grp, n)


def rank_mode():
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")                      # plumbing only (ships the unique id, sums the counters)
    ids = [api.Comm.unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, 0)
    comm = api.Comm(ids[0], world, rank, local)
    g = api.Scene(desc(), local)
    ok = True
    for name, kw in (("interleaved", {}), ("contiguous (master.rs:91-93)", dict(shard_count=0xffffffff))):
        film, st = comm.render_sharded(g, None, 0, spp=SPP, seed=3, **kw)
        t = torch.tensor([st.rays_total(), st.camera_samples], dtype=torch.int64)
        dist.all_reduce(t)
        if rank == 0:
            ref, st1 = g.render(spp=SPP, seed=3)
            good = int(t[0]) == st1.rays_total() and int(t[1]) == st1.camera_samples and np.allclose(film, ref, rtol=2e-4, atol=2e-5)
            print(json.dumps({"mode": "trb_render_sharded " + name, "ranks": world, "rays": int(t[0]), "rays_single": st1.rays_total(),
                              "rmse": float(np.sqrt(np.mean((img(film) - img(ref)) ** 2))), "ok": bool(good)}))
            ok = ok and good
    for name, kw in (("interleaved", {}), ("contiguous (master.rs:91-93)", dict(shard_count=0xffffffff))):
        film, spp, st = comm.render_sharded_adaptive(g, *AD, None, None, 0, seed=3, **kw)
        t = torch.tensor([getattr(st, k) for k in RAYS], dtype=torch.int64)
        dist.all_reduce(t)
        counts = torch.from_numpy(spp.astype(np.int64))
        dist.all_reduce(counts)                          # each rank filled in its own pixels only
        if rank == 0:
            ref, spp1, st1 = g.render_adaptive(*AD, seed=3)
            good = t.tolist() == [getattr(st1, k) for k in RAYS] and bool((counts.numpy() == spp1).all()) and np.allclose(film, ref, rtol=2e-4, atol=2e-5)
            print(json.dumps({"mode": "trb_render_sharded_adaptive " + name, "ranks": world, "adaptive": AD, "rays": int(t[1:].sum()),
                              "rays_single": st1.rays_total(), "pixels_with_other_count": int((counts.numpy() != spp1).sum()),
                              "rmse": float(np.sqrt(np.mean((img(film) - img(ref)) ** 2))), "ok": bool(good)}))
            ok = ok and good
    for name, kw in (("interleaved", {}), ("contiguous (master.rs:91-93)", dict(shard_count=0xffffffff))):
        film, aovs, st = comm.render_sharded_aov(g, None, root=0, spp=SPP, seed=3, **kw)  # non-root ranks pass no buffers
        t = torch.tensor([st.rays_total()], dtype=torch.int64)
        dist.all_reduce(t)
        if rank == 0:
            ref, aref, st1 = g.render_aov(spp=SPP, seed=3)
            good = int(t[0]) == st1.rays_total() and np.allclose(film, ref, rtol=2e-4, atol=2e-5) and aovs_close(aovs, aref)
            print(json.dumps({"mode": "trb_render_sharded_aov " + name, "ranks": world, "nearest_differs": int((aovs["nearest"] != aref["nearest"]).sum()),
                              "ok": bool(good)}))
            ok = ok and good
        film, aovs, spp, st = comm.render_sharded_adaptive_aov(g, *AD, None, root=0, seed=3, **kw)
        counts = torch.from_numpy(spp.astype(np.int64))
        dist.all_reduce(counts)
        if rank == 0:
            ref, aref, spp1, st1 = g.render_adaptive_aov(*AD, seed=3)
            good = bool((counts.numpy() == spp1).all()) and np.allclose(film, ref, rtol=2e-4, atol=2e-5) and aovs_close(aovs, aref)
            print(json.dumps({"mode": "trb_render_sharded_adaptive_aov " + name, "ranks": world, "adaptive": AD,
                              "pixels_with_other_count": int((counts.numpy() != spp1).sum()), "ok": bool(good)}))
            ok = ok and good
    dist.barrier()
    comm.close()
    dist.destroy_process_group()
    return ok


if __name__ == "__main__":
    if "--group" in sys.argv:
        sys.exit(0 if group_mode(int(sys.argv[sys.argv.index("--group") + 1])) else 1)
    sys.exit(0 if rank_mode() else 1)

"""Ray-query throughput on one GPU: trb_intersect (k_intersect, one thread per ray), trb_intersect_records and trb_occluded (the
render's wavefront trace kernel) on the C4 workload (1 M triangles), device buffers, GPU time between CUDA events on one stream.
Then trb_illumination against trb_render_device on the same camera samples. Measures and reports; gates nothing.

    python tools/query_bench.py [--rays 4194304] [--reps 5] [--tris 1000000] [--width 1920 --height 1080] [--out results/query_bench.json]

The rays are incoherent: seeded origins uniform in the Cornell box and directions uniform on the sphere, as a render's bounce rays
are. trb_intersect has no per-ray time and returns (t, inst, prim); trb_intersect_records also builds the whole world-space
Intersection (96 bytes per ray); trb_occluded is timed in both shadow modes. The median of --reps timed calls after one warm-up.

trb_illumination takes the --width x --height camera rays of C4 at 1 spp (trb_camera_rays, key = pixel, sample = 0, clamped), the
camera samples trb_render_device renders at 1 spp with the same seed, so the two compute the same radiance and differ in what
they start from (caller rays vs. the camera) and end with (per-ray means vs. the film). Both report camera samples/s and Mrays/s
over every traced ray (primary, shadow, MIS, continuation).

Last, the five shading queries (trb_bsdf_eval, trb_bsdf_sample, trb_light_sample, trb_light_pdf, trb_emitted; device forms) on the
records of those camera rays and on --rays synthetic records on the material zoo: Mqueries/s and the GB/s of the query, record and
output bytes, with their share of the H100 SXM's 3.35 TB/s HBM3 peak.

Then trb_film_write_device on C4's whole-frame camera samples (--width x --height at --film-spp, trb_render_samples with the regions
of sample_regions()) into a device film: the whole call between CUDA events, and its two phases from torch.profiler's kernel
times (sort = k_film_keys + CUB's radix sort + k_film_starts; gather = k_film_gather). Last, the worst case the order contract
allows: 2^20 samples that all name one region, so each of that region's pixels sums them serially.
--sections film runs only this part.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api, scenebuild as SB  # noqa: E402


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=1 << 22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--film-spp", type=int, default=8)
    ap.add_argument("--sections", default="all", choices=["all", "film"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.sections == "film":
        res = {"device": device_info()}
        film_writes(a, res)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            json.dump(res, open(a.out, "w"), indent=1)
        return
    import torch as T
    dev = T.device("cuda:0")
    g = api.Scene(SB.scene_c4(a.tris, 64, 64, 1).finish())
    g.update_frame(0, 0.0, 0.0)
    rng = np.random.default_rng(0x0C4)
    q = np.zeros(a.rays, F.QUERY_RAY_DTYPE)
    q["o"] = rng.uniform((-14, 1, -10), (14, 23, 18), size=(a.rays, 3))
    d = rng.normal(size=(a.rays, 3))
    q["d"] = d / np.linalg.norm(d, axis=1, keepdims=True)
    q["max_t"] = np.inf
    r = np.zeros(a.rays, F.RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        r[k] = q[k]
    d_q = T.from_numpy(q.view(np.uint8).copy()).to(dev)
    d_r = T.from_numpy(r.view(np.uint8).copy()).to(dev)
    d_hits = T.empty(a.rays * 16, dtype=T.uint8, device=dev)
    d_rec = T.empty(a.rays * F.INTERSECTION_DTYPE.itemsize, dtype=T.uint8, device=dev)
    d_occ = T.empty(a.rays, dtype=T.uint8, device=dev)
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    n = a.rays
    cases = {
        "trb_intersect (k_intersect)": lambda: g.intersect_device(n, d_r.data_ptr(), d_hits.data_ptr(), None, s.cuda_stream),
        "trb_intersect_records": lambda: g.intersect_records_device(n, d_q.data_ptr(), d_rec.data_ptr(), None, s.cuda_stream),
        "trb_occluded (any hit)": lambda: g.occluded_device(n, d_q.data_ptr(), d_occ.data_ptr(), None, s.cuda_stream),
        "trb_occluded (reference closest hit)": lambda: g.occluded_device(n, d_q.data_ptr(), d_occ.data_ptr(), None, s.cuda_stream, reference=True),
    }
    res = {"device": device_info(), "rays": n, "triangles": a.tris, "reps": a.reps, "mrays_per_s": {}, "ms": {}}
    for name, call in cases.items():
        call()  # warm-up (and the first query call grows the path state)
        s.synchronize()
        ms = []
        for _ in range(a.reps):
            e0, e1 = T.cuda.Event(enable_timing=True), T.cuda.Event(enable_timing=True)
            e0.record(s)
            call()
            e1.record(s)
            s.synchronize()
            ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        res["ms"][name] = med
        res["mrays_per_s"][name] = n / med / 1e3
    g.check_error()
    hits = np.frombuffer(d_hits.cpu().numpy().tobytes(), F.HIT_DTYPE)
    rec = np.frombuffer(d_rec.cpu().numpy().tobytes(), F.INTERSECTION_DTYPE)
    res["hit_fraction"] = float((hits["inst"] != F.MISS).mean())
    res["records_match_trb_intersect"] = bool(rec["t"].tobytes() == hits["t"].tobytes() and (rec["inst"] == hits["inst"]).all())
    print("device: %s   %d incoherent rays on C4 (%d triangles), median of %d" % (res["device"], n, a.tris, a.reps))
    for name in cases:
        print("  %-40s %8.3f ms  %8.1f Mrays/s" % (name, res["ms"][name], res["mrays_per_s"][name]))
    print("  hit fraction %.3f, records equal trb_intersect's (t, inst): %s" % (res["hit_fraction"], res["records_match_trb_intersect"]))
    illumination_vs_render(a, res)
    shading_queries(a, res)
    film_writes(a, res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


def illumination_vs_render(a, res):
    import torch as T
    dev = T.device("cuda:0")
    g = api.Scene(SB.scene_c4(a.tris, a.width, a.height, 1).finish())
    g.update_frame(0, 0.0, 0.0)
    rays, _ = g.camera_rays(seed=1)
    blocks = g.block_list().astype(np.int64)
    i = np.arange(len(rays))
    item, pix = i // 64, i % 64
    q = np.zeros(len(rays), F.ILLUM_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        q[k] = rays[k]
    q["key"] = (blocks[item, 1] * 8 + pix // 8) * g.width + blocks[item, 0] * 8 + pix % 8
    n = len(q)
    d_q = T.from_numpy(q.view(np.uint8).copy()).to(dev)
    d_rgb = T.empty(n * 3, dtype=T.float32, device=dev)
    d_film = T.zeros(a.width * a.height * 4, dtype=T.float32, device=dev)
    d_st = T.zeros(9, dtype=T.int64, device=dev)
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    cases = {
        "trb_illumination (camera rays, 1 spp)": lambda st: g.illumination_device(n, d_q.data_ptr(), d_rgb.data_ptr(), spp=1, seed=1, clamp=True,
                                                                               d_stats=st, stream=s.cuda_stream),
        "trb_render_device (1 spp)": lambda st: g.render_device(d_film.data_ptr(), st, s.cuda_stream, seed=1, spp=1),
    }
    res["illumination"] = {"camera_samples": n, "width": a.width, "height": a.height, "ms": {}, "samples_per_s": {}, "mrays_per_s": {}}
    for name, call in cases.items():
        d_st.zero_()
        call(d_st.data_ptr())  # warm-up, and one call's ray counts
        s.synchronize()
        st = F.Stats.from_buffer_copy(d_st.cpu().numpy().tobytes())
        ms = []
        for _ in range(a.reps):
            e0, e1 = T.cuda.Event(enable_timing=True), T.cuda.Event(enable_timing=True)
            e0.record(s)
            call(None)
            e1.record(s)
            s.synchronize()
            ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        r = res["illumination"]
        r["ms"][name] = med
        r["samples_per_s"][name] = st.camera_samples / med * 1e3
        r["mrays_per_s"][name] = st.rays_total() / med / 1e3
    g.check_error()
    print("  %d camera samples of C4 at %dx%d, 1 spp:" % (n, a.width, a.height))
    for name in cases:
        r = res["illumination"]
        print("  %-40s %8.3f ms  %8.2f M samples/s  %8.1f Mrays/s" % (name, r["ms"][name], r["samples_per_s"][name] / 1e6, r["mrays_per_s"][name]))


HBM_PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3
# bytes each query moves: its query, its record (BSDF queries) and its output
SHADING_BYTES = {"trb_bsdf_eval": 32 + 96 + 16, "trb_bsdf_sample": 32 + 96 + 32, "trb_light_sample": 32 + 80, "trb_light_pdf": 32 + 4,
                 "trb_emitted": 32 + 12}


def _unit(v):
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def shading_inputs(g, rec, d, rng):
    """the five queries' inputs at records rec seen along directions d: wo = -d, random wi, u and lights"""
    n = len(rec)
    lights = g.lights()
    eq = np.zeros(n, F.BSDF_EVAL_QUERY_DTYPE)
    eq["wo"], eq["wi"], eq["bxdf"] = -d, _unit(rng.normal(size=(n, 3))), F.BXDF_ALL
    sq = np.zeros(n, F.BSDF_SAMPLE_QUERY_DTYPE)
    sq["wo"], sq["bxdf"], sq["u"], sq["u_comp"] = -d, F.BXDF_ALL, rng.random((n, 2)), rng.random(n)
    lq = np.zeros(n, F.LIGHT_QUERY_DTYPE)
    lq["p"], lq["u"], lq["light"], lq["time"] = rec["p"], rng.random((n, 2)), lights[rng.integers(0, len(lights), n)], rec["time"]
    pq = np.zeros(n, F.LIGHT_PDF_QUERY_DTYPE)
    pq["p"], pq["wi"], pq["light"], pq["time"] = rec["p"], eq["wi"], lq["light"], rec["time"]
    mq = np.zeros(n, F.EMIT_QUERY_DTYPE)
    mq["w"], mq["n"], mq["inst"], mq["time"] = -d, rec["ng"], rec["inst"], rec["time"]
    return {"trb_bsdf_eval": eq, "trb_bsdf_sample": sq, "trb_light_sample": lq, "trb_light_pdf": pq, "trb_emitted": mq}


def time_shading(g, rec, inputs, reps, T):
    """median device time (CUDA events, one stream) of each _device query over the inputs, after one warm-up call"""
    dev = T.device("cuda:0")
    n = len(rec)
    up = lambda a: T.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev)  # noqa: E731
    d_rec = up(rec)
    d_in = {k: up(v) for k, v in inputs.items()}
    d_out = {k: T.empty(n * size, dtype=T.uint8, device=dev) for k, size in (("trb_bsdf_eval", 16), ("trb_bsdf_sample", 32), ("trb_light_sample", 80),
                                                                             ("trb_light_pdf", 4), ("trb_emitted", 12))}
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    st = s.cuda_stream
    calls = {
        "trb_bsdf_eval": lambda: g.bsdf_eval_device(n, d_rec.data_ptr(), d_in["trb_bsdf_eval"].data_ptr(), d_out["trb_bsdf_eval"].data_ptr(), st),
        "trb_bsdf_sample": lambda: g.bsdf_sample_device(n, d_rec.data_ptr(), d_in["trb_bsdf_sample"].data_ptr(), d_out["trb_bsdf_sample"].data_ptr(), st),
        "trb_light_sample": lambda: g.light_sample_device(n, d_in["trb_light_sample"].data_ptr(), d_out["trb_light_sample"].data_ptr(), st),
        "trb_light_pdf": lambda: g.light_pdf_device(n, d_in["trb_light_pdf"].data_ptr(), d_out["trb_light_pdf"].data_ptr(), st),
        "trb_emitted": lambda: g.emitted_device(n, d_in["trb_emitted"].data_ptr(), d_out["trb_emitted"].data_ptr(), st),
    }
    out = {}
    for name, call in calls.items():
        call()
        s.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = T.cuda.Event(enable_timing=True), T.cuda.Event(enable_timing=True)
            e0.record(s)
            call()
            e1.record(s)
            s.synchronize()
            ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        gbs = n * SHADING_BYTES[name] / med / 1e6
        out[name] = {"ms": med, "mqueries_per_s": n / med / 1e3, "gb_per_s": gbs, "hbm_fraction": gbs / HBM_PEAK_GBS}
    return out


def shading_queries(a, res):
    """The shading queries on two workloads: the records of C4's --width x --height camera rays (1 spp; every surface matte, 1 M
    triangles), and --rays synthetic records on the material zoo (every material kind and a MERL table, random frames)."""
    import torch as T
    dev = T.device("cuda:0")
    rng = np.random.default_rng(0x5AD)
    res["shading"] = {}
    # C4 camera rays -> records on the device
    g = api.Scene(SB.scene_c4(a.tris, a.width, a.height, 1).finish())
    g.update_frame(0, 0.0, 0.0)
    rays, _ = g.camera_rays(seed=1)
    q = np.zeros(len(rays), F.QUERY_RAY_DTYPE)
    for k in ("o", "d", "min_t", "max_t"):
        q[k] = rays[k]
    n = len(q)
    d_q = T.from_numpy(q.view(np.uint8).copy()).to(dev)
    d_rec = T.empty(n * F.INTERSECTION_DTYPE.itemsize, dtype=T.uint8, device=dev)
    g.intersect_records_device(n, d_q.data_ptr(), d_rec.data_ptr())
    rec = np.frombuffer(d_rec.cpu().numpy().tobytes(), F.INTERSECTION_DTYPE).copy()
    res["shading"]["c4_camera"] = {"queries": n, "hit_fraction": float((rec["inst"] != F.MISS).mean()),
                                   "results": time_shading(g, rec, shading_inputs(g, rec, q["d"], rng), a.reps, T)}
    del g
    # synthetic records on the material zoo
    desc = SB.scene_materials_zoo(64, 64, 1, SB.synthetic_merl_table()).finish()
    z = api.Scene(desc)
    z.update_frame(0, 0.0, 0.0)
    m = a.rays
    rec = np.zeros(m, F.INTERSECTION_DTYPE)
    rec["material"] = rng.integers(0, desc.n_materials, m)
    rec["p"] = rng.uniform((-14, 1, -10), (14, 23, 18), size=(m, 3))
    rec["n"] = _unit(rng.normal(size=(m, 3)))
    rec["ng"] = rec["n"]
    rec["dp_du"] = _unit(rng.normal(size=(m, 3)))
    rec["inst"] = rng.integers(0, desc.n_instances, m)
    d = _unit(rng.normal(size=(m, 3)))
    d = np.where(((d * rec["n"]).sum(1) > 0)[:, None], -d, d)  # seen from the front
    res["shading"]["zoo_synthetic"] = {"queries": m, "materials": int(desc.n_materials),
                                       "results": time_shading(z, rec, shading_inputs(z, rec, d, rng), a.reps, T)}
    for wl, r in res["shading"].items():
        print("  shading queries, %s (%d queries), median of %d:" % (wl, r["queries"], a.reps))
        for name, x in r["results"].items():
            print("  %-40s %8.3f ms  %8.1f Mqueries/s  %7.1f GB/s (%.1f%% of %.0f GB/s HBM)" % (name, x["ms"], x["mqueries_per_s"], x["gb_per_s"],
                                                                                           100 * x["hbm_fraction"], HBM_PEAK_GBS))


def time_film_write(call, s, reps, T):
    """median over reps of: the call's GPU time between CUDA events, and its sort / gather kernel times from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    call()  # warm-up: grows the scene's sort scratch
    s.synchronize()
    tot, sort, gather = [], [], []
    for _ in range(reps):
        e0, e1 = T.cuda.Event(enable_timing=True), T.cuda.Event(enable_timing=True)
        e0.record(s)
        call()
        e1.record(s)
        s.synchronize()
        tot.append(e0.elapsed_time(e1))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            s.synchronize()
        k = [(e.key, getattr(e, "device_time_total", 0.0) / 1e3) for e in prof.key_averages()]  # us -> ms
        gather.append(sum(ms for name, ms in k if "k_film_gather" in name))
        sort.append(sum(ms for name, ms in k if "k_film_keys" in name or "k_film_starts" in name or "cub" in name.lower()))
    return {"ms": float(np.median(tot)), "sort_ms": float(np.median(sort)), "gather_ms": float(np.median(gather))}


def film_writes(a, res):
    import torch as T
    dev = T.device("cuda:0")
    g = api.Scene(SB.scene_c4(a.tris, a.width, a.height, a.film_spp).finish())
    g.update_frame(0, 0.0, 0.0)
    samples, _ = g.render_samples(seed=1)
    regions = g.sample_regions()
    n = len(samples)
    d_s = T.from_numpy(samples.view(np.float32).reshape(-1, 5).copy()).to(dev)
    d_r = T.from_numpy(regions.view(np.int32).copy()).to(dev)
    d_film = T.zeros((g.height, g.width, 4), dtype=T.float32, device=dev)
    s = T.cuda.Stream()
    s.wait_stream(T.cuda.current_stream())
    frame = time_film_write(lambda: g.film_write_device(n, d_s.data_ptr(), d_r.data_ptr(), d_film.data_ptr(), s.cuda_stream), s, a.reps, T)
    frame.update(samples=n, msamples_per_s=n / frame["ms"] / 1e3)
    m = 1 << 20
    rng = np.random.default_rng(0xF1)
    one = np.zeros(m, F.SAMPLE_DTYPE)
    bx, by = (a.width // 16) * 8, (a.height // 16) * 8
    one["x"], one["y"] = rng.uniform(bx, bx + 8, m), rng.uniform(by, by + 8, m)
    for k in ("r", "g", "b"):
        one[k] = rng.uniform(0, 1, m)
    d_s1 = T.from_numpy(one.view(np.float32).reshape(-1, 5).copy()).to(dev)
    d_r1 = T.full((m,), (by // 8) * (a.width // 8) + bx // 8, dtype=T.int32, device=dev)
    single = time_film_write(lambda: g.film_write_device(m, d_s1.data_ptr(), d_r1.data_ptr(), d_film.data_ptr(), s.cuda_stream), s, a.reps, T)
    single.update(samples=m, msamples_per_s=m / single["ms"] / 1e3)
    g.check_error()
    res["film_write"] = {"c4_frame": frame, "one_region": single, "width": a.width, "height": a.height, "spp": a.film_spp}
    print("  trb_film_write_device, median of %d:" % a.reps)
    for name, x in (("C4 %dx%d, %d spp" % (a.width, a.height, a.film_spp), frame), ("one region", single)):
        print("  %-40s %8.3f ms (sort %.3f, gather %.3f)  %8.1f M samples/s  (%d samples)" % (name, x["ms"], x["sort_ms"], x["gather_ms"],
                                                                                            x["msamples_per_s"], x["samples"]))


if __name__ == "__main__":
    main()

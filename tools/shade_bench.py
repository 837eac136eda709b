"""Where a bench.py step goes, kernel by kernel: the C4 passes bench.py times (1M triangles, 1920 x 1080, --spp-per-step samples
per pixel per pass) under torch.profiler, with the per-round times of k_wf_trace and the split shade kernels k_wf_shade_a / _b / _c,
plus k_wf_generate and the film kernel. Per kernel: the mean over --steps profiled passes of its time per pass, and per bounce
round. Prints one JSON line with the GPU's name, power limit and SM clock, read in the same run.

    python tools/shade_bench.py [--steps 3] [--warmup 2] [--tris 1000000] [--spp-per-step 8]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import api, scenebuild as SB  # noqa: E402

GROUPS = ("k_wf_generate", "k_wf_trace", "k_wf_shade_a", "k_wf_shade_b", "k_wf_shade_c", "k_wf_film")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def group_of(name):
    for g in GROUPS:
        if g + "<" in name or g + "(" in name or name.endswith(g) or (g == "k_wf_film" and g in name):  # k_wf_film or k_wf_film_v2
            return g
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--tris", type=int, default=1_000_000)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--spp", type=int, default=4096)
    ap.add_argument("--spp-per-step", type=int, default=8)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise RuntimeError("shade_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"device": gpu_info(), "workload": "C4 %d triangles, %dx%d, %d spp per pass" % (a.tris, a.width, a.height, a.spp_per_step)}
    g = api.Scene(SB.scene_c4(a.tris, a.width, a.height, a.spp).finish(), 0)
    g.update_frame(0, 0.0, 0.0)
    film = torch.zeros((a.height, a.width, 4), dtype=torch.float32, device=dev)
    stats = torch.zeros(10, dtype=torch.int64, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)  # > the 50 MB L2 of an H100, as bench.py between passes
    stream = torch.cuda.current_stream().cuda_stream

    def step(i):
        flush.fill_(i & 0xFF)
        g.render_device(film.data_ptr(), stats.data_ptr(), stream, spp=a.spp, sample_first=i * a.spp_per_step,
                        sample_count=a.spp_per_step, seed=a.seed)

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(a.steps):
            step(a.warmup + k)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)

    # one pass = k_wf_generate, then per round a trace and its shade kernels, then the film; a trace launch opens a round
    total = {g_: 0.0 for g_ in GROUPS + ("other",)}
    rounds = {}  # (group, round) -> us summed over the passes
    rnd = -1
    names = {}
    for e in kern:
        grp = group_of(e.name)
        if grp == "other" and ("fill" in e.name or "elementwise" in e.name.lower()):
            continue  # the L2 flush between passes
        us = e.time_range.elapsed_us()
        if grp == "k_wf_generate":
            rnd = -1
        elif grp == "k_wf_trace":
            rnd += 1
        total[grp] += us
        names.setdefault(grp, set()).add(e.name.split("(")[0][:80])
        if grp in ("k_wf_trace", "k_wf_shade_a", "k_wf_shade_b", "k_wf_shade_c"):
            rounds[(grp, rnd)] = rounds.get((grp, rnd), 0.0) + us
    n = float(a.steps)
    shade = sum(total[k] for k in ("k_wf_shade_a", "k_wf_shade_b", "k_wf_shade_c")) / n
    step_ms = sum(total.values()) / n / 1e3
    out["ms_per_pass"] = {k: round(v / n / 1e3, 3) for k, v in total.items()}
    out["kernel_ms_per_pass"] = round(step_ms, 3)
    out["shade_ms_per_pass"] = round(shade / 1e3, 3)
    out["shade_share"] = round(shade / 1e3 / step_ms, 4) if step_ms > 0 else None
    n_rounds = 1 + max((r for (_, r) in rounds), default=-1)
    out["per_round_ms"] = {grp: [round(rounds.get((grp, r), 0.0) / n / 1e3, 3) for r in range(n_rounds)]
                           for grp in ("k_wf_trace", "k_wf_shade_a", "k_wf_shade_b", "k_wf_shade_c")}
    out["kernels"] = {k: sorted(v) for k, v in names.items()}
    out["device_after"] = gpu_info()
    g.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""The reference's path tracer written by a caller from the library's parts: Path::illumination (path.rs:45-119) with
sample_one_light and estimate_direct (integrator/mod.rs:106-169), in torch on device tensors. Every step is a batch query on the
render's own device code (intersect_records, occluded, bsdf_eval, bsdf_sample, light_sample, light_pdf, emitted, lights), enqueued on
the current torch stream; every random number is drawn with torch.rand / torch.randint. It keeps the reference's quirks: the emitted
term uses the first hit's geometric normal at every specular bounce (Q1), a BSDF sample the light's pdf rejects ends estimate_direct
with the light-sample term alone (Q7), and each path's samples come from its own stratified arrays (PathSamples). Its estimate has the
expectation of Scene.illumination's; only the random numbers differ.

    python examples/query_path.py [--scene tests/golden/scenes/c2_smallpt.json] [--width 128] [--height 128] [--spp 16]
                                  [--out query_path.png]
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api  # noqa: E402

MISS = -1  # TRB_MISS as int32
BX_NON_SPECULAR = F.BXDF_ALL & ~F.BXDF_SPECULAR
INF = float("inf")


class Parts:
    """The _device queries on device tensors, on the current torch stream. Queries and records are float32 rows whose integer fields
    are written and read through an int32 view of the same storage."""

    def __init__(self, scene):
        self.s = scene
        self.dev = torch.device("cuda", scene.device)
        self.lights = torch.from_numpy(scene.lights().astype(np.int32)).to(self.dev)

    def _st(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _rows(self, n, k):
        return torch.zeros((n, k), dtype=torch.float32, device=self.dev)

    def intersect(self, o, d, min_t, max_t, time):
        """Scene::intersect: (n, 24) trb_intersection rows (t, inst, prim, material, p, n, ng, u, v, time, dp_du, dp_dv, pad)"""
        n = o.shape[0]
        q = self._rows(n, 12)
        q[:, 0:3], q[:, 3:6], q[:, 6], q[:, 7], q[:, 8] = o, d, min_t, max_t, time
        rec = self._rows(n, 24)
        if n:
            self.s.intersect_records_device(n, q.data_ptr(), rec.data_ptr(), stream=self._st())
        return rec

    def occluded(self, shadow):
        n = shadow.shape[0]
        out = torch.zeros(n, dtype=torch.uint8, device=self.dev)
        if n:
            self.s.occluded_device(n, shadow.contiguous().data_ptr(), out.data_ptr(), stream=self._st())
        return out.bool()

    def bsdf_eval(self, rec, wo, wi, bxdf):
        n = rec.shape[0]
        q = self._rows(n, 8)
        q[:, 0:3], q[:, 4:7] = wo, wi
        q.view(torch.int32)[:, 3] = bxdf
        out = self._rows(n, 4)
        if n:
            self.s.bsdf_eval_device(n, rec.data_ptr(), q.data_ptr(), out.data_ptr(), stream=self._st())
        return out[:, 0:3], out[:, 3]

    def bsdf_sample(self, rec, wo, bxdf, u0, u1, uc):
        n = rec.shape[0]
        q = self._rows(n, 8)
        q[:, 0:3], q[:, 4], q[:, 5], q[:, 6] = wo, u0, u1, uc
        q.view(torch.int32)[:, 3] = bxdf
        out = self._rows(n, 8)
        if n:
            self.s.bsdf_sample_device(n, rec.data_ptr(), q.data_ptr(), out.data_ptr(), stream=self._st())
        return out[:, 0:3], out[:, 3], out[:, 4:7], out.view(torch.int32)[:, 7]

    def light_sample(self, p, time, u0, u1, light):
        n = p.shape[0]
        q = self._rows(n, 8)
        q[:, 0:3], q[:, 3], q[:, 4], q[:, 5] = p, time, u0, u1
        q.view(torch.int32)[:, 6] = light
        out = self._rows(n, 20)
        if n:
            self.s.light_sample_device(n, q.data_ptr(), out.data_ptr(), stream=self._st())
        return out[:, 0:3], out[:, 3], out[:, 4:7], out.view(torch.int32)[:, 7] != 0, out[:, 8:20]

    def light_pdf(self, p, time, wi, light):
        n = p.shape[0]
        q = self._rows(n, 8)
        q[:, 0:3], q[:, 3], q[:, 4:7] = p, time, wi
        q.view(torch.int32)[:, 7] = light
        out = torch.zeros(n, dtype=torch.float32, device=self.dev)
        if n:
            self.s.light_pdf_device(n, q.data_ptr(), out.data_ptr(), stream=self._st())
        return out

    def emitted(self, w, time, nrm, inst):
        n = w.shape[0]
        q = self._rows(n, 8)
        q[:, 0:3], q[:, 3], q[:, 4:7] = w, time, nrm
        q.view(torch.int32)[:, 7] = inst
        out = self._rows(n, 3)
        if n:
            self.s.emitted_device(n, q.data_ptr(), out.data_ptr(), stream=self._st())
        return out


def _black(c):
    return (c == 0).all(dim=1)


def _dot(a, b):
    return (a * b).sum(dim=1)


def _unit(v):
    return v / torch.linalg.vector_norm(v, dim=1, keepdim=True)


def _power(f, g):  # mc::power_heuristic with one sample each
    return f * f / (f * f + g * g)


def estimate_direct(parts, rec, wo, nrm, time, light, l0, l1, b0, b1, bc):
    """Integrator::estimate_direct (integrator/mod.rs:122-169) with BxDFType non-specular lobes"""
    p = rec[:, 4:7]
    li, pdf_l, wi, delta, shadow = parts.light_sample(p, time, l0, l1, light)
    cand = (pdf_l > 0) & ~_black(li)
    unocc = torch.zeros_like(cand)
    ci = torch.nonzero(cand).squeeze(1)
    unocc[ci] = ~parts.occluded(shadow[ci])
    f, pdf_b = parts.bsdf_eval(rec, wo, wi, BX_NON_SPECULAR)
    w = torch.where(delta, torch.ones_like(pdf_l), _power(pdf_l, pdf_b))
    a = f * li * (_dot(wi, nrm).abs() * w / pdf_l)[:, None]
    direct = torch.where((unocc & ~_black(f))[:, None], a, torch.zeros_like(a))
    # BSDF sampling (area lights only)
    f2, pdf2, wi2, sampled = parts.bsdf_sample(rec, wo, BX_NON_SPECULAR, b0, b1, bc)
    spec = (sampled & F.BXDF_SPECULAR) != 0
    pl = parts.light_pdf(p, time, wi2, light)
    go = ~delta & (pdf2 > 0) & ~_black(f2) & (spec | (pl != 0))  # pl == 0: `return direct_light` (Q7)
    w2 = torch.where(spec, torch.ones_like(pdf2), _power(pdf2, pl))
    gi = torch.nonzero(go).squeeze(1)
    hit = parts.intersect(p[gi], wi2[gi], 0.001, INF, time[gi])
    lr = parts.emitted(-wi2[gi], time[gi], hit[:, 10:13], light[gi])
    lr = torch.where((hit.view(torch.int32)[:, 1] == light[gi])[:, None], lr, torch.zeros_like(lr))  # the MIS ray hit this light
    b = f2[gi] * lr * (_dot(wi2[gi], nrm[gi]).abs() * w2[gi] / pdf2[gi])[:, None]
    direct[gi] += torch.where(_black(lr)[:, None], torch.zeros_like(b), b)
    return direct


class PathSamples:
    """The per-path sample arrays of Path::illumination (path.rs:48-60): three 2-D arrays (light, BSDF and path direction samples) and
    three 1-D arrays (light, BSDF and path component choices) of max_depth + 1 entries each, entry b used at bounce b. The reference
    fills each with LowDiscrepancy::get_samples_2d / _1d (ld.rs:33-64, 91-119): the first max_depth + 1 points of a (0, 2) sequence
    (van der Corput, Sobol) under a random XOR scramble, shuffled. One path's bounces therefore see stratified, not independent,
    numbers, and its estimate depends on that, so these arrays are kept here; their scrambles and shuffles come from torch."""

    def __init__(self, n, length, gen, dev):
        rev = [int("{:032b}".format(i)[::-1], 2) for i in range(length)]  # van der Corput: the index bit-reversed
        sob = []
        for i in range(length):  # Sobol: the XOR of the generator columns of the index's set bits
            v, c, k = 0, 1 << 31, i
            while k:
                if k & 1:
                    v ^= c
                k >>= 1
                c ^= c >> 1
            sob.append(v)
        self.rev = torch.tensor(rev, dtype=torch.int64, device=dev)
        self.sob = torch.tensor(sob, dtype=torch.int64, device=dev)
        self.perm = torch.rand((n, 6, length), generator=gen, device=dev).argsort(dim=2)  # the shuffles
        self.scr = torch.randint(0, 1 << 32, (n, 9), generator=gen, device=dev, dtype=torch.int64)  # the scrambles

    @staticmethod
    def _f32(bits):  # ld.rs:91-119: the top 24 bits as a float, at most 1 - f32::EPSILON
        return torch.clamp(((bits >> 8) & 0xFFFFFF).float() / float(1 << 24), max=1.0 - 2.0 ** -23)

    def subset(self, k):
        self.perm, self.scr = self.perm[k], self.scr[k]

    def at(self, b):
        """bounce b's l0 l1 b0 b1 lc bc p0 p1 pc as an (n, 9) tensor"""
        i, s = self.perm[:, :, b], self.scr
        v = lambda a, c: self._f32(self.rev[i[:, a]] ^ s[:, c])  # noqa: E731
        w = lambda a, c: self._f32(self.sob[i[:, a]] ^ s[:, c])  # noqa: E731
        return torch.stack([v(0, 0), w(0, 1), v(1, 2), w(1, 3), v(3, 6), v(4, 7), v(2, 4), w(2, 5), v(5, 8)], dim=1)


def illumination(parts, o, d, time, min_depth, max_depth, gen):
    """Scene::intersect then Path::illumination for each ray (o, d) at `time`: one sample per ray, (n, 3) float32 radiance (black on a
    miss). gen: the torch.Generator every random number is drawn from."""
    n, dev = o.shape[0], parts.dev
    L = torch.zeros((n, 3), dtype=torch.float32, device=dev)
    rec = parts.intersect(o, d, 0.0, INF, time)
    idx = torch.nonzero(rec.view(torch.int32)[:, 1] != MISS).squeeze(1)
    rec, ray_d, time = rec[idx], d[idx], time[idx]
    first_ng = rec[:, 10:13]  # the first hit's ng: the emitted term uses it at every bounce (Q1)
    thr = torch.ones((len(idx), 3), dtype=torch.float32, device=dev)
    spec = torch.ones(len(idx), dtype=torch.bool, device=dev)  # bounce 0 counts emission like a specular bounce
    ps = PathSamples(len(idx), max_depth + 1, gen, dev)
    nl = len(parts.lights)
    for bounce in range(max_depth + 1):
        m = len(idx)
        if m == 0:
            break
        inst = rec.view(torch.int32)[:, 1]
        wo = -ray_d
        e = parts.emitted(wo, time, first_ng, inst)  # black for receivers
        L.index_add_(0, idx, torch.where(spec[:, None], thr * e, torch.zeros_like(e)))
        u = ps.at(bounce)  # l0 l1 b0 b1 lc bc p0 p1 pc
        light = parts.lights[torch.clamp((u[:, 4] * nl).long(), max=nl - 1)]  # sample_one_light: no x n_lights weight (Q2)
        nrm = _unit(rec[:, 7:10])  # bsdf.n
        L.index_add_(0, idx, thr * estimate_direct(parts, rec, wo, nrm, time, light, u[:, 0], u[:, 1], u[:, 2], u[:, 3], u[:, 5]))
        f, pdf, wi, sampled = parts.bsdf_sample(rec, wo, F.BXDF_ALL, u[:, 6], u[:, 7], u[:, 8])
        ok = ~_black(f) & (pdf != 0)
        spec = (sampled & F.BXDF_SPECULAR) != 0
        thr = thr * f * (_dot(wi, nrm).abs() / pdf)[:, None]
        if bounce > min_depth:  # Russian roulette (Q8)
            cont = torch.clamp(0.2126 * thr[:, 0] + 0.7152 * thr[:, 1] + 0.0722 * thr[:, 2], min=0.5)
            ok &= ~(torch.rand(m, generator=gen, device=dev) > cont)
            thr = thr / cont[:, None]
        if bounce == max_depth:
            break
        k = torch.nonzero(ok).squeeze(1)
        p, d2 = rec[k, 4:7], _unit(wi[k])
        rec = parts.intersect(p, d2, 0.001, INF, time[k])  # ray.child
        h = torch.nonzero(rec.view(torch.int32)[:, 1] != MISS).squeeze(1)
        k = k[h]
        idx, rec, ray_d, time, first_ng, thr, spec = idx[k], rec[h], d2[h], time[k], first_ng[k], thr[k], spec[k]
        ps.subset(k)
    return L


def render_rays(scene, rays, spp, seed, min_depth, max_depth, clamp=False):
    """Mean of spp samples of illumination() per trb_ray (rays at time 0); each sample clamped to [0, 1] first with clamp=True, as the
    render does. Returns (n, 3) float32 numpy."""
    parts = Parts(scene)
    dev = parts.dev
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    o = torch.from_numpy(np.ascontiguousarray(rays["o"])).to(dev).repeat_interleave(spp, dim=0)
    d = torch.from_numpy(np.ascontiguousarray(rays["d"])).to(dev).repeat_interleave(spp, dim=0)
    time = torch.zeros(len(o), dtype=torch.float32, device=dev)
    c = illumination(parts, o, d, time, min_depth, max_depth, gen)
    if clamp:
        c = c.clamp(0.0, 1.0)
    return c.view(len(rays), spp, 3).mean(dim=1).cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default=os.path.join(REPO, "tests", "golden", "scenes", "c2_smallpt.json"))
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--height", type=int, default=128)
    ap.add_argument("--spp", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="query_path.png")
    a = ap.parse_args()
    lib = F.load_trb()
    desc = C.POINTER(F.SceneDesc)()
    if lib.trb_desc_load_json(a.scene.encode(), a.width, a.height, 1, C.byref(desc)) != F.TRB_OK:
        raise SystemExit(lib.trb_last_error().decode())
    scene = api.Scene(desc.contents)
    scene.update_frame(0, 0.0, 0.0)  # shutter [0, 0]: every camera ray's time is 0
    rays, xy = scene.camera_rays(spp=1)  # one ray per pixel, in block order, with its film position
    integ = desc.contents.integrator
    rgb = render_rays(scene, rays, a.spp, a.seed, integ.min_depth, integ.max_depth, clamp=True)
    film = np.zeros((scene.height, scene.width, 4), np.float32)
    px = np.floor(xy).astype(np.int64)
    film[px[:, 1], px[:, 0], :3] = rgb
    film[px[:, 1], px[:, 0], 3] = 1.0
    img = scene.to_srgb8(film)
    if lib.trb_write_png(a.out.encode(), F.ptr(img), scene.width, scene.height) != F.TRB_OK:
        raise SystemExit(lib.trb_last_error().decode())
    print("%s: %dx%d at %d spp" % (a.out, scene.width, scene.height, a.spp))


if __name__ == "__main__":
    main()

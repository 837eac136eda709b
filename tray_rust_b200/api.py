"""Python host side above the C ABI.

``Scene`` wraps a ``trb_scene`` (GPU, product). The CPU oracle's wrapper with the same methods
(``oracle.pyoracle.OracleScene``) is test infrastructure and lives outside this package.

The reference-shaped mirror (``Config``, ``RenderTarget``, ``Exec.render`` with the argument
meaning of /root/reference/src/exec/mod.rs:17-49) lives in ``tray_rust_b200.exec``.
"""
import ctypes as C

import numpy as np

from . import _ffi as F


class TrbError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("trb status %d: %s" % (status, msg))
        self.status = status


def _cfg(spp=0, sample_first=0, sample_count=0, block_start=0, block_count=0, current_frame=0, seed=1, flags=0,
         shard_index=0, shard_count=0, shard_chunk=0):
    return F.RenderCfg(spp, sample_first, sample_count, block_start, block_count, current_frame, seed, flags,
                       shard_index, shard_count, shard_chunk)


def adaptive_schedule(min_spp, max_spp):
    """trb_adaptive_schedule: Adaptive::new's rounded (min, max, step) and the largest per-pixel sample count."""
    lib = F.load_trb()
    out = [F.u32() for _ in range(4)]
    rc = lib.trb_adaptive_schedule(C.byref(F.Adaptive(min_spp, max_spp)), *(C.byref(x) for x in out))
    if rc != F.TRB_OK:
        raise TrbError(rc, (lib.trb_last_error() or b"").decode())
    return tuple(x.value for x in out)


def film_to_srgb8(film):
    """trb_host_film_to_srgb8: Image::get_srgb8 of an RGBW film of shape (height, width, 4) on the host, without a scene or a GPU.
    Returns (height, width, 3) uint8, the same bytes as Scene.to_srgb8 of the same film."""
    film = np.ascontiguousarray(film, dtype=np.float32)
    if film.ndim != 3 or film.shape[2] != 4:
        raise ValueError("film must have shape (height, width, 4)")
    lib = F.load_trb()
    out = np.zeros(film.shape[:2] + (3,), np.uint8)
    rc = lib.trb_host_film_to_srgb8(film.shape[1], film.shape[0], F.ptr(film), F.ptr(out))
    if rc != F.TRB_OK:
        raise TrbError(rc, (lib.trb_last_error() or b"").decode())
    return out


def build_bvh(boxes, max_geom, device=0):
    """trb_build_bvh: BVH::new over boxes of shape (n, 6) (min xyz, max xyz) with the reference's SAH build, run on GPU `device`.
    Returns (nodes as NODE_DTYPE, ordered_geom as uint32), the bytes trb_host_build_bvh returns."""
    boxes = np.ascontiguousarray(boxes, dtype=np.float32).reshape(-1, 6)
    lib = F.load_trb()
    nn = F.u32()
    rc = lib.trb_build_bvh(device, F.ptr(boxes), len(boxes), max_geom, C.byref(nn), None, None)
    if rc == F.TRB_OK:
        nodes = np.zeros(nn.value, F.NODE_DTYPE)
        order = np.zeros(len(boxes), np.uint32)
        rc = lib.trb_build_bvh(device, F.ptr(boxes), len(boxes), max_geom, C.byref(nn), F.ptr(nodes), F.ptr(order))
    if rc != F.TRB_OK:
        raise TrbError(rc, (lib.trb_last_error() or b"").decode())
    return nodes, order


def build_bvh_device(d_boxes, n, max_geom, d_n_nodes, d_nodes, d_ordered, device=0, stream=None):
    """trb_build_bvh_device: the same build over DEVICE buffers (pointers as ints): d_nodes with room for 2n - 1 nodes, d_ordered
    for n uint32, and the node count written to the device word d_n_nodes. Enqueued on `stream` (a cudaStream_t as an int, e.g.
    torch.cuda.Stream().cuda_stream; None = default stream), which it synchronises once per level of large nodes."""
    lib = F.load_trb()
    rc = lib.trb_build_bvh_device(device, d_boxes, n, max_geom, d_n_nodes, d_nodes, d_ordered, stream)
    if rc != F.TRB_OK:
        raise TrbError(rc, (lib.trb_last_error() or b"").decode())


def decode_nearest(nearest):
    """The (depth float32, inst uint32) of a ``nearest`` AOV buffer: its high and low 32 bits (trb_aov_film)."""
    nearest = np.ascontiguousarray(nearest, dtype=np.uint64)
    return (nearest >> np.uint64(32)).astype(np.uint32).view(np.float32), (nearest & np.uint64(0xffffffff)).astype(np.uint32)


def decode_motion(motion_w):
    """The (height, width, 2) float32 motion in pixels of a ``motion_w`` film (include/trb.h "Motion vectors"): its first two
    channels over its third where that is positive, NaN elsewhere."""
    motion_w = np.asarray(motion_w, dtype=np.float32)
    z = motion_w[..., 2:3]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(z > 0, motion_w[..., :2] / z, np.float32(np.nan)).astype(np.float32)


def _denoise_params(params):
    unknown = set(params) - set(F.DENOISE_DEFAULTS)
    if unknown:
        raise TypeError("unknown denoise parameters: %s" % sorted(unknown))
    p = dict(F.DENOISE_DEFAULTS, **params)
    return F.DenoiseParams(p["iterations"], p["normal_power"], p["sigma_luminance"], p["sigma_depth"])


def _temporal_params(params):
    unknown = set(params) - set(F.DENOISE_DEFAULTS) - set(F.DENOISE_TEMPORAL_DEFAULTS)
    if unknown:
        raise TypeError("unknown temporal denoise parameters: %s" % sorted(unknown))
    t = dict(F.DENOISE_TEMPORAL_DEFAULTS, **{k: v for k, v in params.items() if k in F.DENOISE_TEMPORAL_DEFAULTS})
    spatial = _denoise_params({k: v for k, v in params.items() if k in F.DENOISE_DEFAULTS})
    return F.DenoiseTemporalParams(spatial, t["max_history"], t["depth_tolerance"], t["normal_threshold"], 0)


def _gradient_params(params):
    unknown = set(params) - set(F.DENOISE_DEFAULTS) - set(F.DENOISE_TEMPORAL_DEFAULTS) - set(F.DENOISE_GRADIENT_DEFAULTS)
    if unknown:
        raise TypeError("unknown temporal gradient denoise parameters: %s" % sorted(unknown))
    g = dict(F.DENOISE_GRADIENT_DEFAULTS, **{k: v for k, v in params.items() if k in F.DENOISE_GRADIENT_DEFAULTS})
    temporal = _temporal_params({k: v for k, v in params.items() if k not in F.DENOISE_GRADIENT_DEFAULTS})
    return F.DenoiseGradientParams(temporal, g["gradient_iterations"])


class DenoiseHistory:
    """trb_denoise_history (DESIGN.md §4 "Temporal denoising"): the per-pixel history and frame snapshot of one scene's temporal
    denoise. Empty when created and after reset(); close() (or the scene's close) releases it."""

    def __init__(self, scene):
        self._lib = scene._lib
        self._scene = scene
        h = C.c_void_p()
        scene._check(self._lib.trb_denoise_history_create(scene._h, C.byref(h)))
        self._h = h
        scene._histories.append(self)

    def reset(self):
        self._scene._check(self._lib.trb_denoise_history_reset(self._h))

    def close(self):
        if self._h is not None:
            self._lib.trb_denoise_history_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Base:
    """Shared helpers; subclasses provide self._lib, self._h, self._pfx and self._check."""

    def _n_selected_blocks(self, cfg):
        nb = self.n_blocks(cfg.block_start, cfg.block_count)
        if cfg.shard_count > 1:
            ch = max(1, cfg.shard_chunk)
            nb = sum(1 for j in range(nb) if (j // ch) % cfg.shard_count == cfg.shard_index)
        return nb

    def _n_samples(self, cfg):
        nb = self.n_blocks(cfg.block_start, cfg.block_count)
        if cfg.shard_count > 1:
            ch = max(1, cfg.shard_chunk)
            nb = sum(1 for j in range(nb) if (j // ch) % cfg.shard_count == cfg.shard_index)
        spp = self.spp if cfg.spp == 0 else 1 << (max(1, cfg.spp) - 1).bit_length()
        cnt = cfg.sample_count if cfg.sample_count else spp - cfg.sample_first
        return nb * 64 * cnt

    def n_blocks(self, start=0, count=0):
        n = F.u32()
        self._check(getattr(self._lib, self._pfx + "block_list")(self._h, start, count, C.byref(n), None, 0))
        return n.value

    def block_list(self, start=0, count=0):
        n = self.n_blocks(start, count)
        xy = np.zeros((n, 2), np.uint32)
        m = F.u32()
        self._check(getattr(self._lib, self._pfx + "block_list")(self._h, start, count, C.byref(m), F.ptr(xy), n))
        return xy

    def sample_regions(self, **kw):
        """The region (8x8 block index by * (width / 8) + bx) of every camera sample of the selection, in the order of
        render_samples / camera_rays: what film_write needs to write those samples as the render does."""
        cfg = _cfg(**kw)
        xy = self.block_list(cfg.block_start, cfg.block_count)
        if cfg.shard_count > 1:
            ch = max(1, cfg.shard_chunk)
            xy = xy[[(j // ch) % cfg.shard_count == cfg.shard_index for j in range(len(xy))]]
        per_block = self._n_samples(cfg) // max(1, len(xy))
        return np.repeat(xy[:, 1] * np.uint32(self.width // 8) + xy[:, 0], per_block).astype(np.uint32)

    def bvh(self, which=-1):
        nn, no = F.u32(), F.u32()
        f = getattr(self._lib, self._pfx + "scene_get_bvh")
        self._check(f(self._h, which, C.byref(nn), None, C.byref(no), None))
        nodes = np.zeros(nn.value, F.NODE_DTYPE)
        order = np.zeros(no.value, np.uint32)
        self._check(f(self._h, which, C.byref(nn), F.ptr(nodes), C.byref(no), F.ptr(order)))
        return nodes, order

    def transform(self, inst):
        m, i = np.zeros(16, np.float32), np.zeros(16, np.float32)
        self._check(getattr(self._lib, self._pfx + "scene_get_transform")(self._h, inst, F.ptr(m), F.ptr(i)))
        return m.reshape(4, 4), i.reshape(4, 4)

    def filter_table(self):
        t = np.zeros(256, np.float32)
        self._check(getattr(self._lib, self._pfx + "scene_get_filter_table")(self._h, F.ptr(t)))
        return t.reshape(16, 16)

    def update_frame(self, frame=0, start=0.0, end=0.0):
        self._check(getattr(self._lib, self._pfx + "scene_update_frame")(self._h, frame, start, end))


def _render_halves(render_aov, scene_spp, spp, name, kw):
    """The two half renders of a denoised frame: samples [0, n/2) and [n/2, n) of n = spp (0: scene_spp) rounded up to a power of
    two, into two films, with the AOVs accumulated over both. Returns (a, b, aovs, (stats_a, stats_b))."""
    n = 1
    while n < (spp or scene_spp):
        n *= 2
    if n < 2:
        raise ValueError("a denoised render needs at least 2 samples per pixel (two half renders); got %d" % (spp or scene_spp))
    for k in ("spp", "sample_first", "sample_count"):
        if k in kw:
            raise ValueError("%s chooses %s itself" % (name, k))
    half = n // 2
    a, aovs, st_a = render_aov(spp=n, sample_first=0, sample_count=half, **kw)
    kw["flags"] = kw.get("flags", 0) | F.RENDER_NO_UPDATE  # the first half set the frame
    b, _, st_b = render_aov(albedo=aovs["albedo_w"], normal=aovs["normal_w"], nearest=aovs["nearest"], spp=n, sample_first=half,
                            sample_count=half, **kw)
    return a, b, aovs, (st_a, st_b)


# The bodies of the denoised renders, shared by Scene (its own render_aov) and Group (the group's AOV render, denoised on replica 0):
# render_aov / render_adaptive_aov renders the frame, `denoiser` (a Scene) denoises it.
def _render_denoised(render_aov, denoiser, scene_spp, spp, denoise, kw):
    a, b, aovs, st = _render_halves(render_aov, scene_spp, spp, "render_denoised", kw)
    out = denoiser.denoise(a, b, aovs, **(denoise or {}))
    return out, a + b, aovs, st


def _render_denoised_temporal(render_aov, denoiser, scene_spp, history, spp, seed, current_frame, denoise, gradients, kw):
    frame_seed = (seed + current_frame) % (1 << 32)
    a, b, aovs, st = _render_halves(render_aov, scene_spp, spp, "render_denoised_temporal",
                                    dict(kw, seed=frame_seed, current_frame=current_frame))
    if gradients:
        out = denoiser.denoise_temporal_gradient(history, a, b, aovs, frame_seed, **(denoise or {}))
    else:
        out = denoiser.denoise_temporal(history, a, b, aovs, **(denoise or {}))
    return out, a + b, aovs, st


def _render_denoised_moments(render_aov, denoiser, history, spp, seed, current_frame, denoise, gradients, kw):
    for k in ("sample_first", "sample_count"):
        if k in kw:
            raise ValueError("render_denoised_moments renders the whole sample range; %s is not taken" % k)
    frame_seed = (seed + current_frame) % (1 << 32)
    film, aovs, st = render_aov(spp=spp, seed=frame_seed, current_frame=current_frame, **kw)
    if gradients:
        out = denoiser.denoise_moments_gradient(history, film, aovs, frame_seed, **(denoise or {}))
    else:
        out = denoiser.denoise_moments(history, film, aovs, **(denoise or {}))
    return out, film, aovs, st


def _render_denoised_adaptive(render_adaptive_aov, denoiser, history, min_spp, max_spp, seed, current_frame, denoise, gradients, kw):
    frame_seed = (seed + current_frame) % (1 << 32)
    film, aovs, pixel_spp, st = render_adaptive_aov(min_spp, max_spp, seed=frame_seed, current_frame=current_frame, **kw)
    if gradients:
        out = denoiser.denoise_moments_gradient(history, film, aovs, frame_seed, **(denoise or {}))
    else:
        out = denoiser.denoise_moments(history, film, aovs, **(denoise or {}))
    return out, film, aovs, pixel_spp, st


def _aov_outputs(height, width, film, albedo, normal, nearest, lum=False):
    """The host film and AOV arrays of the AOV renders (Scene and Group), checked or allocated: (film, aovs, AovFilm). aovs holds
    "lum_w" too when `lum` asks for it."""
    if film is None:
        film = np.zeros((height, width, 4), np.float32)
    aovs = {}
    for name, a, shape, dtype, fill in (("albedo_w", albedo, (height, width, 4), np.float32, 0),
                                        ("normal_w", normal, (height, width, 4), np.float32, 0),
                                        ("nearest", nearest, (height, width), np.uint64, np.iinfo(np.uint64).max),
                                        ("lum_w", lum, (height, width, 4), np.float32, 0)):
        if a is True:
            a = np.full(shape, fill, dtype)
        if a is None or a is False:
            continue
        if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
            raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        aovs[name] = a
    if not isinstance(film, np.ndarray) or film.dtype != np.float32 or film.shape != (height, width, 4) or not film.flags.c_contiguous:
        raise ValueError("film must be a C-contiguous float32 array of shape %s" % ((height, width, 4),))
    return film, aovs, F.AovFilm(*(aovs[k].ctypes.data if k in aovs else None for k in ("albedo_w", "normal_w", "nearest")))


class Scene(_Base):
    """A scene resident on one GPU (product path)."""
    _pfx = "trb_"

    def __init__(self, desc, device=0):
        self._lib = F.load_trb()
        self._desc = desc  # keep arrays alive
        h = C.c_void_p()
        self._h = None
        self._histories = []  # DenoiseHistory objects, released before the scene
        self._check(self._lib.trb_scene_create(C.byref(desc), device, C.byref(h)))
        self._h = h
        self.device = device
        self._read_info()

    def _read_info(self):
        w, hh, spp, nb, ni, nl = (F.u32() for _ in range(6))
        self._check(self._lib.trb_scene_info(self._h, *(C.byref(x) for x in (w, hh, spp, nb, ni, nl))))
        self.width, self.height, self.spp, self.total_blocks, self.n_instances, self.n_lights = (x.value for x in (w, hh, spp, nb, ni, nl))

    def _check(self, rc):
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())

    def close(self):
        if self._h is not None:
            for hist in getattr(self, "_histories", []):
                hist.close()
            self._lib.trb_scene_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def render(self, film=None, **kw):
        """trb_render: host film buffer, accumulated into. Returns (film, Stats)."""
        cfg = _cfg(**kw)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        st = F.Stats()
        self._check(self._lib.trb_render(self._h, C.byref(cfg), F.ptr(film), C.byref(st)))
        return film, st

    def render_device(self, d_film_ptr, d_stats_ptr=None, stream=None, **kw):
        cfg = _cfg(**kw)
        self._check(self._lib.trb_render_device(self._h, C.byref(cfg), d_film_ptr, d_stats_ptr, stream))

    def frame_step(self):
        """scene_time / frames in float32: one frame's time, as the renders step the frames."""
        return float(np.float32(self._desc.film.scene_time) / np.float32(self._desc.film.frames))

    def _motion_dt(self, motion):
        """render_*(motion=...): False / None: no motion film; True: one frame back, -scene_time / frames; a number: that dt"""
        if motion is None or motion is False:
            return None
        return -self.frame_step() if motion is True else float(motion)

    def render_aov(self, film=None, albedo=True, normal=True, nearest=True, lum=False, motion=False, **kw):
        """trb_render_aov: the colour film and the AOVs of the same render (DESIGN.md §4 "AOVs"), all accumulated into.
        albedo / normal: True (allocate, zero), False / None (not rendered) or a float32 (height, width, 4) film; nearest: True
        (allocate, all ones), False / None or a uint64 (height, width) array. lum: True or a float32 (height, width, 4) film adds
        the lum_w film of the samples' luminance moments (trb_render_aov_lum, DESIGN.md §4 "Sample variance") as aovs["lum_w"].
        motion: True (dt = -scene_time / frames) or a dt adds the motion_w film (trb_render_aov_motion, include/trb.h "Motion
        vectors") as aovs["motion_w"]; decode_motion turns it into pixels.
        Returns (film, aovs, Stats) where aovs maps "albedo_w", "normal_w" and "nearest" to the arrays rendered."""
        cfg = _cfg(**kw)
        film, aovs, out = _aov_outputs(self.height, self.width, film, albedo, normal, nearest, lum)
        st = F.Stats()
        dt = self._motion_dt(motion)
        if dt is not None:
            aovs["motion_w"] = np.zeros((self.height, self.width, 4), np.float32)
            self._check(self._lib.trb_render_aov_motion(self._h, C.byref(cfg), F.ptr(film), C.byref(out), F.ptr(aovs["lum_w"]) if "lum_w" in aovs else None,
                                                        F.ptr(aovs["motion_w"]), dt, C.byref(st)))
        elif "lum_w" in aovs:
            self._check(self._lib.trb_render_aov_lum(self._h, C.byref(cfg), F.ptr(film), C.byref(out), F.ptr(aovs["lum_w"]), C.byref(st)))
        else:
            self._check(self._lib.trb_render_aov(self._h, C.byref(cfg), F.ptr(film), C.byref(out), C.byref(st)))
        return film, aovs, st

    def render_aov_device(self, d_film, d_albedo=None, d_normal=None, d_nearest=None, d_stats=None, stream=None, d_lum=None, d_motion=None,
                          motion_dt=None, **kw):
        """trb_render_aov_device: device films of height*width*4 float32 (16-byte aligned) and a device nearest buffer of height*width
        uint64 (8-byte aligned; initialise it to all ones), pointers as ints, any AOV None. Enqueued on `stream` (a cudaStream_t as an
        int; None = default stream) without host synchronisation. Never updates the frame. d_lum: a device lum_w film
        (trb_render_aov_lum_device), or None. d_motion: a device motion_w film (trb_render_aov_motion_device) with motion_dt (None:
        -scene_time / frames), or None."""
        cfg = _cfg(**kw)
        out = F.AovFilm(d_albedo, d_normal, d_nearest)
        if d_motion is not None:
            dt = -self.frame_step() if motion_dt is None else float(motion_dt)
            self._check(self._lib.trb_render_aov_motion_device(self._h, C.byref(cfg), d_film, C.byref(out), d_lum, d_motion, dt, d_stats, stream))
        elif d_lum is not None:
            self._check(self._lib.trb_render_aov_lum_device(self._h, C.byref(cfg), d_film, C.byref(out), d_lum, d_stats, stream))
        else:
            self._check(self._lib.trb_render_aov_device(self._h, C.byref(cfg), d_film, C.byref(out), d_stats, stream))

    def render_samples_aov(self, motion=False, **kw):
        """trb_render_samples_aov: (samples as render_samples, AOV records as AOV_SAMPLE_DTYPE in the same order, Stats). motion: True
        (dt = -scene_time / frames) or a dt: trb_render_samples_aov_motion, returning (samples, aov, motion records as
        MOTION_SAMPLE_DTYPE, Stats)."""
        cfg = _cfg(**kw)
        n = self._n_samples(cfg)
        out, aov = np.zeros(n, F.SAMPLE_DTYPE), np.zeros(n, F.AOV_SAMPLE_DTYPE)
        st = F.Stats()
        dt = self._motion_dt(motion)
        if dt is not None:
            mo = np.zeros(n, F.MOTION_SAMPLE_DTYPE)
            self._check(self._lib.trb_render_samples_aov_motion(self._h, C.byref(cfg), n, F.ptr(out), F.ptr(aov), F.ptr(mo), dt, C.byref(st)))
            return out, aov, mo, st
        self._check(self._lib.trb_render_samples_aov(self._h, C.byref(cfg), n, F.ptr(out), F.ptr(aov), C.byref(st)))
        return out, aov, st

    def denoise(self, colour_a, colour_b, aovs, out=None, **params):
        """trb_denoise (DESIGN.md §4 "Denoising"): the two half films of a frame, (height, width, 4) float32, and the AOVs rendered
        over both (a dict with "albedo_w", "normal_w" and "nearest", as render_aov returns it). params: iterations, normal_power,
        sigma_luminance, sigma_depth; a missing one takes its default (F.DENOISE_DEFAULTS). Returns the denoised RGBW film (into
        `out` when given). Scene.render_denoised renders the inputs and calls this."""
        film_shape = (self.height, self.width, 4)
        ins = [("colour_a", colour_a, film_shape, np.float32), ("colour_b", colour_b, film_shape, np.float32),
               ("albedo_w", aovs.get("albedo_w"), film_shape, np.float32), ("normal_w", aovs.get("normal_w"), film_shape, np.float32),
               ("nearest", aovs.get("nearest"), (self.height, self.width), np.uint64)]
        if out is None:
            out = np.zeros(film_shape, np.float32)
        for name, a, shape, dtype in ins + [("out", out, film_shape, np.float32)]:
            if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
                raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        d_in, prm = F.DenoiseInput(*(a.ctypes.data for _, a, _, _ in ins)), _denoise_params(params)
        self._check(self._lib.trb_denoise(self._h, C.byref(d_in), C.byref(prm), F.ptr(out)))
        return out

    def denoise_device(self, d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest, d_out, stream=None, **params):
        """trb_denoise_device: device pointers as ints (films and d_out height*width*4 float32, 16-byte aligned; d_nearest
        height*width uint64, 8-byte aligned), enqueued on `stream` (a cudaStream_t as an int; None = default stream). params as for
        denoise."""
        d_in, prm = F.DenoiseInput(d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest), _denoise_params(params)
        self._check(self._lib.trb_denoise_device(self._h, C.byref(d_in), C.byref(prm), d_out, stream))

    def _temporal_arrays(self, colour_a, colour_b, aovs, out, extra):
        """The five input arrays and the output arrays of a temporal denoise, checked; extra: (name, array or True/False/None,
        shape) of the optional outputs. Returns (ins, outs) as (name, array, shape, dtype) lists."""
        film_shape = (self.height, self.width, 4)
        ins = [("colour_a", colour_a, film_shape, np.float32), ("colour_b", colour_b, film_shape, np.float32),
               ("albedo_w", aovs.get("albedo_w"), film_shape, np.float32), ("normal_w", aovs.get("normal_w"), film_shape, np.float32),
               ("nearest", aovs.get("nearest"), (self.height, self.width), np.uint64)]
        outs = [("out", np.zeros(film_shape, np.float32) if out is None else out, film_shape, np.float32)]
        for name, a, shape, dtype in extra:
            if a is True:
                a = np.zeros(shape, dtype)
            if a is not False and a is not None:
                outs.append((name, a, shape, dtype))
        for name, a, shape, dtype in ins + outs:
            if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
                raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        return ins, outs

    def denoise_temporal_gradient(self, history, colour_a, colour_b, aovs, seed, out=None, motion=False, history_length=False, lam=False,
                                  **params):
        """trb_denoise_temporal_gradient (DESIGN.md §4 "Temporal gradients"): denoise_temporal with temporal gradients. `seed` seeds
        this frame's gradient samples (render_denoised_temporal passes the frame's seed). params: denoise_temporal's plus
        gradient_iterations (trb_denoise_gradient_params.iterations, 0-6, default 3). Returns the denoised RGBW film, or a tuple of it
        with motion, history_length and the (height, width) float32 per-pixel lambda, in that order, where asked for."""
        h, w = self.height, self.width
        ins, outs = self._temporal_arrays(colour_a, colour_b, aovs, out,
                                          [("motion", motion, (h, w, 2), np.float32), ("history_length", history_length, (h, w), np.uint32),
                                           ("lambda", lam, (h, w), np.float32)])
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseInput(*(a.ctypes.data for _, a, _, _ in ins)), _gradient_params(params)
        o = F.DenoiseGradientOutput(*(got[k].ctypes.data if k in got else None for k in ("out", "motion", "history_length", "lambda")))
        self._check(self._lib.trb_denoise_temporal_gradient(self._h, history._h, C.byref(d_in), C.byref(prm), seed % (1 << 32), C.byref(o)))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def denoise_temporal_gradient_device(self, history, d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest, seed, d_out, d_motion=None,
                                         d_history_length=None, d_lambda=None, stream=None, **params):
        """trb_denoise_temporal_gradient_device: denoise_temporal_device's pointers plus d_lambda (height*width float32, 4-byte
        aligned, or None); enqueued on `stream`. params as for denoise_temporal_gradient."""
        d_in, prm = F.DenoiseInput(d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest), _gradient_params(params)
        o = F.DenoiseGradientOutput(d_out, d_motion, d_history_length, d_lambda)
        self._check(self._lib.trb_denoise_temporal_gradient_device(self._h, history._h, C.byref(d_in), C.byref(prm), seed % (1 << 32),
                                                                   C.byref(o), stream))

    def denoise_temporal(self, history, colour_a, colour_b, aovs, out=None, motion=False, history_length=False, **params):
        """trb_denoise_temporal (DESIGN.md §4 "Temporal denoising"): denoise's inputs, rendered at the scene's current frame, with the
        DenoiseHistory `history`, which it reads and then holds this frame. params: denoise's plus max_history, depth_tolerance and
        normal_threshold (F.DENOISE_TEMPORAL_DEFAULTS). Returns the denoised RGBW film (into `out` when given), or a tuple of it with
        the (height, width, 2) float32 motion and the (height, width) uint32 history length where `motion` / `history_length` ask
        for them (True, or an array to write into)."""
        film_shape = (self.height, self.width, 4)
        ins = [("colour_a", colour_a, film_shape, np.float32), ("colour_b", colour_b, film_shape, np.float32),
               ("albedo_w", aovs.get("albedo_w"), film_shape, np.float32), ("normal_w", aovs.get("normal_w"), film_shape, np.float32),
               ("nearest", aovs.get("nearest"), (self.height, self.width), np.uint64)]
        if out is None:
            out = np.zeros(film_shape, np.float32)
        outs = [("out", out, film_shape, np.float32)]
        if motion is True:
            motion = np.zeros((self.height, self.width, 2), np.float32)
        if history_length is True:
            history_length = np.zeros((self.height, self.width), np.uint32)
        if motion is not False and motion is not None:
            outs.append(("motion", motion, (self.height, self.width, 2), np.float32))
        if history_length is not False and history_length is not None:
            outs.append(("history_length", history_length, (self.height, self.width), np.uint32))
        for name, a, shape, dtype in ins + outs:
            if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
                raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseInput(*(a.ctypes.data for _, a, _, _ in ins)), _temporal_params(params)
        o = F.DenoiseTemporalOutput(out.ctypes.data, got["motion"].ctypes.data if "motion" in got else None,
                                    got["history_length"].ctypes.data if "history_length" in got else None)
        self._check(self._lib.trb_denoise_temporal(self._h, history._h, C.byref(d_in), C.byref(prm), C.byref(o)))
        if len(outs) == 1:
            return out
        return tuple(a for _, a, _, _ in outs)

    def denoise_temporal_device(self, history, d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest, d_out, d_motion=None,
                                d_history_length=None, stream=None, **params):
        """trb_denoise_temporal_device: denoise_device's pointers (ints) plus d_motion (height*width*2 float32, 8-byte aligned) and
        d_history_length (height*width uint32), either None; enqueued on `stream`. params as for denoise_temporal."""
        d_in, prm = F.DenoiseInput(d_colour_a, d_colour_b, d_albedo, d_normal, d_nearest), _temporal_params(params)
        o = F.DenoiseTemporalOutput(d_out, d_motion, d_history_length)
        self._check(self._lib.trb_denoise_temporal_device(self._h, history._h, C.byref(d_in), C.byref(prm), C.byref(o), stream))

    def render_denoised_temporal(self, history, spp=0, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """render_denoised for frame `current_frame` of an animation, denoised with `history` (denoise_temporal; the dict `denoise`
        holds its parameters). The two halves are rendered with seed (seed + current_frame) mod 2^32, so that consecutive frames draw
        independent samples (a frame's radiance is a pure function of scene, seed, pixel and sample). With `gradients`, the frame is
        denoised by denoise_temporal_gradient with that frame seed. Returns render_denoised's tuple."""
        return _render_denoised_temporal(self.render_aov, self, self.spp, history, spp, seed, current_frame, denoise, gradients, kw)

    def denoise_moments(self, history, colour, aovs, out=None, motion=False, history_length=False, variance=False, **params):
        """trb_denoise_moments (DESIGN.md §4 "Moment denoising"): one colour film of the frame at any spp, (height, width, 4)
        float32, and the AOVs of the same render (render_aov's dict), rendered at the scene's current frame, with the DenoiseHistory
        `history`. The variance comes from the luminance moments accumulated in the history, or a 7x7 spatial estimate where it is
        short. params: denoise_temporal's. Returns the denoised RGBW film (into `out` when given), or a tuple of it with the motion,
        the history length and the (height, width) float32 variance, in that order, where asked for (True, or an array)."""
        ins, outs = self._moments_arrays(colour, aovs, out, motion, history_length, variance)
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseFrame(*(a.ctypes.data for _, a, _, _ in ins)), _temporal_params(params)
        o = F.DenoiseMomentsOutput(*(got[k].ctypes.data if k in got else None for k in ("out", "motion", "history_length", "variance")))
        self._check(self._lib.trb_denoise_moments(self._h, history._h, C.byref(d_in), C.byref(prm), C.byref(o)))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def _moments_arrays(self, colour, aovs, out, motion, history_length, variance, lam=False, lum=False):
        """The four input arrays and the output arrays of a moment denoise, checked (motion, history_length, variance and lam:
        True, False/None or an array); with `lum`, aovs["lum_w"] is a fifth input. Returns (ins, outs) as (name, array, shape,
        dtype) lists."""
        h, w = self.height, self.width
        film_shape = (h, w, 4)
        ins = [("colour", colour, film_shape, np.float32), ("albedo_w", aovs.get("albedo_w"), film_shape, np.float32),
               ("normal_w", aovs.get("normal_w"), film_shape, np.float32), ("nearest", aovs.get("nearest"), (h, w), np.uint64)]
        if lum:
            ins.append(("lum_w", aovs.get("lum_w"), film_shape, np.float32))
        outs = [("out", np.zeros(film_shape, np.float32) if out is None else out, film_shape, np.float32)]
        for name, a, shape, dtype in (("motion", motion, (h, w, 2), np.float32), ("history_length", history_length, (h, w), np.uint32),
                                      ("variance", variance, (h, w), np.float32), ("lambda", lam, (h, w), np.float32)):
            if a is True:
                a = np.zeros(shape, dtype)
            if a is not False and a is not None:
                outs.append((name, a, shape, dtype))
        for name, a, shape, dtype in ins + outs:
            if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
                raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        return ins, outs

    def denoise_moments_gradient(self, history, colour, aovs, seed, out=None, motion=False, history_length=False, variance=False, lam=False,
                                 **params):
        """trb_denoise_moments_gradient (DESIGN.md §4 "Moment gradients"): denoise_moments with temporal gradients, so a history is
        shortened where the lighting under it changed. `seed` seeds this frame's gradient samples (render_denoised_moments passes
        the frame's seed). params: denoise_moments's plus gradient_iterations (0-6, default 3). Returns the denoised RGBW film, or
        a tuple of it with the motion, the history length, the variance and the (height, width) float32 per-pixel lambda, in that
        order, where asked for (True, or an array)."""
        ins, outs = self._moments_arrays(colour, aovs, out, motion, history_length, variance, lam)
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseFrame(*(a.ctypes.data for _, a, _, _ in ins)), _gradient_params(params)
        o = F.DenoiseMomentsGradientOutput(*(got[k].ctypes.data if k in got else None
                                             for k in ("out", "motion", "history_length", "variance", "lambda")))
        self._check(self._lib.trb_denoise_moments_gradient(self._h, history._h, C.byref(d_in), C.byref(prm), seed % (1 << 32), C.byref(o)))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def denoise_moments_gradient_device(self, history, d_colour, d_albedo, d_normal, d_nearest, seed, d_out, d_motion=None,
                                        d_history_length=None, d_variance=None, d_lambda=None, stream=None, **params):
        """trb_denoise_moments_gradient_device: denoise_moments_device's pointers plus d_lambda (height*width float32, 4-byte
        aligned, or None); enqueued on `stream`. params as for denoise_moments_gradient."""
        d_in, prm = F.DenoiseFrame(d_colour, d_albedo, d_normal, d_nearest), _gradient_params(params)
        o = F.DenoiseMomentsGradientOutput(d_out, d_motion, d_history_length, d_variance, d_lambda)
        self._check(self._lib.trb_denoise_moments_gradient_device(self._h, history._h, C.byref(d_in), C.byref(prm), seed % (1 << 32),
                                                                  C.byref(o), stream))

    def denoise_moments_device(self, history, d_colour, d_albedo, d_normal, d_nearest, d_out, d_motion=None, d_history_length=None,
                               d_variance=None, stream=None, **params):
        """trb_denoise_moments_device: device pointers as ints (d_colour, d_albedo, d_normal and d_out height*width*4 float32,
        16-byte aligned; d_nearest height*width uint64 and d_motion height*width*2 float32, 8-byte aligned; d_history_length
        height*width uint32 and d_variance height*width float32, 4-byte aligned; the last three may be None), enqueued on `stream`.
        params as for denoise_moments."""
        d_in, prm = F.DenoiseFrame(d_colour, d_albedo, d_normal, d_nearest), _temporal_params(params)
        o = F.DenoiseMomentsOutput(d_out, d_motion, d_history_length, d_variance)
        self._check(self._lib.trb_denoise_moments_device(self._h, history._h, C.byref(d_in), C.byref(prm), C.byref(o), stream))

    def render_denoised_moments(self, history, spp=0, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """Frame `current_frame` of an animation rendered once by render_aov at `spp` (0: the scene's; 1 is enough) with seed
        (seed + current_frame) mod 2^32, and denoised with `history` by denoise_moments (the dict `denoise` holds its parameters).
        With `gradients`, the frame is denoised by denoise_moments_gradient with that frame seed. Returns (denoised, film, aovs,
        stats)."""
        return _render_denoised_moments(self.render_aov, self, history, spp, seed, current_frame, denoise, gradients, kw)

    def render_denoised_adaptive(self, history, min_spp, max_spp, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """render_denoised_moments with the Adaptive sampler (DESIGN.md §4 "Adaptive AOVs"): frame `current_frame` rendered once by
        render_adaptive_aov(min_spp, max_spp) with seed (seed + current_frame) mod 2^32, and denoised with `history` by
        denoise_moments, or with `gradients` by denoise_moments_gradient with that frame seed. For a single image pass
        denoise={"max_history": 1}. Returns (denoised, film, aovs, pixel_spp, stats)."""
        return _render_denoised_adaptive(self.render_adaptive_aov, self, history, min_spp, max_spp, seed, current_frame, denoise, gradients, kw)

    def denoise_variance(self, colour, aovs, out=None, variance=False, **params):
        """trb_denoise_variance (DESIGN.md §4 "Sample variance"): one colour film, (height, width, 4) float32, denoised with the
        variance of each pixel's own samples. aovs: render_aov(lum=True)'s dict ("albedo_w", "normal_w", "nearest" and "lum_w").
        params: denoise's. Returns the denoised RGBW film (into `out` when given), or a tuple of it and the (height, width) float32
        variance where asked for (True, or an array)."""
        h, w = self.height, self.width
        film_shape = (h, w, 4)
        ins = [("colour", colour, film_shape, np.float32), ("albedo_w", aovs.get("albedo_w"), film_shape, np.float32),
               ("normal_w", aovs.get("normal_w"), film_shape, np.float32), ("nearest", aovs.get("nearest"), (h, w), np.uint64),
               ("lum_w", aovs.get("lum_w"), film_shape, np.float32)]
        outs = [("out", np.zeros(film_shape, np.float32) if out is None else out, film_shape, np.float32)]
        if variance is True:
            variance = np.zeros((h, w), np.float32)
        if variance is not False and variance is not None:
            outs.append(("variance", variance, (h, w), np.float32))
        for name, a, shape, dtype in ins + outs:
            if not isinstance(a, np.ndarray) or a.dtype != dtype or a.shape != shape or not a.flags.c_contiguous:
                raise ValueError("%s must be a C-contiguous %s array of shape %s" % (name, np.dtype(dtype).name, shape))
        d_in, prm = F.DenoiseFrame(*(a.ctypes.data for _, a, _, _ in ins[:4])), _denoise_params(params)
        self._check(self._lib.trb_denoise_variance(self._h, C.byref(d_in), ins[4][1].ctypes.data, C.byref(prm), outs[0][1].ctypes.data,
                                                   outs[1][1].ctypes.data if len(outs) > 1 else None))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def denoise_variance_device(self, d_colour, d_albedo, d_normal, d_nearest, d_lum, d_out, d_variance=None, stream=None, **params):
        """trb_denoise_variance_device: device pointers as ints (d_colour, d_albedo, d_normal, d_lum and d_out height*width*4
        float32, 16-byte aligned; d_nearest height*width uint64, 8-byte aligned; d_variance height*width float32, 4-byte aligned, or
        None), enqueued on `stream`. params as for denoise."""
        d_in, prm = F.DenoiseFrame(d_colour, d_albedo, d_normal, d_nearest), _denoise_params(params)
        self._check(self._lib.trb_denoise_variance_device(self._h, C.byref(d_in), d_lum, C.byref(prm), d_out, d_variance, stream))

    def render_denoised_variance(self, spp=0, adaptive=None, denoise=None, **kw):
        """A still frame rendered once with the AOVs and the lum_w film, and denoised by denoise_variance with the parameters in the
        dict `denoise` (None: the defaults): by render_aov at `spp` samples per pixel (0: the scene's), or with adaptive=(min_spp,
        max_spp) by render_adaptive_aov. kw: the render's (seed, current_frame, flags, block_start, block_count). Returns (denoised,
        film, aovs, stats), with pixel_spp before stats for an Adaptive render."""
        if adaptive is not None:
            if spp:
                raise ValueError("render_denoised_variance: the Adaptive sampler chooses the sample counts; spp is not taken")
            film, aovs, pixel_spp, st = self.render_adaptive_aov(adaptive[0], adaptive[1], lum=True, **kw)
            return self.denoise_variance(film, aovs, **(denoise or {})), film, aovs, pixel_spp, st
        film, aovs, st = self.render_aov(lum=True, spp=spp, **kw)
        return self.denoise_variance(film, aovs, **(denoise or {})), film, aovs, st

    def denoise_variance_temporal(self, history, colour, aovs, out=None, motion=False, history_length=False, variance=False, **params):
        """trb_denoise_variance_temporal (DESIGN.md §4 "Variance temporal denoising"): one colour film of the frame and the AOVs of
        the same render with its lum_w film (render_aov(lum=True)'s dict), rendered at the scene's current frame, with the
        DenoiseHistory `history`. The variance of each pixel's own samples is carried through the history. params:
        denoise_temporal's. Returns denoise_moments's film or tuple."""
        ins, outs = self._moments_arrays(colour, aovs, out, motion, history_length, variance, lum=True)
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseFrame(*(a.ctypes.data for _, a, _, _ in ins[:4])), _temporal_params(params)
        o = F.DenoiseMomentsOutput(*(got[k].ctypes.data if k in got else None for k in ("out", "motion", "history_length", "variance")))
        self._check(self._lib.trb_denoise_variance_temporal(self._h, history._h, C.byref(d_in), ins[4][1].ctypes.data, C.byref(prm), C.byref(o)))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def denoise_variance_temporal_gradient(self, history, colour, aovs, seed, out=None, motion=False, history_length=False, variance=False,
                                           lam=False, **params):
        """trb_denoise_variance_temporal_gradient: denoise_variance_temporal with temporal gradients. `seed` seeds this frame's
        gradient samples. params: denoise_moments_gradient's. Returns denoise_moments_gradient's film or tuple."""
        ins, outs = self._moments_arrays(colour, aovs, out, motion, history_length, variance, lam, lum=True)
        got = {name: a for name, a, _, _ in outs}
        d_in, prm = F.DenoiseFrame(*(a.ctypes.data for _, a, _, _ in ins[:4])), _gradient_params(params)
        o = F.DenoiseMomentsGradientOutput(*(got[k].ctypes.data if k in got else None
                                             for k in ("out", "motion", "history_length", "variance", "lambda")))
        self._check(self._lib.trb_denoise_variance_temporal_gradient(self._h, history._h, C.byref(d_in), ins[4][1].ctypes.data, C.byref(prm),
                                                                     seed % (1 << 32), C.byref(o)))
        if len(outs) == 1:
            return outs[0][1]
        return tuple(a for _, a, _, _ in outs)

    def denoise_variance_temporal_device(self, history, d_colour, d_albedo, d_normal, d_nearest, d_lum, d_out, d_motion=None,
                                         d_history_length=None, d_variance=None, stream=None, **params):
        """trb_denoise_variance_temporal_device: denoise_moments_device's pointers plus d_lum (height*width*4 float32, 16-byte
        aligned); enqueued on `stream`. params as for denoise_variance_temporal."""
        d_in, prm = F.DenoiseFrame(d_colour, d_albedo, d_normal, d_nearest), _temporal_params(params)
        o = F.DenoiseMomentsOutput(d_out, d_motion, d_history_length, d_variance)
        self._check(self._lib.trb_denoise_variance_temporal_device(self._h, history._h, C.byref(d_in), d_lum, C.byref(prm), C.byref(o), stream))

    def denoise_variance_temporal_gradient_device(self, history, d_colour, d_albedo, d_normal, d_nearest, d_lum, seed, d_out, d_motion=None,
                                                  d_history_length=None, d_variance=None, d_lambda=None, stream=None, **params):
        """trb_denoise_variance_temporal_gradient_device: denoise_variance_temporal_device's pointers plus d_lambda (height*width
        float32, 4-byte aligned, or None); enqueued on `stream`. params as for denoise_variance_temporal_gradient."""
        d_in, prm = F.DenoiseFrame(d_colour, d_albedo, d_normal, d_nearest), _gradient_params(params)
        o = F.DenoiseMomentsGradientOutput(d_out, d_motion, d_history_length, d_variance, d_lambda)
        self._check(self._lib.trb_denoise_variance_temporal_gradient_device(self._h, history._h, C.byref(d_in), d_lum, C.byref(prm),
                                                                            seed % (1 << 32), C.byref(o), stream))

    def render_denoised_variance_temporal(self, history, spp=0, adaptive=None, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """Frame `current_frame` of an animation rendered once with the AOVs and the lum_w film, with seed (seed + current_frame)
        mod 2^32: by render_aov at `spp` (0: the scene's), or with adaptive=(min_spp, max_spp) by render_adaptive_aov. Denoised with
        `history` by denoise_variance_temporal, or with `gradients` by denoise_variance_temporal_gradient with that frame seed (the
        dict `denoise` holds the parameters). Returns render_denoised_variance's tuple."""
        frame_seed = (seed + current_frame) % (1 << 32)
        kw = dict(kw, seed=frame_seed, current_frame=current_frame)
        if adaptive is not None:
            if spp:
                raise ValueError("render_denoised_variance_temporal: the Adaptive sampler chooses the sample counts; spp is not taken")
            film, aovs, pixel_spp, st = self.render_adaptive_aov(adaptive[0], adaptive[1], lum=True, **kw)
        else:
            film, aovs, st = self.render_aov(lum=True, spp=spp, **kw)
        if gradients:
            out = self.denoise_variance_temporal_gradient(history, film, aovs, frame_seed, **(denoise or {}))
        else:
            out = self.denoise_variance_temporal(history, film, aovs, **(denoise or {}))
        return (out, film, aovs, pixel_spp, st) if adaptive is not None else (out, film, aovs, st)

    def render_denoised(self, spp=0, denoise=None, **kw):
        """A denoised frame at `spp` samples per pixel (0: the scene's), rounded up to a power of two as every render rounds it:
        samples [0, spp/2) and [spp/2, spp) are rendered into two films by render_aov, with the albedo, normal and nearest AOVs
        accumulated over both, and denoised with the parameters in the dict `denoise` (None: the defaults). kw: render_aov's
        (seed, current_frame, flags, block_start, block_count). Returns (denoised, film, aovs, (stats_a, stats_b)), where film is
        the sum of the two halves, the noisy spp-sample film. Raises ValueError below 2 spp."""
        return _render_denoised(self.render_aov, self, self.spp, spp, denoise, kw)

    def _mesh_verts(self, mesh):
        if not 0 <= mesh < self._desc.n_meshes:
            raise ValueError("mesh index %d out of range (%d meshes)" % (mesh, self._desc.n_meshes))
        return self._desc.meshes[mesh].n_verts

    def _mesh_arrays(self, mesh, positions, normals, texcoords):
        """the three arrays as float32 pointers (None kept), each checked against the mesh's vertex count"""
        nv = self._mesh_verts(mesh)
        arrays = []
        for name, a, k in (("positions", positions, 3), ("normals", normals, 3), ("texcoords", texcoords, 2)):
            if a is not None:
                a = np.ascontiguousarray(a, np.float32)
                if a.size != nv * k or (a.ndim != 1 and a.shape != (nv, k)):
                    raise ValueError("%s must have shape (%d, %d), got %s" % (name, nv, k, a.shape))
            arrays.append(a)
        return arrays

    def update_mesh(self, mesh, positions=None, normals=None, texcoords=None):
        """trb_scene_update_mesh: replace mesh `mesh`'s positions (n_verts x 3), normals (n_verts x 3) and / or texcoords
        (n_verts x 2); None keeps an array. New positions rebuild the mesh's BVH and refresh the current frame."""
        arrays = self._mesh_arrays(mesh, positions, normals, texcoords)
        self._check(self._lib.trb_scene_update_mesh(self._h, mesh, *(None if a is None else F.ptr(a) for a in arrays)))

    def refit_mesh(self, mesh, positions, normals=None, texcoords=None):
        """trb_scene_refit_mesh: move mesh `mesh`'s vertices to `positions` (n_verts x 3) keeping its BVH's partition (the boxes are
        recomputed bottom-up on the device) and refresh the current frame; normals (n_verts x 3) and texcoords (n_verts x 2) may be
        replaced in the same call. Cheaper than update_mesh, but the tree's quality drops as the mesh deforms."""
        arrays = self._mesh_arrays(mesh, positions, normals, texcoords)
        self._check(self._lib.trb_scene_refit_mesh(self._h, mesh, *(None if a is None else F.ptr(a) for a in arrays)))

    def refit_mesh_device(self, mesh, d_positions, d_normals=None, d_texcoords=None, stream=None):
        """trb_scene_refit_mesh_device: the same from device pointers (ints) holding float32 arrays of the mesh's vertex count,
        read on `stream` (a cudaStream_t as an int; None = default stream)."""
        self._mesh_verts(mesh)
        self._check(self._lib.trb_scene_refit_mesh_device(self._h, mesh, d_positions, d_normals, d_texcoords, stream))

    def update_mesh_device(self, mesh, d_positions=None, d_normals=None, d_texcoords=None, stream=None):
        """trb_scene_update_mesh_device: the same from device pointers (ints) holding float32 arrays of the mesh's vertex count,
        read on `stream` (a cudaStream_t as an int; None = default stream)."""
        self._mesh_verts(mesh)
        self._check(self._lib.trb_scene_update_mesh_device(self._h, mesh, d_positions, d_normals, d_texcoords, stream))

    def _edit_range(self, name, first, count):
        n = getattr(self._desc, "n_" + name)
        if first < 0 or count < 0 or first + count > n:
            raise ValueError("%s [%d, %d) out of range (%d entries)" % (name, first, first + count, n))

    def _edit(self, name, dtype, first, a):
        a = np.asarray(a)
        if a.dtype != dtype or a.ndim != 1:
            raise ValueError("%s must be a 1-d array of dtype %s, got %s %s" % (name, dtype, a.dtype, a.shape))
        self._edit_range(name, first, len(a))
        a = np.ascontiguousarray(a)
        self._check(getattr(self._lib, "trb_scene_update_" + name)(self._h, first, len(a), F.ptr(a)))

    def update_keyframes(self, first, keyframes):
        """trb_scene_update_keyframes: replace keyframes[first:first + len(keyframes)] (F.KEYFRAME_DTYPE), the TRS control points of
        instance, group and camera transforms; a frame already set is rebuilt."""
        self._edit("keyframes", F.KEYFRAME_DTYPE, first, keyframes)

    def update_keyframes_device(self, first, count, d_keyframes, stream=None):
        """trb_scene_update_keyframes_device: the same from a device pointer (int) to `count` keyframes in F.KEYFRAME_DTYPE's layout,
        read on `stream` (a cudaStream_t as an int; None = default stream)."""
        self._edit_range("keyframes", first, count)
        self._check(self._lib.trb_scene_update_keyframes_device(self._h, first, count, d_keyframes, stream))

    def update_color_keys(self, first, keys):
        """trb_scene_update_color_keys: replace color_keys[first:first + len(keys)] (F.COLOR_KEY_DTYPE), emission colours and times."""
        self._edit("color_keys", F.COLOR_KEY_DTYPE, first, keys)

    def update_materials(self, first, materials):
        """trb_scene_update_materials: replace materials[first:first + len(materials)] (F.MATERIAL_DTYPE)."""
        self._edit("materials", F.MATERIAL_DTYPE, first, materials)

    def replace_objects(self, objects):
        """trb_scene_replace_objects: replace the cameras, instances, splines, keyframes, knots, colour keys and fov floats with the
        section `objects` (F.SceneObjects, e.g. SceneBuilder.objects()); meshes, materials, textures, film and integrator stay. Counts
        may change: this adds and removes objects, lights and cameras. A frame already set is rebuilt."""
        self._check(self._lib.trb_scene_replace_objects(self._h, C.byref(objects)))
        self._replaced(objects)

    def replace_meshes(self, section, objects=None):
        """trb_scene_replace_meshes: replace the mesh list with `section` (F.SceneMeshes, e.g. SceneBuilder.meshes()): kept meshes
        (keep[i], an index of the current list) stay built, MESH_NEW entries are uploaded and built, unnamed meshes are released. With
        `objects` (F.SceneObjects) the object section is replaced too; without, the instances' mesh indices index the new list. A
        frame already set is rebuilt."""
        self._check(self._lib.trb_scene_replace_meshes(self._h, C.byref(section), None if objects is None else C.byref(objects)))
        self._replaced(objects, section)

    def replace_meshes_device(self, section, objects=None, stream=None):
        """trb_scene_replace_meshes_device: the same with the new meshes' four arrays as device pointers on the scene's GPU, read on
        `stream` (a cudaStream_t as an int; None = default stream)."""
        self._check(self._lib.trb_scene_replace_meshes_device(self._h, C.byref(section), None if objects is None else C.byref(objects), stream))
        self._replaced(objects, section)

    def replace_settings(self, film=None, integrator=None):
        """trb_scene_replace_settings: replace the film (F.Film, or a dict of its fields like SceneBuilder.film) and / or the integrator
        (F.Integrator, or a (type, min_depth, max_depth) tuple like SceneBuilder.integrator); None keeps the current one. A frame
        already set is rebuilt."""
        if isinstance(film, dict):
            film = F.Film(**film)
        if isinstance(integrator, tuple):
            integrator = F.Integrator(*integrator)
        self._check(self._lib.trb_scene_replace_settings(self._h, None if film is None else C.byref(film),
                                                           None if integrator is None else C.byref(integrator)))
        self._replaced(film=film, integrator=integrator)

    def replace_materials(self, section, objects=None):
        """trb_scene_replace_materials: replace the materials, MERL tables, textures and images with `section` (F.SceneMaterials, e.g.
        SceneBuilder.materials_section()). With `objects` (F.SceneObjects) the object section is replaced too; without, the instances'
        material indices index the new list. A frame already set is rebuilt."""
        self._check(self._lib.trb_scene_replace_materials(self._h, C.byref(section), None if objects is None else C.byref(objects)))
        self._replaced(objects, materials=section)

    def replace_materials_device(self, section, objects=None, stream=None):
        """trb_scene_replace_materials_device: the same with the MERL tables and each image's rgba8 as device pointers on the scene's
        GPU, read on `stream` (a cudaStream_t as an int; None = default stream)."""
        self._check(self._lib.trb_scene_replace_materials_device(self._h, C.byref(section), None if objects is None else C.byref(objects),
                                                                 stream))
        self._replaced(objects, materials=section)

    def _replaced(self, objects=None, section=None, materials=None, film=None, integrator=None):
        """the description after a replacement: the object section, the mesh list (kept meshes keep their entries), the material section,
        the film and / or the integrator"""
        desc = F.SceneDesc.from_buffer_copy(self._desc)  # a copy: the caller's description (it may belong to the loader) stays as it is
        for name, _ in F.SceneObjects._fields_ if objects is not None else ():
            setattr(desc, name, getattr(objects, name))
        for name, _ in F.SceneMaterials._fields_ if materials is not None else ():
            setattr(desc, name, getattr(materials, name))
        if film is not None:
            desc.film = film
        if integrator is not None:
            desc.integrator = integrator
        meshes = None
        if section is not None:
            n = section.n_meshes
            meshes = (F.Mesh * max(1, n))()
            for i in range(n):
                k = section.keep[i]
                meshes[i] = section.meshes[i] if k == F.MESH_NEW else self._desc.meshes[k]
            desc.meshes, desc.n_meshes = meshes, n
        desc._keep = (self._desc, objects, section, meshes, materials)  # the arrays they point into
        self._desc = desc
        w, hh, spp, nb, ni, nl = (F.u32() for _ in range(6))
        self._check(self._lib.trb_scene_info(self._h, *(C.byref(x) for x in (w, hh, spp, nb, ni, nl))))
        self.width, self.height, self.spp, self.total_blocks, self.n_instances, self.n_lights = (x.value for x in (w, hh, spp, nb, ni, nl))

    def set_option(self, name, value):
        """trb_scene_set_option: launch-shape options (never change results)."""
        self._check(self._lib.trb_scene_set_option(self._h, name.encode(), int(value)))

    def check_error(self):
        """trb_scene_check_error: drain the device, raise on a latched traversal-stack overflow."""
        self._check(self._lib.trb_scene_check_error(self._h))

    def trace_time(self):
        """(total ms, launches) of the trace kernel for launches made with RENDER_TIME_TRACE since the last call."""
        ms, n = F.f32(), F.u32()
        self._check(self._lib.trb_scene_trace_time(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def render_samples(self, **kw):
        cfg = _cfg(**kw)
        n = self._n_samples(cfg)
        out = np.zeros(n, F.SAMPLE_DTYPE)
        st = F.Stats()
        self._check(self._lib.trb_render_samples(self._h, C.byref(cfg), n, F.ptr(out), C.byref(st)))
        return out, st

    def render_adaptive(self, min_spp, max_spp, film=None, **kw):
        """trb_render_adaptive: the Adaptive sampler over the selected blocks, film accumulated into.
        Returns (film, pixel_spp (height, width) uint32, zero outside the selection, Stats)."""
        cfg = _cfg(**kw)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_render_adaptive(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(film), F.ptr(spp), C.byref(st)))
        return film, spp, st

    def render_adaptive_device(self, min_spp, max_spp, d_film_ptr, d_pixel_spp_ptr=None, d_stats_ptr=None, stream=None, **kw):
        """trb_render_adaptive_device: the Adaptive sampler into a device film (accumulated into), enqueued on `stream` (a
        cudaStream_t as an int, e.g. torch.cuda.Stream().cuda_stream; None = default stream) without host synchronisation.
        d_pixel_spp_ptr: device buffer of height*width uint32 (only the selected pixels are written) or None; d_stats_ptr: a
        device trb_stats (72 bytes) or None. Never updates the frame."""
        cfg = _cfg(**kw)
        self._check(self._lib.trb_render_adaptive_device(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), d_film_ptr, d_pixel_spp_ptr,
                                                         d_stats_ptr, stream))

    def render_samples_adaptive(self, min_spp, max_spp, **kw):
        """trb_render_samples_adaptive: (samples (blocks, 64, max_per_pixel) flattened, unused slots zero; pixel_spp; Stats)."""
        cfg = _cfg(**kw)
        n = self._n_selected_blocks(cfg) * 64 * adaptive_schedule(min_spp, max_spp)[3]
        out = np.zeros(n, F.SAMPLE_DTYPE)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_render_samples_adaptive(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), n, F.ptr(out), F.ptr(spp),
                                                          C.byref(st)))
        return out, spp, st

    def render_adaptive_aov(self, min_spp, max_spp, film=None, albedo=True, normal=True, nearest=True, lum=False, motion=False, **kw):
        """trb_render_adaptive_aov: render_adaptive with the AOVs of the samples it takes (DESIGN.md §4 "Adaptive AOVs"), all
        accumulated into; albedo / normal / nearest / lum / motion as for render_aov (lum: trb_render_adaptive_aov_lum, motion:
        trb_render_adaptive_aov_motion). Returns (film, aovs, pixel_spp, Stats)."""
        cfg = _cfg(**kw)
        film, aovs, out = _aov_outputs(self.height, self.width, film, albedo, normal, nearest, lum)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        ad = F.Adaptive(min_spp, max_spp)
        dt = self._motion_dt(motion)
        if dt is not None:
            aovs["motion_w"] = np.zeros((self.height, self.width, 4), np.float32)
            self._check(self._lib.trb_render_adaptive_aov_motion(self._h, C.byref(cfg), C.byref(ad), F.ptr(film), C.byref(out),
                                                                 F.ptr(aovs["lum_w"]) if "lum_w" in aovs else None, F.ptr(aovs["motion_w"]), dt,
                                                                 F.ptr(spp), C.byref(st)))
        elif "lum_w" in aovs:
            self._check(self._lib.trb_render_adaptive_aov_lum(self._h, C.byref(cfg), C.byref(ad), F.ptr(film), C.byref(out), F.ptr(aovs["lum_w"]),
                                                              F.ptr(spp), C.byref(st)))
        else:
            self._check(self._lib.trb_render_adaptive_aov(self._h, C.byref(cfg), C.byref(ad), F.ptr(film), C.byref(out), F.ptr(spp), C.byref(st)))
        return film, aovs, spp, st

    def render_adaptive_aov_device(self, min_spp, max_spp, d_film, d_albedo=None, d_normal=None, d_nearest=None, d_pixel_spp=None, d_stats=None,
                                   stream=None, d_lum=None, d_motion=None, motion_dt=None, **kw):
        """trb_render_adaptive_aov_device: render_adaptive_device's pointers plus the AOV buffers of render_aov_device (any None).
        Enqueued on `stream` without host synchronisation. Never updates the frame. d_lum: a device lum_w film
        (trb_render_adaptive_aov_lum_device), or None; d_motion / motion_dt as for render_aov_device
        (trb_render_adaptive_aov_motion_device)."""
        cfg = _cfg(**kw)
        out = F.AovFilm(d_albedo, d_normal, d_nearest)
        ad = F.Adaptive(min_spp, max_spp)
        if d_motion is not None:
            dt = -self.frame_step() if motion_dt is None else float(motion_dt)
            self._check(self._lib.trb_render_adaptive_aov_motion_device(self._h, C.byref(cfg), C.byref(ad), d_film, C.byref(out), d_lum, d_motion, dt,
                                                                        d_pixel_spp, d_stats, stream))
        elif d_lum is not None:
            self._check(self._lib.trb_render_adaptive_aov_lum_device(self._h, C.byref(cfg), C.byref(ad), d_film, C.byref(out), d_lum, d_pixel_spp,
                                                                     d_stats, stream))
        else:
            self._check(self._lib.trb_render_adaptive_aov_device(self._h, C.byref(cfg), C.byref(ad), d_film, C.byref(out), d_pixel_spp, d_stats,
                                                                 stream))

    def render_samples_adaptive_aov(self, min_spp, max_spp, **kw):
        """trb_render_samples_adaptive_aov: (samples as render_samples_adaptive, AOV records as AOV_SAMPLE_DTYPE in the same layout,
        unused slots zero; pixel_spp; Stats)."""
        cfg = _cfg(**kw)
        n = self._n_selected_blocks(cfg) * 64 * adaptive_schedule(min_spp, max_spp)[3]
        out, aov = np.zeros(n, F.SAMPLE_DTYPE), np.zeros(n, F.AOV_SAMPLE_DTYPE)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_render_samples_adaptive_aov(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), n, F.ptr(out), F.ptr(aov),
                                                              F.ptr(spp), C.byref(st)))
        return out, aov, spp, st

    def camera_rays(self, **kw):
        cfg = _cfg(**kw)
        n = self._n_samples(cfg)
        rays, xy = np.zeros(n, F.RAY_DTYPE), np.zeros((n, 2), np.float32)
        self._check(self._lib.trb_camera_rays(self._h, C.byref(cfg), n, F.ptr(rays), F.ptr(xy)))
        return rays, xy

    def camera_rays_device(self, d_rays, d_xy, stream=None, **kw):
        """trb_camera_rays_device: the camera rays (RAY_DTYPE, 32 B) and film positions (2 float32) of the selection into device
        buffers of n = blocks * 64 * sample_count records (4-byte aligned), enqueued on `stream` (a cudaStream_t as an int; None =
        default stream) without host synchronisation. Returns n."""
        cfg = _cfg(**kw)
        n = self._n_samples(cfg)
        self._check(self._lib.trb_camera_rays_device(self._h, C.byref(cfg), n, d_rays, d_xy, stream))
        return n

    def film_write(self, samples, regions, film=None):
        """trb_film_write: RenderTarget::write once per region that has samples, regions in Morton-list order, each region's
        samples (SAMPLE_DTYPE) in input order; regions[i] is the 8x8 block index of sample i (sample_regions() for render_samples'
        order; an index >= total_blocks skips the sample). `film` (height, width, 4) float32 is added into in place; a zero film
        when None. Returns the film. Bit-reproducible: no float atomics."""
        samples = np.ascontiguousarray(samples, dtype=F.SAMPLE_DTYPE)
        regions = np.ascontiguousarray(regions, dtype=np.uint32)
        assert len(samples) == len(regions)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        assert film.dtype == np.float32 and film.flags.c_contiguous and film.size == self.height * self.width * 4
        self._check(self._lib.trb_film_write(self._h, len(samples), F.ptr(samples), F.ptr(regions), F.ptr(film)))
        return film

    def film_write_device(self, n, d_samples, d_regions, d_film, stream=None):
        """trb_film_write_device: n samples (20 B), n uint32 regions and the RGBW film, device buffers 4-byte aligned, enqueued on
        `stream` without host synchronisation (except once, when the scene's sort scratch grows)."""
        self._check(self._lib.trb_film_write_device(self._h, n, d_samples, d_regions, d_film, stream))

    def intersect(self, rays):
        rays = np.ascontiguousarray(rays, dtype=F.RAY_DTYPE)
        hits = np.zeros(len(rays), F.HIT_DTYPE)
        st = F.Stats()
        self._check(self._lib.trb_intersect(self._h, len(rays), F.ptr(rays), F.ptr(hits), C.byref(st)))
        return hits, st

    def intersect_device(self, n, d_rays, d_hits, d_stats=None, stream=None):
        self._check(self._lib.trb_intersect_device(self._h, n, d_rays, d_hits, d_stats, stream))

    def intersect_records(self, rays, stats=False):
        """trb_intersect_records: Scene::intersect of each QUERY_RAY_DTYPE ray at its own time. Returns (INTERSECTION_DTYPE records,
        Stats); stats=True also counts node / triangle / instance tests."""
        rays = np.ascontiguousarray(rays, dtype=F.QUERY_RAY_DTYPE)
        out = np.zeros(len(rays), F.INTERSECTION_DTYPE)
        st = F.Stats()
        self._check(self._lib.trb_intersect_records(self._h, len(rays), F.ptr(rays), F.ptr(out), F.RENDER_STATS if stats else 0, C.byref(st)))
        return out, st

    def intersect_records_device(self, n, d_rays, d_out, d_stats=None, stream=None, stats=False):
        """trb_intersect_records_device: device buffers of n query rays (48 B each) and n records (96 B each), both 16-byte
        aligned, enqueued on `stream` (a cudaStream_t as an int; None = default stream) without host synchronisation."""
        self._check(self._lib.trb_intersect_records_device(self._h, n, d_rays, d_out, F.RENDER_STATS if stats else 0, d_stats, stream))

    def occluded(self, rays, reference=False, stats=False):
        """trb_occluded: OcclusionTester::occluded of each QUERY_RAY_DTYPE segment at its own time. Returns (bool array, Stats).
        reference=True walks to the closest hit like the reference (its test counters); the default stops at the first hit."""
        rays = np.ascontiguousarray(rays, dtype=F.QUERY_RAY_DTYPE)
        out = np.zeros(len(rays), np.uint8)
        st = F.Stats()
        flags = (F.RENDER_STATS if stats else 0) | (F.RENDER_REFERENCE_SHADOW if reference else 0)
        self._check(self._lib.trb_occluded(self._h, len(rays), F.ptr(rays), F.ptr(out), flags, C.byref(st)))
        return out.astype(bool), st

    def occluded_device(self, n, d_rays, d_occluded, d_stats=None, stream=None, reference=False, stats=False):
        """trb_occluded_device: n query rays (16-byte aligned) -> n uint8 flags, enqueued on `stream` without host synchronisation."""
        flags = (F.RENDER_STATS if stats else 0) | (F.RENDER_REFERENCE_SHADOW if reference else 0)
        self._check(self._lib.trb_occluded_device(self._h, n, d_rays, d_occluded, flags, d_stats, stream))

    def illumination(self, rays, spp=1, seed=1, clamp=False, stats=None, reference=False):
        """trb_illumination: Integrator::illumination along each ILLUM_RAY_DTYPE ray, spp samples from the camera-sample streams
        (seed, key, sample + j). Returns the (n, 3) float32 means. clamp=True clamps each sample to [0, 1] first, as a render does.
        stats: None, or a Stats that receives the counters, node / triangle / instance tests included. reference=True traces shadow
        rays to the closest hit like the reference (same radiance, the reference's test counters)."""
        rays = np.ascontiguousarray(rays, dtype=F.ILLUM_RAY_DTYPE)
        out = np.zeros((len(rays), 3), np.float32)
        flags = (F.RENDER_STATS if stats is not None else 0) | (F.RENDER_REFERENCE_SHADOW if reference else 0) | (F.QUERY_CLAMP if clamp else 0)
        self._check(self._lib.trb_illumination(self._h, len(rays), F.ptr(rays), spp, seed, F.ptr(out), flags,
                                               C.byref(stats) if stats is not None else None))
        return out

    def illumination_device(self, n, d_rays, d_rgb, spp=1, seed=1, clamp=False, d_stats=None, stream=None, stats=False, reference=False):
        """trb_illumination_device: n illumination rays (48 B each, 16-byte aligned) -> n * 3 float32 means in d_rgb, enqueued on
        `stream` (a cudaStream_t as an int; None = default stream) without host synchronisation."""
        flags = (F.RENDER_STATS if stats else 0) | (F.RENDER_REFERENCE_SHADOW if reference else 0) | (F.QUERY_CLAMP if clamp else 0)
        self._check(self._lib.trb_illumination_device(self._h, n, d_rays, spp, seed, d_rgb, flags, d_stats, stream))

    # ---- shading queries: the render's BSDF and light functions on caller inputs (trace nothing) ----
    def bsdf_eval(self, records, queries):
        """trb_bsdf_eval: Material::bsdf at each INTERSECTION_DTYPE record, then BSDF::eval and BSDF::pdf of the BSDF_EVAL_QUERY_DTYPE
        query. Returns (n, 4) float32: r, g, b, pdf. A missed record or a material out of range gives zeros."""
        rec = np.ascontiguousarray(records, dtype=F.INTERSECTION_DTYPE)
        q = np.ascontiguousarray(queries, dtype=F.BSDF_EVAL_QUERY_DTYPE)
        assert len(rec) == len(q)
        out = np.zeros((len(q), 4), np.float32)
        self._check(self._lib.trb_bsdf_eval(self._h, len(q), F.ptr(rec), F.ptr(q), F.ptr(out)))
        return out

    def bsdf_eval_device(self, n, d_rec, d_q, d_out, stream=None):
        """trb_bsdf_eval_device: n records (96 B), n queries (32 B) -> n * 4 float32, device buffers 16-byte aligned, enqueued on
        `stream` (a cudaStream_t as an int; None = default stream) without host synchronisation."""
        self._check(self._lib.trb_bsdf_eval_device(self._h, n, d_rec, d_q, d_out, stream))

    def bsdf_sample(self, records, queries):
        """trb_bsdf_sample: Material::bsdf at each record, then BSDF::sample of the BSDF_SAMPLE_QUERY_DTYPE query. Returns
        BSDF_SAMPLE_DTYPE (f, pdf, wi, sampled type bits)."""
        rec = np.ascontiguousarray(records, dtype=F.INTERSECTION_DTYPE)
        q = np.ascontiguousarray(queries, dtype=F.BSDF_SAMPLE_QUERY_DTYPE)
        assert len(rec) == len(q)
        out = np.zeros(len(q), F.BSDF_SAMPLE_DTYPE)
        self._check(self._lib.trb_bsdf_sample(self._h, len(q), F.ptr(rec), F.ptr(q), F.ptr(out)))
        return out

    def bsdf_sample_device(self, n, d_rec, d_q, d_out, stream=None):
        """trb_bsdf_sample_device: n records, n queries -> n BSDF_SAMPLE_DTYPE results (32 B), device buffers 16-byte aligned."""
        self._check(self._lib.trb_bsdf_sample_device(self._h, n, d_rec, d_q, d_out, stream))

    def light_sample(self, queries):
        """trb_light_sample: Light::sample_incident of each LIGHT_QUERY_DTYPE query. Returns LIGHT_SAMPLE_DTYPE (li, pdf, wi, delta and
        the shadow ray as a QUERY_RAY_DTYPE, ready for occluded())."""
        q = np.ascontiguousarray(queries, dtype=F.LIGHT_QUERY_DTYPE)
        out = np.zeros(len(q), F.LIGHT_SAMPLE_DTYPE)
        self._check(self._lib.trb_light_sample(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def light_sample_device(self, n, d_q, d_out, stream=None):
        """trb_light_sample_device: n queries (32 B) -> n LIGHT_SAMPLE_DTYPE results (80 B), device buffers 16-byte aligned."""
        self._check(self._lib.trb_light_sample_device(self._h, n, d_q, d_out, stream))

    def light_pdf(self, queries):
        """trb_light_pdf: Light::pdf of each LIGHT_PDF_QUERY_DTYPE query. Returns (n,) float32."""
        q = np.ascontiguousarray(queries, dtype=F.LIGHT_PDF_QUERY_DTYPE)
        out = np.zeros(len(q), np.float32)
        self._check(self._lib.trb_light_pdf(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def light_pdf_device(self, n, d_q, d_pdf, stream=None):
        """trb_light_pdf_device: n queries (32 B, 16-byte aligned) -> n float32 (4-byte aligned)."""
        self._check(self._lib.trb_light_pdf_device(self._h, n, d_q, d_pdf, stream))

    def emitted(self, queries):
        """trb_emitted: Emitter::radiance of each EMIT_QUERY_DTYPE query (black for receivers). Returns (n, 3) float32."""
        q = np.ascontiguousarray(queries, dtype=F.EMIT_QUERY_DTYPE)
        out = np.zeros((len(q), 3), np.float32)
        self._check(self._lib.trb_emitted(self._h, len(q), F.ptr(q), F.ptr(out)))
        return out

    def emitted_device(self, n, d_q, d_rgb, stream=None):
        """trb_emitted_device: n queries (32 B, 16-byte aligned) -> n * 3 float32 (4-byte aligned)."""
        self._check(self._lib.trb_emitted_device(self._h, n, d_q, d_rgb, stream))

    def lights(self):
        """trb_scene_lights: the instance indices of the light list, in sample_one_light's order."""
        out = np.zeros(self.n_lights, np.uint32)
        self._check(self._lib.trb_scene_lights(self._h, F.ptr(out)))
        return out

    def to_srgb8(self, film):
        film = np.ascontiguousarray(film, dtype=np.float32)
        out = np.zeros((self.height, self.width, 3), np.uint8)
        self._check(self._lib.trb_film_to_srgb8(self._h, F.ptr(film), F.ptr(out)))
        return out


class Comm:
    """One rank of a multi-GPU job (one process per GPU): NCCL communicator owned by libtrb (trb_comm_*). The 128-byte
    unique id is created by rank 0 with ``Comm.unique_id()`` and shipped to the other ranks by any transport."""

    def __init__(self, uid, n_ranks, rank, device):
        self._lib = F.load_trb()
        h = C.c_void_p()
        self._h = None
        buf = (C.c_char * 128).from_buffer_copy(bytes(uid))
        rc = self._lib.trb_comm_create(buf, n_ranks, rank, device, C.byref(h))
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())
        self._h, self.n_ranks, self.rank, self.device = h, n_ranks, rank, device

    @staticmethod
    def unique_id():
        lib = F.load_trb()
        buf = (C.c_char * 128)()
        rc = lib.trb_nccl_unique_id(buf)
        if rc != F.TRB_OK:
            raise TrbError(rc, (lib.trb_last_error() or b"").decode())
        return bytes(buf)

    def _check(self, rc):
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())

    def reduce_film(self, d_film_ptr, n_floats, root=0, stream=None):
        """SUM-reduce a device film to `root` (in place), enqueued on `stream` (trb_comm_reduce_film: ncclReduce)."""
        self._check(self._lib.trb_comm_reduce_film(self._h, d_film_ptr, n_floats, root, stream))

    def render_sharded(self, scene, film=None, root=0, **kw):
        """trb_render_sharded: this rank's tile shard at full spp, ONE film reduce, root adds into its host film."""
        cfg = _cfg(**kw)
        if film is None and self.rank == root:
            film = np.zeros((scene.height, scene.width, 4), np.float32)
        st = F.Stats()
        self._check(self._lib.trb_render_sharded(scene._h, self._h, C.byref(cfg), root, F.ptr(film) if film is not None else None, C.byref(st)))
        return film, st

    def render_sharded_adaptive(self, scene, min_spp, max_spp, film=None, pixel_spp=None, root=0, **kw):
        """trb_render_sharded_adaptive: this rank's shard with the Adaptive sampler, ONE film reduce, root adds into its host
        film. Returns (film (None off the root), pixel_spp (height, width) uint32 with this rank's pixels filled in, Stats)."""
        cfg = _cfg(**kw)
        if film is None and self.rank == root:
            film = np.zeros((scene.height, scene.width, 4), np.float32)
        if pixel_spp is None:
            pixel_spp = np.zeros((scene.height, scene.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_render_sharded_adaptive(scene._h, self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), root,
                                                          F.ptr(film) if film is not None else None, F.ptr(pixel_spp), C.byref(st)))
        return film, pixel_spp, st

    def _sharded_aov_outputs(self, scene, root, film, albedo, normal, nearest):
        """render_aov's host arrays on the root; on the other ranks only the arrays passed (they render and reduce every AOV anyway)"""
        if self.rank == root:
            return _aov_outputs(scene.height, scene.width, film, albedo, normal, nearest)
        return film, {}, None

    def render_sharded_aov(self, scene, film=None, albedo=True, normal=True, nearest=True, root=0, **kw):
        """trb_render_sharded_aov: render_sharded with the AOVs (DESIGN.md §4 "Multi-GPU AOVs"); every rank renders its shard of the
        colour film and the three AOVs, ONE NCCL group reduces them to the root. On the root albedo / normal / nearest are as for
        Scene.render_aov and the result equals it; elsewhere they are ignored. Returns (film, aovs, Stats): film None and aovs
        empty off the root, Stats this rank's."""
        cfg = _cfg(**kw)
        film, aovs, out = self._sharded_aov_outputs(scene, root, film, albedo, normal, nearest)
        st = F.Stats()
        self._check(self._lib.trb_render_sharded_aov(scene._h, self._h, C.byref(cfg), root, F.ptr(film) if film is not None else None,
                                                     C.byref(out) if out is not None else None, C.byref(st)))
        return film, aovs, st

    def render_sharded_adaptive_aov(self, scene, min_spp, max_spp, film=None, albedo=True, normal=True, nearest=True, pixel_spp=None, root=0, **kw):
        """trb_render_sharded_adaptive_aov: render_sharded_adaptive with the AOVs, as render_sharded_aov. Returns (film, aovs,
        pixel_spp (this rank's pixels filled in), Stats)."""
        cfg = _cfg(**kw)
        film, aovs, out = self._sharded_aov_outputs(scene, root, film, albedo, normal, nearest)
        if pixel_spp is None:
            pixel_spp = np.zeros((scene.height, scene.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_render_sharded_adaptive_aov(scene._h, self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), root,
                                                              F.ptr(film) if film is not None else None,
                                                              C.byref(out) if out is not None else None, F.ptr(pixel_spp), C.byref(st)))
        return film, aovs, pixel_spp, st

    def close(self):
        if self._h is not None:
            self._lib.trb_comm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Replica(Scene):
    """A Group's replica as a Scene (trb_group_scene): every Scene call on it, without ownership; the group destroys it. Its
    DenoiseHistory objects are released when the group closes."""

    def __init__(self, group, index):
        self._lib, self._desc, self._histories = group._lib, group._desc, []
        h = self._lib.trb_group_scene(group._h, index)
        if not h:
            raise ValueError("replica %d out of range (%d devices)" % (index, len(group.devices)))
        self._h, self.device = C.c_void_p(h), group.devices[index]
        self._group = group  # keeps the replica alive while the view is
        self._read_info()

    def close(self):
        for hist in self._histories:
            hist.close()
        self._h = None


class Group:
    """One process driving several GPUs (trb_group_*): a scene replica per device, tile-sharded render, one film reduce.
    The AOV renders reduce the AOVs with the film; the denoised renders render on every device and denoise on replica 0
    (scene(0)), so their DenoiseHistory is DenoiseHistory(group.scene(0))."""

    def __init__(self, desc, devices):
        self._lib = F.load_trb()
        self._desc = desc
        devs = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        self._h = None
        rc = self._lib.trb_group_create(C.byref(desc), devs, len(devices), C.byref(h))
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())
        self._h, self.devices = h, list(devices)
        self.width, self.height = desc.film.width, desc.film.height
        self._replicas = {}

    def _check(self, rc):
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())

    def scene(self, index=0):
        """Replica `index` as a Scene (trb_group_scene), borrowed: valid until the group closes."""
        if index not in self._replicas:
            self._replicas[index] = _Replica(self, index)
        return self._replicas[index]

    @property
    def spp(self):
        return self.scene(0).spp

    def render(self, film=None, **kw):
        cfg = _cfg(**kw)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        st = F.Stats()
        rc = self._lib.trb_group_render(self._h, C.byref(cfg), F.ptr(film), C.byref(st))
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())
        return film, st

    def render_adaptive(self, min_spp, max_spp, film=None, **kw):
        """trb_group_render_adaptive: the Adaptive sampler on every replica, one reduce. Returns (film, pixel_spp, Stats)."""
        cfg = _cfg(**kw)
        if film is None:
            film = np.zeros((self.height, self.width, 4), np.float32)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        rc = self._lib.trb_group_render_adaptive(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(film), F.ptr(spp), C.byref(st))
        if rc != F.TRB_OK:
            raise TrbError(rc, (self._lib.trb_last_error() or b"").decode())
        return film, spp, st

    def render_aov(self, film=None, albedo=True, normal=True, nearest=True, **kw):
        """trb_group_render_aov: Scene.render_aov on all the group's devices (DESIGN.md §4 "Multi-GPU AOVs"): every replica renders
        its shard of the colour film and the three AOVs, ONE NCCL group reduces them to devices[0]. Arguments and result as for
        Scene.render_aov; equal to it up to float addition order (nearest exactly)."""
        cfg = _cfg(**kw)
        film, aovs, out = _aov_outputs(self.height, self.width, film, albedo, normal, nearest)
        st = F.Stats()
        self._check(self._lib.trb_group_render_aov(self._h, C.byref(cfg), F.ptr(film), C.byref(out), C.byref(st)))
        return film, aovs, st

    def render_adaptive_aov(self, min_spp, max_spp, film=None, albedo=True, normal=True, nearest=True, **kw):
        """trb_group_render_adaptive_aov: Scene.render_adaptive_aov on all the group's devices, as render_aov. Returns (film, aovs,
        pixel_spp, Stats); pixel_spp equals the one-GPU counts exactly."""
        cfg = _cfg(**kw)
        film, aovs, out = _aov_outputs(self.height, self.width, film, albedo, normal, nearest)
        spp = np.zeros((self.height, self.width), np.uint32)
        st = F.Stats()
        self._check(self._lib.trb_group_render_adaptive_aov(self._h, C.byref(cfg), C.byref(F.Adaptive(min_spp, max_spp)), F.ptr(film), C.byref(out),
                                                            F.ptr(spp), C.byref(st)))
        return film, aovs, spp, st

    def render_denoised(self, spp=0, denoise=None, **kw):
        """Scene.render_denoised with both halves rendered by render_aov on all devices, denoised on replica 0."""
        return _render_denoised(self.render_aov, self.scene(0), self.spp, spp, denoise, kw)

    def render_denoised_temporal(self, history, spp=0, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """Scene.render_denoised_temporal rendered by render_aov on all devices; `history` is a DenoiseHistory of scene(0)."""
        return _render_denoised_temporal(self.render_aov, self.scene(0), self.spp, history, spp, seed, current_frame, denoise, gradients, kw)

    def render_denoised_moments(self, history, spp=0, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """Scene.render_denoised_moments rendered by render_aov on all devices; `history` is a DenoiseHistory of scene(0)."""
        return _render_denoised_moments(self.render_aov, self.scene(0), history, spp, seed, current_frame, denoise, gradients, kw)

    def render_denoised_adaptive(self, history, min_spp, max_spp, seed=1, current_frame=0, denoise=None, gradients=False, **kw):
        """Scene.render_denoised_adaptive rendered by render_adaptive_aov on all devices; `history` is a DenoiseHistory of scene(0)."""
        return _render_denoised_adaptive(self.render_adaptive_aov, self.scene(0), history, min_spp, max_spp, seed, current_frame, denoise,
                                         gradients, kw)

    def close(self):
        if self._h is not None:
            for r in self._replicas.values():
                r.close()
            self._replicas = {}
            self._lib.trb_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bits(a):
    """uint32 view of a float32 array (bit-exact comparisons)."""
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)

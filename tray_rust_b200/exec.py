"""Reference-shaped host interface for the render path (the Python mirror of what a Rust `impl Exec` would be).

Names, argument meaning and error behaviour follow /root/reference:
  * ``Config``        exec::Config            src/exec/mod.rs:17-37
  * ``FrameInfo``     film::FrameInfo         src/film/mod.rs:26-36
  * ``RenderTarget``  film::RenderTarget      src/film/render_target.rs (the RGBW f32 film; get_render / get_renderf32 / clear)
  * ``Scene``         scene::Scene            src/scene.rs:93-182 (load_file, update_frame)
  * ``Exec``          trait exec::Exec        src/exec/mod.rs:41-49
  * ``B200``          the replacement for exec::MultiThreaded (src/exec/multithreaded.rs): one GPU, or one rank of
                      a tile-sharded multi-GPU job (``select_blocks`` exactly as exec::distrib uses it, master.rs:88-120)

Where the reference panics, these raise ``TrbError`` carrying the C ABI status.
"""
import ctypes as C
import dataclasses

import numpy as np

from . import _ffi as F
from . import api
from .api import TrbError  # noqa: F401


@dataclasses.dataclass
class FrameInfo:
    frames: int = 1
    time: float = 0.0
    start: int = 0
    end: int = 0


@dataclasses.dataclass(frozen=True)
class Adaptive:
    """sampler::Adaptive (sampler/adaptive.rs): min_spp per pixel, then more in rounds while the pixel's samples disagree,
    up to about max_spp. Both are rounded up to powers of two."""
    min_spp: int
    max_spp: int


@dataclasses.dataclass
class Config:
    """exec::Config. ``num_threads`` is accepted for signature compatibility and ignored (the GPU decides).
    ``seed`` is new: the reference seeds each worker's StdRng from the OS (multithreaded.rs:79)."""
    out_path: str = ""
    scene_file: str = ""
    spp: int = 0
    num_threads: int = 0
    frame_info: FrameInfo = dataclasses.field(default_factory=FrameInfo)
    current_frame: int = 0
    select_blocks: tuple = (0, 0)  # (start, count) into the Morton-sorted block list; count 0 = all
    seed: int = 1
    sampler: Adaptive = None  # None: LowDiscrepancy at ``spp``; an Adaptive value: the adaptive sampler (``spp`` unused)


class RenderTarget:
    """The film: width*height RGBW float32, the layout of RenderTarget::get_renderf32 (render_target.rs:243-265)."""

    def __init__(self, width, height):
        if width % 2 or height % 2:
            raise ValueError("Image with dimension (%d, %d) not evenly divided by blocks of (2, 2)" % (width, height))  # render_target.rs:43-45
        self.width, self.height = width, height
        self.pixels = np.zeros((height, width, 4), np.float32)

    def dimensions(self):
        return (self.width, self.height)

    def clear(self):
        self.pixels[...] = 0.0

    def get_renderf32(self):
        return self.pixels.reshape(-1).copy()

    def add_pixels(self, pixels):
        """film::Image::add_pixels (film/image.rs:21-33): how the distributed master combines worker films."""
        self.pixels += np.asarray(pixels, np.float32).reshape(self.pixels.shape)


class Scene:
    """scene::Scene bound to one GPU."""

    def __init__(self, gpu_scene, desc_keepalive=None):
        self._g = gpu_scene
        self._keep = desc_keepalive

    @staticmethod
    def load_file(path, device=0, width=0, height=0, spp=0):
        """Scene::load_file (scene.rs:101): returns (scene, render_target, spp, frame_info). width/height/spp > 0
        override the film section (the BASELINE.json configs do)."""
        lib = F.load_trb()
        d = C.POINTER(F.SceneDesc)()
        rc = lib.trb_desc_load_json(path.encode(), width, height, spp, C.byref(d))
        if rc != F.TRB_OK:
            raise TrbError(rc, (lib.trb_last_error() or b"").decode())
        try:
            film = d.contents.film
            fi = FrameInfo(film.frames, film.scene_time, film.start_frame, film.end_frame)
            g = api.Scene(d.contents, device)
            g._desc = None
            rt = RenderTarget(film.width, film.height)
            return Scene(g), rt, int(film.samples), fi
        finally:
            lib.trb_desc_free(d)

    @staticmethod
    def from_desc(desc, device=0):
        return Scene(api.Scene(desc, device), desc)

    @property
    def gpu(self):
        return self._g

    def update_frame(self, frame, start, end):
        self._g.update_frame(frame, start, end)

    def close(self):
        self._g.close()


class Exec:
    """trait Exec { fn render(&mut self, scene, rt, config); } (exec/mod.rs:41-49)"""

    def render(self, scene, rt, config):
        raise NotImplementedError


class B200(Exec):
    """Renders the frame ``config.current_frame`` on the scene's GPU and accumulates into ``rt``.
    Blocking, like MultiThreaded::render. ``last_stats`` holds the ray counters of the call; with an Adaptive sampler
    ``last_pixel_spp`` holds each pixel's sample count ((height, width), zero outside the selected blocks)."""

    def __init__(self, samples_per_pass=0):
        self.samples_per_pass = samples_per_pass  # 0: the whole spp in one launch
        self.last_stats = None
        self.last_pixel_spp = None

    def render(self, scene, rt, config):
        g = scene.gpu
        if rt.dimensions() != (g.width, g.height):
            raise ValueError("render target does not match the scene's film")
        if config.sampler is not None:
            _, spp, st = g.render_adaptive(config.sampler.min_spp, config.sampler.max_spp, rt.pixels, block_start=config.select_blocks[0],
                                           block_count=config.select_blocks[1], current_frame=config.current_frame, seed=config.seed)
            self.last_stats, self.last_pixel_spp = st, spp
            return st
        self.last_pixel_spp = None
        spp = config.spp if config.spp else g.spp
        spp_p2 = 1 << (max(1, spp) - 1).bit_length()
        step = self.samples_per_pass or spp_p2
        first, total = True, None
        for s0 in range(0, spp_p2, step):
            cnt = min(step, spp_p2 - s0)
            _, st = g.render(rt.pixels, spp=spp, sample_first=s0, sample_count=cnt, block_start=config.select_blocks[0],
                             block_count=config.select_blocks[1], current_frame=config.current_frame, seed=config.seed,
                             flags=0 if first else F.RENDER_NO_UPDATE)
            first = False
            if total is None:
                total = st
            else:
                for k, _t in st._fields_:
                    setattr(total, k, getattr(total, k) + getattr(st, k))
        self.last_stats = total
        return total


def get_render(scene, rt):
    """RenderTarget::get_render (render_target.rs:185-210): sRGB8, computed on the scene's GPU."""
    return scene.gpu.to_srgb8(rt.pixels)

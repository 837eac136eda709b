"""A 360-degree equirectangular view of the Cornell box from its centre, path-traced along caller rays with Scene.illumination.
The reference's perspective camera cannot produce this view; here the camera is a few lines of numpy.

    python examples/panorama.py [--width 1024] [--height 512] [--spp 64] [--out panorama.png]
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tray_rust_b200 import _ffi as F, api  # noqa: E402


def equirect_rays(width, height, centre):
    """One ray per pixel: longitude across the image (-pi at the left edge, looking down -z at the centre column), latitude from
    +y at the top row to -y at the bottom; key = the pixel's row-major index."""
    x, y = np.meshgrid(np.arange(width), np.arange(height))
    phi = (x + 0.5) / width * 2.0 * np.pi - np.pi
    theta = (y + 0.5) / height * np.pi
    q = np.zeros(width * height, F.ILLUM_RAY_DTYPE)
    q["o"] = centre
    q["d"] = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], axis=-1).reshape(-1, 3)
    q["max_t"] = np.inf
    q["key"] = np.arange(width * height)
    return q


def to_srgb8(rgb):
    """Colorf::to_srgb of the clamped means (color.rs), as trb_film_to_srgb8 converts a film."""
    v = np.clip(rgb, 0.0, 1.0)
    s = np.where(v <= 0.0031308, 12.92 * v, 1.055 * np.power(v, 1.0 / 2.4) - 0.055)
    return np.minimum(s * 255.0, 255.0).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--spp", type=int, default=64)
    ap.add_argument("--out", default="panorama.png")
    a = ap.parse_args()
    lib = F.load_trb()
    desc = C.POINTER(F.SceneDesc)()
    path = os.path.join(REPO, "tests", "golden", "scenes", "c1_cornell_box.json").encode()
    if lib.trb_desc_load_json(path, 64, 64, 1, C.byref(desc)) != F.TRB_OK:
        raise SystemExit(lib.trb_last_error().decode())
    scene = api.Scene(desc.contents)
    scene.update_frame(0, 0.0, 0.0)
    st = F.Stats()
    rgb = scene.illumination(equirect_rays(a.width, a.height, (0.0, 12.0, 0.0)), spp=a.spp, seed=1, clamp=True, stats=st)
    img = np.ascontiguousarray(to_srgb8(rgb).reshape(a.height, a.width, 3))
    if lib.trb_write_png(a.out.encode(), F.ptr(img), a.width, a.height) != F.TRB_OK:
        raise SystemExit(lib.trb_last_error().decode())
    print("%s: %dx%d at %d spp, %d rays traced in %.1f ms of GPU time" % (a.out, a.width, a.height, a.spp, st.rays_total(), st.kernel_ms))


if __name__ == "__main__":
    main()

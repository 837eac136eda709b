"""trb_tray on the GPU: single-node frame loops, the master driving two real trb_workers, trb_tray --worker against trb_worker,
and the host sRGB conversion against the device's."""
import os
import socket
import sys

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import api, exec as X

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def programs():
    H.build_programs()
    sys.path.insert(0, os.path.join(H.REPO, "tests", "golden"))
    import make_scenes
    merl = os.path.join(H.SCENES, "merl", "synthetic.binary")  # c5_tr15_like's measured material, generated where needed
    if not os.path.exists(merl):
        make_scenes.write_synthetic_merl(merl)


def assert_close_srgb(got, want):
    """Films of two renders differ only by the order of their atomic adds (about 1e-5), which can move a byte by one."""
    d = np.abs(got.astype(int) - want.astype(int))
    assert d.max() <= 1 and np.count_nonzero(d) < 1e-3 * d.size, (d.max(), np.count_nonzero(d))


def run(args, timeout=600):
    p = H.Proc(args)
    try:
        rc, out, err = p.finish(timeout=timeout)
    finally:
        p.kill()
    assert rc == 0, err
    return out


def test_single_node_keyframed_frames(tmp_path):
    d = tmp_path / "frames"
    out = run([H.TRAY, H.C5, "--spp", "1", "--start-frame", "0", "--end-frame", "2", "-o", str(d)])
    scene, _, _, _ = X.Scene.load_file(H.C5, 0, 0, 0, 1)
    try:
        pngs = []
        for k in range(3):
            png = d / ("frame%05d.png" % k)
            assert "Frame %d: rendered to '%s'" % (k, png) in out
            film, _ = scene.gpu.render(seed=1, current_frame=k)
            want = scene.gpu.to_srgb8(film)
            assert np.array_equal(api.film_to_srgb8(film), want)  # the host conversion, on a rendered film
            pngs.append(H.read_png(png))
            assert_close_srgb(pngs[-1], want)
        assert np.count_nonzero(pngs[0] != pngs[2]) > 0.05 * pngs[0].size  # the frame loop moves the animation
    finally:
        scene.close()
    assert "Rendering entire sequence took" in out


def test_single_node_one_file(tmp_path):
    png = tmp_path / "one.png"
    run([H.TRAY, H.CORNELL, "-o", str(png), "--seed", "7"])
    scene, _, _, _ = X.Scene.load_file(H.CORNELL)
    try:
        film, _ = scene.gpu.render(seed=7)
        assert_close_srgb(H.read_png(png), scene.gpu.to_srgb8(film))
    finally:
        scene.close()


def lock_block_mask(film):
    """RenderTarget::get_rendered_blocks (render_target.rs:215-241): the 2x2 lock blocks whose four weights are non-zero."""
    h, w = film.shape[:2]
    full = (film[..., 3] != 0).reshape(h // 2, 2, w // 2, 2).all(axis=(1, 3))
    return np.repeat(np.repeat(full, 2, axis=0), 2, axis=1)


@pytest.mark.parametrize("scene_path,frames,spp", [(H.CORNELL, (0, 0), 4), (H.C5, (0, 1), 1)], ids=["cornell", "c5_tr15_like"])
def test_master_and_two_workers(tmp_path, scene_path, frames, spp):
    seed = 5
    ports = [H.free_port() for _ in range(2)]
    procs = []
    d = tmp_path / "frames"
    try:
        for p in ports:
            procs.append(H.Proc([H.WORKER, "--port", str(p), "--seed", str(seed), "--spp", str(spp)]))
            procs[-1].wait_line("listening for master")
        master = H.Proc([H.TRAY, scene_path, "--master"] + ["127.0.0.1:%d" % p for p in ports]
                        + ["--start-frame", str(frames[0]), "--end-frame", str(frames[1]), "-o", str(d)])
        procs.append(master)
        rc, out, err = master.finish(timeout=600)
        assert rc == 0, err
        for w in procs[:2]:
            assert w.finish(timeout=60)[0] == 0
    finally:
        for p in procs:
            p.kill()
    scene, _, _, _ = X.Scene.load_file(scene_path, 0, 0, 0, spp)
    try:
        g = scene.gpu
        nb = g.n_blocks()
        ranges = [(0, nb // 2), (nb // 2, nb - nb // 2)]  # master.rs:88-93, 217-224
        for f in range(frames[0], frames[1] + 1):
            acc = np.zeros((g.height, g.width, 4), np.float32)
            for start, count in ranges:
                film, _ = g.render(seed=seed, block_start=start, block_count=count, current_frame=f)
                m = lock_block_mask(film)
                acc[m] += film[m]
            assert_close_srgb(H.read_png(d / ("frame%05d.png" % f)), api.film_to_srgb8(acc))
            assert "Frame %d: rendered to" % f in out
    finally:
        scene.close()


def test_host_and_device_srgb8_are_bit_identical():
    rng = np.random.default_rng(31)
    d = H.load_desc(H.CORNELL, 64, 48)
    try:
        g = api.Scene(d.contents, 0)
        for _ in range(4):
            film = H.special_film(rng, 48, 64)
            assert np.array_equal(api.film_to_srgb8(film), g.to_srgb8(film))
        g.close()
    finally:
        H.free_desc(d)


def worker_frame(args, port):
    w = H.Proc(args + ["--port", str(port), "--seed", "5", "--spp", "4"])
    try:
        w.wait_line("listening for master")
        with socket.create_connection(("127.0.0.1", port), timeout=30) as s:
            s.sendall(H.encode_instructions(H.CORNELL, (0, 0), 100, 50))
            s.settimeout(H.TIMEOUT)
            buf = H.recv_message(s)
        rc, _, err = w.finish(timeout=60)
        assert rc == 0, err
    finally:
        w.kill()
    return H.decode_frame(buf)


def test_tray_worker_sends_trb_workers_frame():
    a = worker_frame([H.TRAY, "--worker"], H.free_port())
    b = worker_frame([H.WORKER], H.free_port())
    assert a[0] == b[0] == 0 and a[1] == b[1] == (2, 2)
    assert len(a[2]) > 0 and np.array_equal(a[2], b[2])
    assert np.allclose(a[3], b[3], rtol=2e-4, atol=2e-5)

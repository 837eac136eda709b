"""trb_tray without a GPU: the distributed master (exec/distrib/master.rs) against stand-in workers written in Python, its failure
modes, the single-node argument checks, and trb_host_film_to_srgb8 (Image::get_srgb8) against the oracle."""
import os
import socket

import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import api, _ffi as F

CORNELL_REL = os.path.relpath(H.CORNELL, H.REPO)  # the master sends the scene path exactly as typed


@pytest.fixture(scope="module", autouse=True)
def programs():
    H.build_programs()


@pytest.fixture(scope="module")
def cornell_oracle():
    from oracle import pyoracle as O
    d = H.load_desc(H.CORNELL)
    o = O.OracleScene(d.contents)
    yield o
    o.close()
    H.free_desc(d)


def lock_blocks_of(rng, n, region=(40, 30)):
    """n distinct 2x2 lock blocks (pixel coordinates) inside the top-left region, so that workers overlap."""
    idx = rng.choice(region[0] * region[1], size=n, replace=False)
    return np.stack([2 * (idx % region[0]), 2 * (idx // region[0])], axis=1)


def crafted_frames(rng, n_workers, frames):
    """{(worker, frame): (blocks, pixels)} of random RGBW blocks, about a tenth of the weights zero."""
    out = {}
    for wk in range(n_workers):
        for f in frames:
            blocks = lock_blocks_of(rng, 500)
            px = rng.uniform(0.0, 2.0, size=(len(blocks), 4, 4)).astype(np.float32)
            px[..., 3] = rng.uniform(0.25, 2.0, size=px.shape[:2])
            px[..., 3][rng.random(px.shape[:2]) < 0.1] = 0.0
            out[(wk, f)] = (blocks, px)
    return out


def add_blocks(img, blocks, px):
    """Image::add_blocks (film/image.rs:36-50) in numpy, block by block."""
    for (x, y), p in zip(blocks, px):
        img[y:y + 2, x:x + 2] += p.reshape(2, 2, 4)


def start_master(workers, *extra, scene=CORNELL_REL):
    return H.Proc([H.TRAY, scene, "--master", *workers, "--start-frame", "0", "--end-frame", "1", *extra])


def accept_all(listeners):
    conns = [ls.accept()[0] for ls in listeners]
    for c in conns:
        c.settimeout(H.TIMEOUT)
    return conns


def close_all(*groups):
    for g in groups:
        for s in g:
            s.close()


def run_master_with_stand_ins(tmp_path, n_workers, order, out_arg, rng, wait_for=None):
    """The stand-ins check their Instructions, then send the crafted Frames in `order`. wait_for = (index into order, frame):
    before sending order[index], wait until the master has written that frame."""
    listeners = [H.listener() for _ in range(n_workers)]
    names = ["127.0.0.1:%d" % ls.getsockname()[1] for ls in listeners]
    sent = crafted_frames(rng, n_workers, (0, 1))
    m = start_master(names, "-o", out_arg)
    conns = []
    try:
        conns = accept_all(listeners)
        n_blocks = 100 * 75  # 800x600 in 8x8 blocks
        per = n_blocks // n_workers
        for i, c in enumerate(conns):
            count = per if i < n_workers - 1 else n_blocks - per * (n_workers - 1)
            assert H.recv_message(c) == H.encode_instructions(CORNELL_REL, (0, 1), i * per, count)
        for k, (wk, f) in enumerate(order):
            if wait_for and k == wait_for[0]:
                m.wait_line("Frame %d: rendered to" % wait_for[1])
            conns[wk].sendall(H.encode_frame(f, *sent[(wk, f)]))
        rc, out, err = m.finish()
        assert rc == 0, err
    finally:
        m.kill()
        close_all(conns, listeners)
    expect = {}
    for f in (0, 1):
        img = np.zeros((600, 800, 4), np.float32)
        for wk in range(n_workers):
            add_blocks(img, *sent[(wk, f)])
        expect[f] = img
    return out, expect, sent


def coverage(sent, n_workers, f):
    cov = np.zeros((600, 800), np.int32)
    for wk in range(n_workers):
        for x, y in sent[(wk, f)][0]:
            cov[y:y + 2, x:x + 2] += 1
    return cov


def test_master_two_stand_ins_bit_exact(tmp_path, cornell_oracle):
    rng = np.random.default_rng(11)
    d = tmp_path / "frames"
    order = [(1, 1), (0, 0), (1, 0), (0, 1)]  # frame 1 from one worker before frame 0 from the other
    out, expect, sent = run_master_with_stand_ins(tmp_path, 2, order, str(d), rng)
    assert (coverage(sent, 2, 0) == 2).any()  # the workers overlap
    for f in (0, 1):
        png = d / ("frame%05d.png" % f)
        assert "Frame %d: rendered to '%s'" % (f, png) in out
        assert "Frame %d: time between receiving first and last tile" % f in out
        # two adds from zero commute, so the image is bit-exact whatever the arrival order
        assert np.array_equal(H.read_png(png), cornell_oracle.to_srgb8(expect[f]))
    assert "Rendering entire sequence took" in out


def test_master_three_stand_ins(tmp_path, cornell_oracle):
    rng = np.random.default_rng(12)
    d = tmp_path / "frames"
    order = [(2, 1), (0, 0), (1, 1), (2, 0), (1, 0), (0, 1)]
    _, expect, sent = run_master_with_stand_ins(tmp_path, 3, order, str(d), rng)
    for f in (0, 1):
        got = H.read_png(d / ("frame%05d.png" % f)).astype(int)
        want = cornell_oracle.to_srgb8(expect[f]).astype(int)
        cov = coverage(sent, 3, f)
        assert (cov == 3).any()
        # a pixel that three workers cover is a sum of three adds in arrival order, which can move the last bit
        assert np.array_equal(got[cov < 3], want[cov < 3])
        assert np.abs(got - want).max() <= 1


def test_master_single_file_outputs(tmp_path, cornell_oracle):
    rng = np.random.default_rng(13)
    order = [(1, 1), (0, 0), (1, 0), (0, 1)]
    png = tmp_path / "one.png"
    out, expect, _ = run_master_with_stand_ins(tmp_path, 2, order, str(png), rng, wait_for=(3, 0))
    assert out.index("Frame 0: rendered to") < out.index("Frame 1: rendered to")
    assert np.array_equal(H.read_png(png), cornell_oracle.to_srgb8(expect[1]))  # rewritten by every frame: the last one stays
    ppm = tmp_path / "x.ppm"
    _, expect, _ = run_master_with_stand_ins(tmp_path, 2, order, str(ppm), rng, wait_for=(3, 0))
    assert open(ppm, "rb").read(3) == b"P6\n"
    assert np.array_equal(H.read_ppm(ppm), cornell_oracle.to_srgb8(expect[1]))


# ---- failure modes: a non-zero exit within the timeout, and a message that names the worker --------------------------------

def one_block(frame, x=0, y=0):
    return H.encode_frame(frame, [(x, y)], np.ones(16, np.float32))


FAILURES = {
    "closes_mid_frame": (lambda: one_block(0)[:30], ["hung up", "frame 0"]),
    "block_outside": (lambda: one_block(0, 800, 0), ["block (800, 0)", "outside", "frame 0"]),
    "pixel_count": (lambda: H.encode_frame(0, [(0, 0), (2, 0)], np.ones(16, np.float32)), ["pixel floats", "frame 0"]),
    "duplicate_frame": (lambda: one_block(0) + one_block(0), ["frame 0 twice"]),
    "frame_outside_range": (lambda: one_block(5), ["frame 5", "outside the range [0, 1]"]),
    "implausible_size": (lambda: one_block(0, 0, 0)[8:16] + one_block(0)[8:], ["implausible Frame size"]),
    "size_mismatch": (lambda: H.encode_frame(0, [(0, 0)], np.ones(16, np.float32), encoded_size=100) + b"\0" * 20, ["frame 0", "pixel floats"]),
}


@pytest.mark.parametrize("case", sorted(FAILURES))
def test_master_refuses_a_bad_worker(case, tmp_path):
    payload, needles = FAILURES[case]
    listeners = [H.listener() for _ in range(2)]
    names = ["127.0.0.1:%d" % ls.getsockname()[1] for ls in listeners]
    m = start_master(names, "-o", str(tmp_path))
    conns = []
    try:
        conns = accept_all(listeners)
        for c in conns:
            H.recv_message(c)
        conns[0].sendall(one_block(0))       # a good worker
        conns[1].sendall(payload())          # and a bad one
        if case == "closes_mid_frame":
            conns[1].close()
        rc, out, err = m.finish(timeout=60)
    finally:
        m.kill()
        close_all(conns, listeners)
    assert rc != 0
    assert names[1] in err, err
    for n in needles:
        assert n in err, err


def test_master_names_an_unreachable_worker():
    port = H.free_port()
    m = H.Proc([H.TRAY, CORNELL_REL, "--master", "127.0.0.1:%d" % port])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc != 0 and "failed to contact worker 127.0.0.1:%d" % port in err, err


def test_master_bare_host_means_port_63234():
    # The closed port comes second: if something does listen on 63234 here, the master only connects and then stops at the
    # closed port, before sending anything.
    port = H.free_port()
    m = H.Proc([H.TRAY, CORNELL_REL, "--master", "127.0.0.1", "127.0.0.1:%d" % port])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc != 0
    if "127.0.0.1:%d" % port in err:
        pytest.skip("something listens on 127.0.0.1:63234 on this machine")
    assert "failed to contact worker 127.0.0.1:63234" in err, err


def test_master_refuses_more_workers_than_blocks(tmp_path):
    scene = tmp_path / "tiny.json"
    scene.write_text(open(H.CORNELL).read().replace('"width":800,"height":600', '"width":16,"height":8'))
    os.symlink(os.path.join(H.SCENES, "models"), tmp_path / "models")  # the scene's meshes, relative to the scene file
    ports = [H.free_port() for _ in range(3)]
    m = H.Proc([H.TRAY, str(scene), "--master"] + ["127.0.0.1:%d" % p for p in ports])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc != 0 and "3 workers for 2 blocks" in err, err


def test_master_hang_up_before_the_last_frame(tmp_path):
    ls = H.listener()
    name = "127.0.0.1:%d" % ls.getsockname()[1]
    m = start_master([name], "-o", str(tmp_path))
    c = None
    try:
        c = ls.accept()[0]
        H.recv_message(c)
        c.sendall(one_block(0))
        c.close()
        rc, out, err = m.finish(timeout=60)
    finally:
        m.kill()
        ls.close()
        if c is not None:
            c.close()
    assert rc != 0 and "Frame 0: rendered to" in out
    assert "worker %s hung up before frame 1" % name in err, err


# ---- trb_host_film_to_srgb8 == Image::get_srgb8 --------------------------------------------------------------------------

def test_host_film_to_srgb8_matches_the_oracle():
    from oracle import pyoracle as O
    rng = np.random.default_rng(21)
    d = H.load_desc(H.CORNELL, 64, 48)
    try:
        o = O.OracleScene(d.contents)
        for _ in range(4):
            film = H.special_film(rng, 48, 64)
            assert np.array_equal(api.film_to_srgb8(film), o.to_srgb8(film))
        o.close()
    finally:
        H.free_desc(d)
    lib = F.load_trb()
    assert lib.trb_host_film_to_srgb8(4, 4, None, None) == F.TRB_INVALID_ARG
    assert lib.trb_host_film_to_srgb8(0, 0, None, None) == F.TRB_OK


# ---- single node without a GPU -----------------------------------------------------------------------------------------------

def test_single_node_argument_errors_come_before_the_scene(tmp_path):
    missing = str(tmp_path / "no_such_scene.json")  # never read: the arguments are refused first
    for args, needle in ((["--start-frame", "3", "--end-frame", "1"], "end frame 1 is before start frame 3"),
                         (["-o", str(tmp_path / "a.jpg")], "JPEG output is not built"),
                         (["-o", str(tmp_path / "a.tiff")], "unsupported image format")):
        m = H.Proc([H.TRAY, missing] + args)
        try:
            rc, _, err = m.finish(timeout=60)
        finally:
            m.kill()
        assert rc == 1 and needle in err and "no_such_scene" not in err, err


def test_single_node_without_a_gpu_exits_3(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_cli_gpu.py")
    out = tmp_path / "frames"
    m = H.Proc([H.TRAY, H.CORNELL, "-o", str(out), "--spp", "1"])
    try:
        rc, _, err = m.finish(timeout=60)
    finally:
        m.kill()
    assert rc == 3 and "no CPU fallback" in err, err
    assert out.is_dir()


def test_tray_worker_parses_instructions_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_cli_gpu.py")
    port = H.free_port()
    w = H.Proc([H.TRAY, "--worker", "--port", str(port), "-n", "4"])
    try:
        w.wait_line("listening for master")
        with socket.create_connection(("127.0.0.1", port), timeout=30) as s:
            s.sendall(H.encode_instructions(H.CORNELL, (0, 0), 100, 50))
            rc, out, err = w.finish(timeout=60)
    finally:
        w.kill()
    assert 'scene: "%s", frames: (0, 0), block_start: 100, block_count: 50' % H.CORNELL in out
    assert rc == 3 and "no CPU fallback" in err

"""AOV renders and denoised frames on the sharded and group paths, on an H100: a group of one device and a one-rank communicator
give what the one-GPU calls give; the shard decomposition the NCCL reduce sums (films added, nearest min-reduced, pixel counts
united) equals the full render on one GPU; validation refuses before anything renders and writes none of the caller's buffers;
trb_tray --devices and trb_worker --devices write what --device writes; and, on a node with two or more GPUs, Group([0, 1]) against
Scene on device 0.

Two renders of the same film are not bit-identical: the film kernels add samples into pixels with atomics, whose order varies from
run to run (DESIGN.md §2), so films compare within the film tolerance of the other multi-GPU tests (rtol 2e-4, atol 2e-5), while
nearest (an atomic minimum), pixel_spp and the counters compare exactly. Denoised frames compare bit for bit against the denoise
call on the same render, and within a stated tolerance against a separate render."""
import numpy as np
import pytest

import cli_helpers as H
from tray_rust_b200 import _ffi as F, api, scenebuild as SB
from test_queries_gpu import json_desc

pytestmark = pytest.mark.gpu
COUNTERS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation", "node_tests", "tri_tests", "inst_tests"]
MULTI = pytest.mark.skipif("__import__('torch').cuda.device_count() < 2", reason="needs two or more GPUs")

# name -> (scene description factory, current_frame); each render updates the frame itself
SCENES = {
    "c1": (lambda: json_desc("c1_cornell_box.json", 64, 48, 4), 0),
    "zoo_merl": (lambda: SB.scene_materials_zoo(64, 64, 4, SB.synthetic_merl_table()).finish(), 0),
    "keyframed": (lambda: SB.scene_animated(64, 64, 4).finish(), 2),
}


def counters(st):
    return [getattr(st, k) for k in COUNTERS]


def films_close(a, b):
    assert a.shape == b.shape and np.allclose(a, b, rtol=2e-4, atol=2e-5)


def aovs_match(got, want):
    assert sorted(got) == sorted(want)
    for k in ("albedo_w", "normal_w"):
        if k in want:
            films_close(got[k], want[k])
    assert got["nearest"].tobytes() == want["nearest"].tobytes()


def one_rank_comm():
    """A one-rank communicator, or None when libnccl.so.2 does not load in this process."""
    import torch
    torch.cuda.init()  # PyTorch's libnccl, if it has one, is the copy libtrb picks up
    try:
        return api.Comm(api.Comm.unique_id(), 1, 0, 0)
    except api.TrbError as e:
        if e.status == F.TRB_NCCL:
            return None
        raise


# ---- one device: the group and the one-rank communicator give the one-GPU result --------------------------------------------

@pytest.mark.parametrize("name", sorted(SCENES))
def test_one_device_group_and_one_rank_comm_equal_the_scene(name):
    make, frame = SCENES[name]
    s, grp = api.Scene(make()), api.Group(make(), [0])
    comm = one_rank_comm()
    kw = dict(seed=9, current_frame=frame)
    film, aovs, st = s.render_aov(**kw)
    assert (aovs["nearest"] != np.iinfo(np.uint64).max).any()
    runs = {"group": grp.render_aov(**kw)}
    if comm is not None:
        runs["sharded"] = comm.render_sharded_aov(s, **kw)
        runs["sharded_contiguous"] = comm.render_sharded_aov(s, shard_count=0xffffffff, **kw)
    for how, (f, a, t) in runs.items():
        films_close(f, film)
        aovs_match(a, aovs)
        assert counters(t) == counters(st), how
    afilm, aaovs, aspp, ast = s.render_adaptive_aov(2, 16, **kw)
    assert (aspp > 2).any()
    aruns = {"group": grp.render_adaptive_aov(2, 16, **kw)}
    if comm is not None:
        aruns["sharded"] = comm.render_sharded_adaptive_aov(s, 2, 16, **kw)
    for how, (f, a, p, t) in aruns.items():
        films_close(f, afilm)
        aovs_match(a, aaovs)
        assert p.tobytes() == aspp.tobytes() and counters(t) == counters(ast), how
    if comm is not None:
        comm.close()
    grp.close()
    s.close()


def test_null_aov_members_are_skipped_and_nearest_is_min_merged():
    make, _ = SCENES["c1"]
    s, grp = api.Scene(make()), api.Group(make(), [0])
    comm = one_rank_comm()
    prior = np.full((48, 64), np.iinfo(np.uint64).max, np.uint64)
    prior[::3] = 7  # nearer than any hit: kept by the min-merge
    film, aovs, _ = s.render_aov(albedo=None, normal=True, nearest=prior.copy(), seed=3)
    assert sorted(aovs) == ["nearest", "normal_w"] and (aovs["nearest"][::3] == 7).all()
    calls = [lambda: grp.render_aov(albedo=None, normal=True, nearest=prior.copy(), seed=3)]
    if comm is not None:
        calls.append(lambda: comm.render_sharded_aov(s, albedo=None, normal=True, nearest=prior.copy(), seed=3))
    for call in calls:
        f, a, _ = call()
        films_close(f, film)
        aovs_match(a, aovs)
    if comm is not None:
        comm.close()


# ---- what the reduce computes, on one GPU ------------------------------------------------------------------------------------

def contiguous_ranges(n_blocks, n):
    """shard_cfg's contiguous ranges (shard_count 0xffffffff): floor(B / N) blocks each, the remainder to the last rank"""
    per = n_blocks // n
    return [dict(block_start=r * per, block_count=(n_blocks - r * per) if r == n - 1 else per) for r in range(n)]


def resolved_rmse(a, b):
    """RMSE of the resolved pixel values (value / W) where the reference's weight is non-zero"""
    m = b[..., 3] != 0
    return float(np.sqrt(np.mean((a[m][:, :3] / a[m][:, 3:] - b[m][:, :3] / b[m][:, 3:]) ** 2)))


@pytest.mark.parametrize("layout", ["chunk1", "contiguous"])
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("adaptive", [False, True], ids=["ld", "adaptive"])
def test_shard_films_sum_and_nearest_min_to_the_full_render(n, layout, adaptive):
    s = api.Scene(SB.scene_materials_zoo(64, 64, 4, SB.synthetic_merl_table()).finish())
    s.update_frame()
    kw = dict(seed=21, flags=F.RENDER_NO_UPDATE)
    shards = ([dict(shard_index=r, shard_count=n, shard_chunk=1) for r in range(n)] if layout == "chunk1"
              else contiguous_ranges(s.n_blocks(), n))

    def render(**extra):
        if adaptive:
            return s.render_adaptive_aov(2, 16, **kw, **extra)
        f, a, t = s.render_aov(**kw, **extra)
        return f, a, np.zeros((64, 64), np.uint32), t

    film, aovs, spp, st = render()
    acc = {"film": np.zeros_like(film), "albedo_w": np.zeros_like(film), "normal_w": np.zeros_like(film)}
    near = np.full_like(aovs["nearest"], np.iinfo(np.uint64).max)
    spp_sum = np.zeros_like(spp)
    cams = 0
    for sh in shards:
        f, a, p, t = render(**sh)
        assert 0 < t.camera_samples < st.camera_samples  # a real part of the image, not all of it
        acc["film"] += f; acc["albedo_w"] += a["albedo_w"]; acc["normal_w"] += a["normal_w"]
        near = np.minimum(near, a["nearest"])
        assert not (spp_sum.astype(bool) & p.astype(bool)).any()  # the shards' pixels are disjoint
        spp_sum += p
        cams += t.camera_samples
    assert resolved_rmse(acc["film"], film) < 1e-5
    assert resolved_rmse(acc["albedo_w"], aovs["albedo_w"]) < 1e-5
    assert resolved_rmse(acc["normal_w"], aovs["normal_w"]) < 1e-5
    assert near.tobytes() == aovs["nearest"].tobytes()
    assert spp_sum.tobytes() == spp.tobytes() and cams == st.camera_samples


# ---- validation before anything renders ---------------------------------------------------------------------------------------

def _sentinels():
    film = np.full((32, 32, 4), 3.5, np.float32)
    return film, dict(albedo=np.full((32, 32, 4), 2.5, np.float32), normal=np.full((32, 32, 4), -1.5, np.float32),
                      nearest=np.full((32, 32), 12345, np.uint64))


@pytest.mark.parametrize("integrator", [F.INTEGRATOR_WHITTED, F.INTEGRATOR_NORMALS_DEBUG, "megakernel"])
def test_unsupported_renders_are_refused_and_write_nothing(integrator):
    b = SB.scene_materials_zoo(32, 32, 4)
    flags = 0
    if integrator == "megakernel":
        flags = F.RENDER_MEGAKERNEL
    else:
        b.integrator = (integrator, 0, 4)
    s, grp = api.Scene(b.finish()), api.Group(b.finish(), [0])
    comm = one_rank_comm()
    calls = {"group": lambda f, a: grp.render_aov(f, flags=flags, **a),
             "group_adaptive": lambda f, a: grp.render_adaptive_aov(2, 8, f, flags=flags, **a)}
    if comm is not None:
        calls["sharded"] = lambda f, a: comm.render_sharded_aov(s, f, flags=flags, **a)
        calls["sharded_adaptive"] = lambda f, a: comm.render_sharded_adaptive_aov(s, 2, 8, f, flags=flags, **a)
    for how, call in calls.items():
        film, bufs = _sentinels()
        want = (film.copy(), {k: v.copy() for k, v in bufs.items()})
        with pytest.raises(api.TrbError) as e:
            call(film, bufs)
        assert e.value.status == F.TRB_UNSUPPORTED, how
        assert film.tobytes() == want[0].tobytes() and all(bufs[k].tobytes() == want[1][k].tobytes() for k in bufs), how
    if comm is not None:
        comm.close()


def test_bad_arguments_of_a_one_rank_comm():
    comm = one_rank_comm()
    if comm is None:
        pytest.skip("libnccl.so.2 does not load in this process")
    s = api.Scene(SB.scene_materials_zoo(32, 32, 4).finish())
    lib, st, film = F.load_trb(), F.Stats(), np.zeros((32, 32, 4), np.float32)
    aov = F.AovFilm(None, None, None)
    cfg = api._cfg()
    # the root needs a film and an AOV struct; a root out of range; the Adaptive sampler owns the sample schedule
    assert lib.trb_render_sharded_aov(s._h, comm._h, cfg, 0, None, aov, st) == F.TRB_INVALID_ARG
    assert lib.trb_render_sharded_aov(s._h, comm._h, cfg, 0, F.ptr(film), None, st) == F.TRB_INVALID_ARG
    assert lib.trb_render_sharded_aov(s._h, comm._h, cfg, 1, F.ptr(film), aov, st) == F.TRB_INVALID_ARG
    assert lib.trb_render_sharded_adaptive_aov(s._h, comm._h, api._cfg(spp=4), F.Adaptive(2, 8), 0, F.ptr(film), aov, None,
                                               st) == F.TRB_INVALID_ARG
    assert not film.any()
    comm.close()


# ---- denoised renders on a group -------------------------------------------------------------------------------------------

# A group's render and a scene's render of the same frame differ by the atomic add order of their films (about 1e-7 relative);
# the denoiser's edge-stopping weights are smooth in their inputs, so the denoised frames differ by the same order. 1e-4 relative
# (plus 1e-5 absolute) is a margin of about 100 over that and far below any change a denoise parameter makes.
DENOISED_TOL = dict(rtol=1e-4, atol=1e-5)


def _denoise_cases():
    return {
        "spatial": lambda r, h, k: r.render_denoised(4, seed=5, current_frame=k),
        "temporal": lambda r, h, k: r.render_denoised_temporal(h, 4, seed=5, current_frame=k),
        "temporal_gradients": lambda r, h, k: r.render_denoised_temporal(h, 4, seed=5, current_frame=k, gradients=True),
        "moments": lambda r, h, k: r.render_denoised_moments(h, 1, seed=5, current_frame=k),
        "moment_gradients": lambda r, h, k: r.render_denoised_moments(h, 1, seed=5, current_frame=k, gradients=True),
        "adaptive": lambda r, h, k: r.render_denoised_adaptive(h, 2, 8, seed=5, current_frame=k),
    }


def _redenoise(case, scene, hist, res, k):
    """the denoise call of `case` on scene with hist, over the render outputs res of frame k (when the case's inputs are returned)"""
    if case in ("moments", "adaptive"):
        return scene.denoise_moments(hist, res[1], res[2])
    if case == "moment_gradients":
        return scene.denoise_moments_gradient(hist, res[1], res[2], (5 + k) % (1 << 32))
    return None  # the half films of the two-half modes are not returned


@pytest.mark.parametrize("case", sorted(_denoise_cases()))
def test_one_device_group_denoised_helpers_equal_the_scene_helpers(case):
    call = _denoise_cases()[case]
    make = lambda: SB.scene_animated(64, 64, 4).finish()  # noqa: E731
    s, grp = api.Scene(make()), api.Group(make(), [0])
    hs, hg = api.DenoiseHistory(s), api.DenoiseHistory(grp.scene(0))
    check = api.Scene(make())
    hc = api.DenoiseHistory(check)
    for k in range(3):
        want, got = call(s, hs, k), call(grp, hg, k)
        assert len(want) == len(got)
        assert np.allclose(got[0], want[0], **DENOISED_TOL), (case, k, float(np.abs(got[0] - want[0]).max()))
        films_close(got[1], want[1])
        aovs_match(got[2], want[2])
        if case == "adaptive":
            assert got[3].tobytes() == want[3].tobytes()
        # the group's helper is the denoise call on replica 0 over the group's own render, bit for bit
        check.update_frame(*((k, k / 4.0, (k + 1) / 4.0)))
        redo = _redenoise(case, check, hc, got, k)
        if redo is not None:
            assert redo.tobytes() == got[0].tobytes(), (case, k)
    grp.close()


def test_group_replica_view_is_borrowed():
    grp = api.Group(SB.scene_materials_zoo(16, 16, 4).finish(), [0])
    r = grp.scene(0)
    assert r is grp.scene(0) and (r.width, r.height) == (16, 16) and grp.spp == 4
    h = api.DenoiseHistory(r)
    grp.close()
    assert r._h is None and h._h is None
    with pytest.raises(ValueError):
        api.Group(SB.scene_materials_zoo(16, 16, 4).finish(), [0]).scene(1)


# ---- the command line ----------------------------------------------------------------------------------------------------------

def assert_close_srgb(got, want):
    """Two renders' films differ by the order of their atomic adds (about 1e-5), which can move a byte by one."""
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


@pytest.mark.parametrize("mode", [[], ["--denoise"], ["--denoise-temporal", "--temporal-gradients"], ["--denoise-moments", "--moment-gradients"],
                                  ["--adaptive", "2", "8", "--denoise-moments"]],
                         ids=["plain", "denoise", "temporal_gradients", "moment_gradients", "adaptive_moments"])
def test_tray_devices_0_writes_what_device_0_writes(tmp_path, mode):
    H.build_programs()
    spp = [] if "--adaptive" in mode else ["--spp", "4"]
    common = [H.CORNELL, "--seed", "7", "--start-frame", "0", "--end-frame", "1"] + spp + mode
    one, group = tmp_path / "one", tmp_path / "group"
    run([H.TRAY] + common + ["--device", "0", "-o", str(one)])
    out = run([H.TRAY] + common + ["--devices", "0", "-o", str(group)])
    for k in range(2):
        assert "Frame %d: rendered to" % k in out
        assert_close_srgb(H.read_png(group / ("frame%05d.png" % k)), H.read_png(one / ("frame%05d.png" % k)))


def _master_with_one_worker(tmp_path, worker_args, name):
    port = H.free_port()
    d = tmp_path / name
    w = H.Proc([H.WORKER, "--port", str(port), "--seed", "5", "--spp", "4"] + worker_args)
    procs = [w]
    try:
        w.wait_line("listening for master")
        m = H.Proc([H.TRAY, H.CORNELL, "--master", "127.0.0.1:%d" % port, "-o", str(d)])
        procs.append(m)
        rc, _, err = m.finish(timeout=600)
        assert rc == 0, err
        assert w.finish(timeout=60)[0] == 0
    finally:
        for p in procs:
            p.kill()
    return H.read_png(d / "frame00000.png")


def test_master_driving_a_devices_worker_writes_the_device_frame(tmp_path):
    H.build_programs()
    assert_close_srgb(_master_with_one_worker(tmp_path, ["--devices", "0"], "group"), _master_with_one_worker(tmp_path, ["--device", "0"], "one"))


# ---- two or more GPUs -------------------------------------------------------------------------------------------------------

@MULTI
@pytest.mark.parametrize("name", sorted(SCENES))
def test_group_of_two_equals_the_scene(name):
    make, frame = SCENES[name]
    s, grp = api.Scene(make(), 0), api.Group(make(), [0, 1])
    kw = dict(seed=9, current_frame=frame)
    film, aovs, st = s.render_aov(**kw)
    f, a, t = grp.render_aov(**kw)
    assert resolved_rmse(f, film) < 1e-5 and resolved_rmse(a["albedo_w"], aovs["albedo_w"]) < 1e-5
    assert resolved_rmse(a["normal_w"], aovs["normal_w"]) < 1e-5
    assert a["nearest"].tobytes() == aovs["nearest"].tobytes() and counters(t) == counters(st)
    film, aovs, spp, st = s.render_adaptive_aov(2, 16, **kw)
    f, a, p, t = grp.render_adaptive_aov(2, 16, **kw)
    assert resolved_rmse(f, film) < 1e-5 and resolved_rmse(a["albedo_w"], aovs["albedo_w"]) < 1e-5
    assert a["nearest"].tobytes() == aovs["nearest"].tobytes() and p.tobytes() == spp.tobytes() and counters(t) == counters(st)
    grp.close()


@MULTI
@pytest.mark.parametrize("case", sorted(_denoise_cases()))
def test_group_of_two_denoised_helpers_equal_the_scene_helpers(case):
    # the two-GPU sum adds the shards' films in another order than one GPU's atomics: the same 1e-7-relative difference as two
    # one-GPU renders, so the same tolerance holds
    call = _denoise_cases()[case]
    make = lambda: SB.scene_animated(64, 64, 4).finish()  # noqa: E731
    s, grp = api.Scene(make(), 0), api.Group(make(), [0, 1])
    hs, hg = api.DenoiseHistory(s), api.DenoiseHistory(grp.scene(0))
    for k in range(3):
        want, got = call(s, hs, k), call(grp, hg, k)
        assert np.allclose(got[0], want[0], **DENOISED_TOL), (case, k, float(np.abs(got[0] - want[0]).max()))
    grp.close()


@MULTI
def test_group_of_two_refuses_replicas_of_different_film_sizes_and_writes_nothing():
    b = SB.scene_materials_zoo(32, 32, 4)
    grp = api.Group(b.finish(), [0, 1])
    lib = F.load_trb()
    assert lib.trb_scene_replace_settings(lib.trb_group_scene(grp._h, 1), F.Film(**dict(b.film, width=64)), None) == F.TRB_OK
    for call in (lambda f, a: grp.render_aov(f, **a), lambda f, a: grp.render_adaptive_aov(2, 8, f, **a)):
        film, bufs = _sentinels()
        want = (film.copy(), {k: v.copy() for k, v in bufs.items()})
        with pytest.raises(api.TrbError) as e:
            call(film, bufs)
        assert e.value.status == F.TRB_INVALID_ARG and "different film sizes" in str(e.value)
        assert film.tobytes() == want[0].tobytes() and all(bufs[k].tobytes() == want[1][k].tobytes() for k in bufs)
    grp.close()


@MULTI
def test_tray_devices_0_1_denoise_moments_is_close_to_device_0(tmp_path):
    H.build_programs()
    common = [H.CORNELL, "--seed", "7", "--spp", "4", "--denoise-moments"]
    run([H.TRAY] + common + ["--device", "0", "-o", str(tmp_path / "one.png")])
    run([H.TRAY] + common + ["--devices", "0,1", "-o", str(tmp_path / "two.png")])
    assert_close_srgb(H.read_png(tmp_path / "two.png"), H.read_png(tmp_path / "one.png"))

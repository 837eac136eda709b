"""The Adaptive sampler on the stream-ordered and multi-GPU render paths: trb_render_adaptive_device (device film, a caller's
stream, no host synchronisation), trb_render_sharded_adaptive and trb_group_render_adaptive, each against the blocking
trb_render_adaptive on one H100. Per-pixel sample counts and ray counters must be equal, films equal up to the order of
the float additions."""
import ctypes as C
import os

import numpy as np
import pytest

from tray_rust_b200 import _ffi as F, api, dist, scenebuild as SB

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SCENES = os.path.join(HERE, "golden", "scenes")
RAYS = ["camera_samples", "rays_primary", "rays_shadow", "rays_mis", "rays_continuation"]


def torch():
    import torch as t
    return t


def counters(st):
    return [getattr(st, k) for k in RAYS]


def films_close(a, b):
    assert np.allclose(a, b, rtol=2e-4, atol=2e-5)


def c2_scene():
    lib = F.load_trb()
    d = C.POINTER(F.SceneDesc)()
    assert lib.trb_desc_load_json(os.path.join(SCENES, "c2_smallpt.json").encode(), 128, 128, 16, C.byref(d)) == F.TRB_OK, lib.trb_last_error()
    g = api.Scene(d.contents)
    g._desc = None  # trb_scene_create deep-copies the description
    lib.trb_desc_free(d)
    return g


SCENE_MAKERS = {
    "c2_smallpt": c2_scene,
    "zoo_split": lambda: api.Scene(SB.scene_materials_zoo(64, 64, 8, SB.synthetic_merl_table()).finish()),
    "keyframed": lambda: api.Scene(SB.scene_animated(48, 48, 4, frames=4, scene_time=1.0, animated_fov=True).finish()),
}


class DeviceOut:
    """torch buffers of one device render: film (h, w, 4) f32, pixel counts (h, w) u32 as int32, trb_stats (72 bytes)."""

    def __init__(self, g, stream=None):
        T = torch()
        self.film = T.zeros((g.height, g.width, 4), dtype=T.float32, device="cuda:%d" % g.device)
        self.spp = T.zeros((g.height, g.width), dtype=T.int32, device=self.film.device)
        self.stats = T.zeros(9, dtype=T.int64, device=self.film.device)
        if stream is not None:
            stream.wait_stream(T.cuda.current_stream(self.film.device))  # the zeros are written on the current stream

    def render(self, g, mn, mx, stream=None, **kw):
        g.render_adaptive_device(mn, mx, self.film.data_ptr(), self.spp.data_ptr(), self.stats.data_ptr(),
                                 stream.cuda_stream if stream is not None else None, **kw)

    def host(self):
        st = F.Stats.from_buffer_copy(self.stats.cpu().numpy().tobytes())
        return self.film.cpu().numpy(), self.spp.cpu().numpy().view(np.uint32), st


def device_render(g, mn, mx, **kw):
    T = torch()
    s = T.cuda.Stream(device=g.device)
    out = DeviceOut(g, s)
    out.render(g, mn, mx, s, **kw)
    s.synchronize()
    return out.host()


@pytest.mark.parametrize("name", sorted(SCENE_MAKERS))
@pytest.mark.parametrize("shadow", [0, F.RENDER_REFERENCE_SHADOW], ids=["any_hit", "reference_shadow"])
def test_device_path_matches_the_host_path(name, shadow):
    g = SCENE_MAKERS[name]()
    g.update_frame(0, 0.0, 0.25)
    kw = dict(seed=7, flags=shadow | F.RENDER_NO_UPDATE)
    hf, hspp, hst = g.render_adaptive(2, 16, **kw)
    df, dspp, dst = device_render(g, 2, 16, **kw)
    assert (dspp == hspp).all(), "per-pixel sample counts differ: %d pixels" % int((dspp != hspp).sum())
    assert counters(dst) == counters(hst) and int(dspp.sum()) == dst.camera_samples
    assert (hspp > 2).any(), "some pixel should refine"
    films_close(df, hf)


def test_call_returns_without_waiting_for_the_stream():
    T = torch()
    g = c2_scene()
    g.update_frame(0, 0.0, 0.0)
    kw = dict(seed=3, flags=F.RENDER_NO_UPDATE)
    hf, hspp, hst = g.render_adaptive(2, 32, **kw)
    device_render(g, 2, 32, **kw)  # first use allocates the sampler state and the path state (that may synchronise)
    s = T.cuda.Stream()
    out = DeviceOut(g, s)
    with T.cuda.stream(s):
        T.cuda._sleep(2_000_000_000)  # about a second of GPU time ahead of the render
    out.render(g, 2, 32, s, **kw)
    assert not s.query(), "the call waited for its stream"
    with T.cuda.stream(s):  # stream order: these see the finished film
        snap = out.film.clone()
        total = out.film.sum(dim=(0, 1))
    s.synchronize()
    df, dspp, dst = out.host()
    assert (dspp == hspp).all() and counters(dst) == counters(hst)
    films_close(df, hf)
    assert T.equal(snap, out.film)
    assert np.allclose(total.cpu().numpy(), df.reshape(-1, 4).sum(axis=0, dtype=np.float64), rtol=1e-4)


def live_blocks_per_round(spp, blocks, sch):
    """blocks with a pixel still sampling at the start of each round, from the final counts"""
    mn, _, step, mpp = sch
    rounds = 1 + (mpp - mn) // step
    per_block = np.array([spp[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8].max() for bx, by in blocks])
    return [len(blocks)] + [int((per_block > mn + (r - 1) * step).sum()) for r in range(1, rounds)]


@pytest.mark.parametrize("name", ["c4_margins", "keyframed"])
def test_mostly_empty_passes_change_only_addition_order(name):
    # c4_margins: the Cornell box in a 2:1 frame, whose black margins stop sampling after round 0, so the late rounds keep
    # fewer blocks than the selection and their last passes start past the live count. keyframed: the per-path transform
    # tables of passes that are only partly live.
    g = api.Scene(SB.scene_c4(2000, 128, 64, 1).finish()) if name == "c4_margins" else SCENE_MAKERS[name]()
    g.update_frame(0, 0.0, 0.25)
    kw = dict(seed=5, flags=F.RENDER_NO_UPDATE)
    df, dspp, dst = device_render(g, 2, 32, **kw)
    sch = api.adaptive_schedule(2, 32)
    bp = 4  # blocks per pass in the rounds after the first (16 in round 0): every round is several passes
    g.set_option("pass.paths", 64 * sch[2] * bp)
    sf, sspp, sst = device_render(g, 2, 32, **kw)
    hf, hspp, hst = g.render_adaptive(2, 32, **kw)
    g.set_option("pass.paths", 1 << 24)
    nb = g.n_blocks()
    live = live_blocks_per_round(dspp, g.block_list(), sch)
    if name == "c4_margins":
        assert any(-(-n // bp) < -(-nb // bp) for n in live[1:]), ("no round enqueued a pass past its live blocks", live)
    for f, spp, st in ((sf, sspp, sst), (hf, hspp, hst)):
        assert (spp == dspp).all() and counters(st) == counters(dst)
        films_close(f, df)


def test_shards_on_one_gpu_add_up_to_one_call():
    T = torch()
    g = c2_scene()
    g.update_frame(0, 0.0, 0.0)
    kw = dict(seed=9, flags=F.RENDER_NO_UPDATE)
    ff, fspp, fst = device_render(g, 2, 32, **kw)
    nb = g.n_blocks()
    layouts = {"interleaved": [dict(shard_index=i, shard_count=3, shard_chunk=8) for i in range(3)],
               "contiguous": [dict(zip(("block_start", "block_count"), dist.shard_blocks(nb, i, 3))) for i in range(3)]}
    for name, shards in layouts.items():
        s = T.cuda.Stream()
        out = DeviceOut(g, s)  # one film, accumulated over the shards
        spps, rays = [], np.zeros(len(RAYS), np.int64)
        for sh in shards:
            one = DeviceOut(g, s)
            out.render(g, 2, 32, s, **kw, **sh)
            one.render(g, 2, 32, s, **kw, **sh)  # the same shard alone, for its own counts and counters
            s.synchronize()
            _, spp, st = one.host()
            spps.append(spp)
            rays += np.array(counters(st), np.int64)
        s.synchronize()
        film, _, st = out.host()
        assert counters(st) == rays.tolist() == counters(fst), name
        assert ((np.stack(spps) > 0).sum(axis=0) == 1).all(), name + ": shards must be disjoint and cover the image"
        assert (sum(spps) == fspp).all(), name + ": a pixel's count depends on its shard"
        films_close(film, ff)


def test_error_statuses_of_the_new_entry_points():
    T = torch()
    desc = SB.scene_materials_zoo(16, 16, 4).finish()
    g = api.Scene(desc)
    g.update_frame(0, 0.0, 0.0)
    out = DeviceOut(g)
    grp = api.Group(SB.scene_materials_zoo(16, 16, 4).finish(), [0])
    comm = one_rank_comm()
    bad = [(dict(spp=4), F.TRB_INVALID_ARG), (dict(sample_first=1), F.TRB_INVALID_ARG), (dict(sample_count=2), F.TRB_INVALID_ARG),
           (dict(flags=F.RENDER_MEGAKERNEL), F.TRB_UNSUPPORTED)]
    calls = {"device": lambda mn, mx, **kw: out.render(g, mn, mx, **kw),
             "group": lambda mn, mx, **kw: grp.render_adaptive(mn, mx, **kw)}
    if comm is not None:
        calls["sharded"] = lambda mn, mx, **kw: comm.render_sharded_adaptive(g, mn, mx, **kw)
    for name, call in calls.items():
        for kw, status in bad + [(dict(mn=8, mx=4), F.TRB_INVALID_ARG)]:
            kw = dict(kw)
            mn, mx = kw.pop("mn", 2), kw.pop("mx", 8)
            with pytest.raises(api.TrbError) as e:
                call(mn, mx, **kw)
            assert e.value.status == status, (name, kw)
    b = SB.scene_materials_zoo(16, 16, 4)
    b.integrator = (F.INTEGRATOR_WHITTED, 0, 4)
    w = api.Scene(b.finish())
    w.update_frame(0, 0.0, 0.0)
    with pytest.raises(api.TrbError) as e:
        out.render(w, 2, 8)
    assert e.value.status == F.TRB_UNSUPPORTED
    wg = api.Group(b.finish(), [0])
    with pytest.raises(api.TrbError) as e:
        wg.render_adaptive(2, 8)
    assert e.value.status == F.TRB_UNSUPPORTED
    if comm is not None:
        with pytest.raises(api.TrbError) as e:
            comm.render_sharded_adaptive(w, 2, 8)
        assert e.value.status == F.TRB_UNSUPPORTED
        lib = F.load_trb()  # the root rank needs a film
        st = F.Stats()
        rc = lib.trb_render_sharded_adaptive(g._h, comm._h, C.byref(api._cfg()), C.byref(F.Adaptive(2, 8)), 0, None, None, C.byref(st))
        assert rc == F.TRB_INVALID_ARG
        comm.close()
    with pytest.raises(api.TrbError) as e:  # the device path never updates the frame
        api.Scene(desc).render_adaptive_device(2, 8, out.film.data_ptr())
    assert e.value.status == F.TRB_INVALID_ARG
    T.cuda.synchronize()


def one_rank_comm():
    """A one-rank communicator, or None when libnccl.so.2 does not load in this process."""
    torch()  # PyTorch's libnccl, if it has one, is the copy libtrb picks up
    try:
        return api.Comm(api.Comm.unique_id(), 1, 0, 0)
    except api.TrbError as e:
        if e.status == F.TRB_NCCL:
            return None
        raise


def test_one_rank_sharded_call_equals_the_single_gpu_call():
    comm = one_rank_comm()
    if comm is None:
        pytest.skip("libnccl.so.2 does not load in this process: %s" % (F.load_trb().trb_last_error() or b"").decode())
    g = c2_scene()
    kw = dict(seed=11, current_frame=0)
    hf, hspp, hst = g.render_adaptive(2, 32, **kw)
    for extra in ({}, dict(shard_count=0xffffffff)):
        film, spp, st = comm.render_sharded_adaptive(g, 2, 32, **kw, **extra)
        assert (spp == hspp).all() and counters(st) == counters(hst), extra
        films_close(film, hf)
    comm.close()


def test_one_device_group_equals_the_single_gpu_call():
    desc = SB.scene_materials_zoo(64, 64, 8, SB.synthetic_merl_table()).finish()
    g = api.Scene(desc)
    hf, hspp, hst = g.render_adaptive(2, 16, seed=13)
    grp = api.Group(SB.scene_materials_zoo(64, 64, 8, SB.synthetic_merl_table()).finish(), [0])
    film, spp, st = grp.render_adaptive(2, 16, seed=13)
    assert (spp == hspp).all() and counters(st) == counters(hst)
    films_close(film, hf)
    grp.close()

"""The blocking host forms on an H100 free what they stage when the launch after staging is refused (DESIGN.md §8 "Error behaviour").

On a scene with wide mesh leaves the option-selected experimental trace variants are refused with TRB_UNSUPPORTED once the wavefront
runs, which the sample renders reach after their outputs are staged in device buffers. Repeated refused calls of each sample render,
plain and Adaptive, with and without AOV records, leave the device's free memory as it was.
"""
import pytest

from tray_rust_b200 import _ffi as F, api
from test_illumination_gpu import SCENES

pytestmark = pytest.mark.gpu


def test_sample_renders_refused_after_staging_free_their_buffers():
    import torch
    desc, frame = SCENES["zoo"]()
    w = api.Scene(desc)
    w.set_option("trace.wide_leaf", 1)
    w.update_frame(*frame)
    calls = {"render_samples": lambda: w.render_samples(spp=2, seed=1),
             "render_samples_aov": lambda: w.render_samples_aov(spp=2, seed=1),
             "render_samples_adaptive": lambda: w.render_samples_adaptive(2, 8, seed=1),
             "render_samples_adaptive_aov": lambda: w.render_samples_adaptive_aov(2, 8, seed=1)}
    for call in calls.values():  # the scene's own buffers (path state, AOV records, Adaptive state, block list) exist from here on
        call()
    w.set_option("trace.pipe", 0)
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        for name, call in calls.items():
            with pytest.raises(api.TrbError) as e:
                call()
            assert e.value.status == F.TRB_UNSUPPORTED and "trace.wide_leaf" in str(e.value), name
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free
    w.set_option("trace.pipe", 36)
    w.render_samples(spp=2, seed=1)
    w.close()

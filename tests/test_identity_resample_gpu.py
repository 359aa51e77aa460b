"""The real resample kernels on store inputs known exactly: geometries whose resample returns the loaded pixels (F == p, pinned
on the oracle by tests/test_identity_resample.py), on a 4096 x 4096 frame of 16 x 16 blocks that puts every (colour, alpha)
byte pair over every canvas alpha byte.  Each kernel's store epilogue then sees all 2^24 (colour, alpha, canvas alpha) inputs
that a BGRA frame can give it:
  * the tile kernel: Box 1:1;
  * the generic pair: Box 1:1 with OPT_FORCE_GENERIC;
  * the ring kernel: Box 2:1 on the frame with every pixel doubled into a constant 2 x 2 block.
Every compositing mode, both working spaces, no matrix, sepia (the tile kernel's 3x3 form) and sepia with a bias (the general
form), bit-exact against oracle.scale_and_render; the expected frame is computed once and every kernel is compared with it."""
import numpy as np
import pytest

import oracle
from tests import util
from tests.test_identity_resample import MATTE, canvas, doubled, matrices, source

pytestmark = pytest.mark.gpu
N = 4096


@pytest.fixture(scope="module")
def ifb():
    import imageflow_b200
    assert imageflow_b200.device_count() > 0, "CUDA extension loaded but no device: GPU tests cannot fall back"
    return imageflow_b200


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def frames(torch_mod):
    src, cv = source(), canvas()
    assert src.shape == (N, N, 4)
    return src, cv, torch_mod.from_numpy(src).cuda(), torch_mod.from_numpy(doubled(src)).cuda()


def _run(ifb, torch, ti, tc, linear, compose, m, force_generic):
    b = ifb.Batch(0)
    assert b.ring_status()[0], b.ring_status()[1]
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, int(force_generic))
    p = ifb.ScaleAndRenderParams(w=N, h=N, interpolation_filter=ifb.Filter(24), scale_in_colorspace=ifb.WorkingFloatspace(int(linear)))
    b.scale_and_render_many([(ifb.BitmapWindow.from_torch(ti, alpha_meaningful=True),
                              ifb.BitmapWindow.from_torch(tc, compose=ifb.BitmapCompositing(compose), matte_bgra=MATTE), p, m)],
                            stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    cnt = dict(fused=b.fused_jobs, tile=b.tile_jobs, generic=b.generic_jobs)
    b.close()
    return cnt


@pytest.mark.parametrize("linear", [True, False], ids=["linear", "srgb"])
@pytest.mark.parametrize("compose", [0, 1, 2], ids=["replace", "blend_self", "blend_matte"])
def test_every_kernel_on_every_store_input(ifb, torch_mod, frames, linear, compose):
    torch = torch_mod
    src, cv, t_src, t_src2 = frames
    kernels = [("tile", t_src, False), ("generic", t_src, True), ("fused", t_src2, False)]
    for name, m in matrices().items():
        exp = cv.copy()
        oracle.scale_and_render(src, exp, filter=24, linear=linear, alpha_meaningful=True, compose=compose, matte=MATTE, color_matrix=m)
        for kind, ti, force in kernels:
            tc = torch.from_numpy(cv).cuda()
            cnt = _run(ifb, torch, ti, tc, linear, compose, m, force)
            assert cnt[kind] == 1 and sum(cnt.values()) == 1, (kind, name, cnt)
            got = tc.cpu().numpy()
            assert np.array_equal(got, exp), (kind, name, util.diff_stats(got, exp))

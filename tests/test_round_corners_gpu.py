"""Rounded corners on the GPU (round_corners_kernel), bit-exact against the oracle: through the drop-in call on host windows and
through Batch.round_corners on device windows, with mixed batches, odd sizes, padded strides, sub-windows of larger bitmaps whose
other bytes must stay as they were, and 4K / 8K frames."""
import numpy as np
import pytest

from tests import round_corners_oracle as rco
from tests.cpu_emu.run_round_corners_cases import RADII

pytestmark = pytest.mark.gpu


def _mode(kind, radius):
    import imageflow_b200 as ifb
    return ifb.RoundCornersMode(kind, tuple(float(v) for v in radius))


def _jobs(rng, n):
    out = []
    for i in range(n):
        w, h = [(int(rng.integers(1, 60)), int(rng.integers(1, 60))), (int(rng.integers(60, 700)), int(rng.integers(60, 500)))][i % 2]
        kind = int(rng.integers(0, 5))
        radius = [float(rng.choice(RADII)) if rng.random() < 0.3 else float(rng.uniform(0, min(w, h) * 0.7)) for _ in range(4)]
        if kind in (0, 3):
            radius = [float(rng.uniform(-10, 120)) for _ in range(4)]
        matte = tuple(int(v) for v in rng.integers(0, 256, 4)) if rng.random() < 0.8 else (0, 0, 0, 0)
        out.append((w, h, kind, radius, matte))
    return out


def _noise(rng, shape):
    a = rng.integers(0, 256, shape, dtype=np.uint8)
    a.reshape(-1)[3::4][rng.random(a.size // 4) < 0.2] = 0
    return a


def test_drop_in_matches_oracle_on_sub_windows():
    import imageflow_b200 as ifb
    assert ifb.device_count() > 0
    rng = np.random.default_rng(11)
    for (w, h, kind, radius, matte) in _jobs(rng, 80) + [(3840, 2160, 1, (100.0,) * 4, (0, 0, 0, 0)), (3840, 2160, 2, (0,) * 4, (30, 60, 90, 255)),
                                                        (7680, 4320, 3, (10.0, 20.0, 30.0, 40.0), (255, 255, 255, 128))]:
        ox, oy, pad = int(rng.integers(0, 5)), int(rng.integers(0, 4)), int(rng.integers(0, 3))
        big = _noise(rng, (h + oy + 2, w + ox + pad + 1, 4))
        exp = big.copy()
        rco.round_corners(exp[oy:oy + h, ox:ox + w], kind, radius, matte)
        win = ifb.BitmapWindow.from_numpy(big).window(ox, oy, ox + w, oy + h)
        ifb.flow_bitmap_bgra_clear_around_rounded_corners(win, _mode(kind, radius), matte)
        assert np.array_equal(big, exp), (w, h, kind, radius, matte, np.argwhere(np.any(big != exp, axis=2))[:4].tolist())


def test_batch_matches_oracle_in_one_launch():
    import torch
    import imageflow_b200 as ifb
    assert ifb.device_count() > 0 and torch.cuda.is_available()
    b = ifb.Batch(0)
    rng = np.random.default_rng(12)
    for n in (1, 7, 64):
        jobs = _jobs(rng, n)
        if n == 1:
            jobs.append((30, 20, 1, [0.0] * 4, (1, 2, 3, 4)))              # a job with nothing to do: no launch of its own
        # windows stacked in one device bitmap, each at a random column offset, with gap rows and a padded pitch
        bw = max(w for w, *_ in jobs) + 9
        pitch = (bw * 4 + 63) // 64 * 64 + 4 * int(rng.integers(0, 4))
        rows = sum(h + 1 for _, h, *_ in jobs) + 1
        host = _noise(rng, (rows, pitch))
        exp = host.copy()
        dev = torch.from_numpy(host).cuda()
        batch_jobs, y, touched = [], 1, 0
        for (w, h, kind, radius, matte) in jobs:
            x0 = int(rng.integers(0, bw - w + 1))
            view = np.lib.stride_tricks.as_strided(exp.reshape(-1)[y * pitch + x0 * 4:], (h, w, 4), (pitch, 4, 1))
            touched += int(rco.round_corners(view, kind, radius, matte, want_mask=True).any())
            win = ifb.BitmapWindow(dev.data_ptr() + y * pitch + x0 * 4, w, h, pitch, _keep=dev)
            batch_jobs.append((win, _mode(kind, radius), matte))
            y += h + 1
        before = b.kernel_launches
        b.round_corners(batch_jobs, stream="own")
        b.sync()
        assert b.kernel_launches == before + (1 if touched else 0)        # one launch, none when no job touches a pixel
        got = dev.cpu().numpy()
        assert np.array_equal(got, exp), (n, np.argwhere(got != exp)[:4].tolist())


def test_batch_4k_and_8k_frames():
    import torch
    import imageflow_b200 as ifb
    b = ifb.Batch(0)
    rng = np.random.default_rng(13)
    for (w, h, kind, radius) in [(3840, 2160, 1, (100.0,) * 4), (3840, 2160, 2, (0,) * 4), (2160, 3840, 2, (0,) * 4),
                                 (7680, 4320, 4, (400.0, 0.3, 2000.0, 77.7)), (7680, 4320, 0, (100.0,) * 4)]:
        host = _noise(rng, (h, w, 4))
        exp = host.copy()
        rco.round_corners(exp, kind, radius, (5, 6, 7, 200))
        dev = torch.from_numpy(host).cuda()
        b.round_corners([(ifb.BitmapWindow.from_torch(dev), _mode(kind, radius), (5, 6, 7, 200))], stream="own")
        b.sync()
        assert torch.equal(dev.cpu(), torch.from_numpy(exp)), (w, h, kind)

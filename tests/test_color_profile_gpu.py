"""Colour profiles to sRGB on the GPU (transform_to_srgb_kernel through Batch.transform_to_srgb), byte for byte against the oracle of
tests/profile_oracle.py fed the planner's tables: every RGB triple of every fixture profile in place with noise and cut-out alpha; 4K
frames with padded strides and sub-windows in sentinel bytes; decoder rows of all four formats against pixel_convert followed by the
in-place transform; calls of 1, 7, 64 and 1024 jobs with mixed profiles as one launch; sRGB and zero-area jobs that write nothing;
one refused profile that fails the whole call; and the config-2 resample of a transformed Display P3 frame against the oracle."""
import os

import numpy as np
import pytest

import oracle
from tests import pixel_convert_oracle as po
from tests import profile_oracle as pf

pytestmark = pytest.mark.gpu
GOLDEN_GRAY = os.path.join(os.path.dirname(__file__), "golden", "gray.icc")


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _profiles():
    ifb = _ifb()
    out = {n: (ifb.SourceProfile.icc(b) if k == "icc" else ifb.SourceProfile.icc_gray(b)) for n, (k, b) in pf.fixtures().items()}
    out["golden_gray"] = ifb.SourceProfile.icc_gray(open(GOLDEN_GRAY, "rb").read())
    return out


PROFILE_NAMES = sorted(list(pf.fixtures()) + ["golden_gray"])


@pytest.fixture(scope="module")
def lut16k():
    from tests import cpu_emu
    return cpu_emu.transfer_tables(_ifb())[2]


def _mixed(ifb):
    """profiles of several kinds, for mixed calls"""
    p = _profiles()
    return [p["display_p3_v4"], p["adobe_rgb_v2"], p["gray22_v2"], ifb.SourceProfile.cicp(9, 1), ifb.SourceProfile.cicp(12, 13),
            ifb.SourceProfile.gamma_primaries(0.45455, *pf.P3_XY), p["prophoto_v2"], ifb.SourceProfile.srgb()]


def _expect(ifb, profile, bgra, lut):
    return pf.apply_plan(ifb.source_profile_plan(profile), lut, bgra)


@pytest.mark.parametrize("alpha", ["noise", "cutout"])
@pytest.mark.parametrize("name", PROFILE_NAMES)
def test_every_triple_in_place(name, alpha, lut16k):
    """a 4096 x 4096 frame holding every RGB triple, transformed in place: equal to the oracle, alpha untouched"""
    import torch
    from imageflow_b200 import synth
    ifb = _ifb()
    frame = np.empty((4096, 4096, 4), np.uint8)
    frame[..., :3] = pf.all_triples()
    frame[..., 3] = (np.random.default_rng(5).integers(0, 256, (4096, 4096), dtype=np.uint8) if alpha == "noise"
                     else synth.cutout_np(4096, 4096, seed=3)[..., 3])
    want = _expect(ifb, _profiles()[name], frame, lut16k)
    t = torch.from_numpy(frame).cuda()
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    b.transform_to_srgb([(ifb.BitmapWindow.from_torch(t), None, _profiles()[name])], stream="own")
    b.sync()
    assert b.kernel_launches == n0 + 1
    got = t.cpu().numpy()
    assert np.array_equal(got[..., 3], frame[..., 3])
    bad = np.argwhere(np.any(got != want, axis=2))
    assert bad.size == 0, (len(bad), [(tuple(frame[y, x]), tuple(got[y, x]), tuple(want[y, x])) for y, x in bad[:4]])


def test_4k_frames_with_padded_strides_and_sub_windows(lut16k):
    """3840 x 2160 and odd sub-windows at odd origins of padded bitmaps, sentinel bytes around, mixed profiles in one call"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(9)
    sizes = [(3840, 2160), (3839, 2159), (1001, 777), (5, 3), (1, 1)]
    jobs, checks = [], []
    for i, (w, h) in enumerate(sizes):
        prof = _mixed(ifb)[i % 7]
        x, y = 1 + i % 3, 2 + i % 2
        full = rng.integers(0, 256, (h + 5, w + 9, 4), dtype=np.uint8)
        t = torch.from_numpy(full).cuda()
        want = full.copy()
        want[y:y + h, x:x + w] = _expect(ifb, prof, full[y:y + h, x:x + w], lut16k)
        win = ifb.BitmapWindow.from_torch(t[y:y + h, x:x + w])
        if i % 2:                                                # half the jobs out of place, into another padded bitmap
            dfull = rng.integers(0, 256, (h + 3, w + 6, 4), dtype=np.uint8)
            td = torch.from_numpy(dfull).cuda()
            dwant = dfull.copy()
            dwant[1:1 + h, 2:2 + w] = want[y:y + h, x:x + w]
            jobs.append((win, ifb.BitmapWindow.from_torch(td[1:1 + h, 2:2 + w]), prof))
            checks += [(t, full), (td, dwant)]
        else:
            jobs.append((win, None, prof))
            checks.append((t, want))
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    b.transform_to_srgb(jobs, stream="own")
    b.sync()
    assert b.kernel_launches == n0 + 1
    for t, want in checks:
        got = t.cpu().numpy()
        assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()


@pytest.mark.parametrize("channels", [3, 4, 1, 2], ids=["rgb24", "rgba32", "gray8", "grayalpha8"])
def test_rows_equal_pixel_convert_then_in_place(channels, lut16k):
    """decoder rows into BGRA (RGB24 at an odd pitch and byte offset) equal pixel_convert followed by the in-place transform on the
    device, and the oracle"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(40 + channels)
    w, h = 3840, 2160
    for prof in (_profiles()["display_p3_v4"], _profiles()["gray22_v2"], ifb.SourceProfile.srgb()):
        pitch = w * channels + (7 if channels == 3 else 4 * channels)
        raw = torch.from_numpy(rng.integers(0, 256, h * pitch + 16, dtype=np.uint8)).cuda()
        off = 5 if channels in (1, 3) else 8
        rows = raw[off:off + (h - 1) * pitch + w * channels].as_strided((h, w, channels), (pitch, channels, 1))
        src = rows.cpu().numpy()
        a = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        c = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        b = ifb.Batch(0)
        b.transform_to_srgb([(ifb.PixelRows.from_torch(rows), ifb.BitmapWindow.from_torch(a), prof)], stream="own")
        cw = ifb.BitmapWindow.from_torch(c)
        b.pixel_convert([ifb.pixel_op_for(channels)(ifb.PixelRows.from_torch(rows), cw)], stream="own")
        b.transform_to_srgb([(cw, None, prof)], stream="own")
        b.sync()
        got, two = a.cpu().numpy(), c.cpu().numpy()
        assert np.array_equal(got, two)
        assert np.array_equal(got, _expect(ifb, prof, po.convert(ifb.pixel_op_for(channels).OP, src), lut16k))
        assert np.array_equal(rows.cpu().numpy(), src)


@pytest.mark.parametrize("n", [1, 7, 64, 1024])
def test_a_call_of_n_jobs_with_mixed_profiles_is_one_launch(n, lut16k):
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(n)
    mixed = _mixed(ifb)[:7] if n < 1024 else [_profiles()["display_p3_v4"]]
    jobs, checks = [], []
    for i in range(n):
        w, h = (512, 384) if n == 1024 else (int(rng.integers(1, 300)), int(rng.integers(1, 200)))
        prof = mixed[i % len(mixed)]
        frame = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        t = torch.from_numpy(frame).cuda()
        jobs.append((ifb.BitmapWindow.from_torch(t), None, prof))
        if i < 64:
            checks.append((t, _expect(ifb, prof, frame, lut16k)))
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    b.transform_to_srgb(jobs, stream="own")
    b.sync()
    assert b.kernel_launches == n0 + 1
    for t, want in checks:
        assert np.array_equal(t.cpu().numpy(), want)


def test_srgb_and_zero_area_jobs_write_nothing():
    import torch
    ifb = _ifb()
    frame = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (64, 64, 4), dtype=np.uint8)).cuda()
    before = frame.cpu().numpy()
    p3 = _profiles()["display_p3_v4"]
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    b.transform_to_srgb([(ifb.BitmapWindow.from_torch(frame), None, ifb.SourceProfile.srgb()),
                         (ifb.BitmapWindow.from_torch(frame), None, ifb.SourceProfile.cicp(1, 13)),
                         (ifb.BitmapWindow.from_torch(frame[:0]), None, p3),
                         (ifb.BitmapWindow.from_torch(frame[:, :0]), None, ifb.SourceProfile.icc(b"broken"))], stream="own")
    b.sync()
    assert b.kernel_launches == n0 and np.array_equal(frame.cpu().numpy(), before)


@pytest.mark.parametrize("bad", ["unsupported", "malformed", "mismatch"])
def test_one_refused_profile_fails_the_call_and_writes_nothing(bad):
    import torch
    ifb = _ifb()
    refused = {"unsupported": (ifb.SourceProfile.cicp(9, 16), ifb.ErrorKind.MethodNotImplemented),
               "malformed": (ifb.SourceProfile.icc(pf.fixtures()["display_p3_v4"][1][:300]), ifb.ErrorKind.InvalidArgument),
               "mismatch": (ifb.SourceProfile.icc_gray(pf.fixtures()["adobe_rgb_v2"][1]), ifb.ErrorKind.InvalidArgument)}[bad]
    bufs = [torch.full((40, 70, 4), 7, dtype=torch.uint8, device="cuda") for _ in range(5)]
    jobs = [(ifb.BitmapWindow.from_torch(t[2:38, 3:67]), None, _mixed(ifb)[i]) for i, t in enumerate(bufs)]
    jobs[3] = (jobs[3][0], None, refused[0])
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    with pytest.raises(ifb.FlowError) as e:
        b.transform_to_srgb(jobs, stream="own")
    b.sync()
    assert e.value.kind == refused[1] and "transform to srgb job 3" in str(e.value)
    assert b.kernel_launches == n0 and all(bool((t == 7).all()) for t in bufs)


def test_config_2_resample_of_a_transformed_p3_frame_equals_the_oracle(lut16k):
    """3840x2160 Display P3 -> sRGB in place, then 3840x2160 -> 512x288 Robidoux in linear light: against the oracle's resample of the
    oracle's transformed frame"""
    import torch
    ifb = _ifb()
    p3 = _profiles()["display_p3_v4"]
    frame = np.random.default_rng(21).integers(0, 256, (2160, 3840, 4), dtype=np.uint8)
    frame[..., 3] = 255
    mid = _expect(ifb, p3, frame, lut16k)
    want = np.zeros((288, 512, 4), np.uint8)
    oracle.scale_and_render(mid, want, filter=2, linear=True, alpha_meaningful=False)
    t = torch.from_numpy(frame).cuda()
    out = torch.zeros((288, 512, 4), dtype=torch.uint8, device="cuda")
    b = ifb.Batch(0)
    win = ifb.BitmapWindow.from_torch(t)
    b.transform_to_srgb([(win, None, p3)], stream="own")
    b.scale_and_render_many([(win, ifb.BitmapWindow.from_torch(out), ifb.ScaleAndRenderParams(w=512, h=288))], stream="own")
    b.sync()
    assert np.array_equal(t.cpu().numpy(), mid)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()

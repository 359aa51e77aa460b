"""JPEG encoder colour stages on the GPU (bgra_to_ycbcr_kernel through Batch.bgra_to_ycbcr), byte for byte: every case of
tests/golden/ycbcr_enc_golden.npz (pinned against libjpeg-turbo) in one launch; tests/ycbcr_enc_oracle.py on seeded frames up to
4032 x 3024 at every sampling; cut-out alpha, where the planes equal ifb200_batch_apply_matte on a copy followed by an opaque conversion
and the source is untouched; a 1024-job call of mixed samplings, sizes and mattes as one launch; back-to-back calls on two streams; the
emulation's multi-job launches at every phase; and one frame whose source passes 2^32 bytes.  Every source and plane is a sub-window of
a padded tensor, with sentinel bytes around it that must come back unchanged."""
import ctypes as C

import numpy as np
import pytest

from tests import ycbcr_enc_oracle as eo
from tests.cpu_emu import run_ycbcr_enc_cases as rye
from tests.test_ycbcr_enc_oracle import CASES, MATTE, golden_case

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _padded(rng, a, x, y, extra_w, extra_h):
    """a (2-D plane or (H, W, 4) frame) as the window at (x, y) of a CUDA tensor of random sentinel bytes; -> (tensor, window, host copy)"""
    import torch
    shape = (a.shape[0] + y + extra_h, a.shape[1] + x + extra_w) + a.shape[2:]
    full = rng.integers(0, 256, shape, dtype=np.uint8)
    full[y:y + a.shape[0], x:x + a.shape[1]] = a
    t = torch.from_numpy(full).cuda()
    return t, t[y:y + a.shape[0], x:x + a.shape[1]], full


def _run(jobs_np, rng, stream="own", b=None):
    """one call of bgra_to_ycbcr over [(sampling, bgra, matte or None, expected (y, cb, cr))] with the source and every plane a padded
    sub-window; -> (batch, [(tensor, expected full tensor)])"""
    ifb = _ifb()
    b = b or ifb.Batch(0)
    recs, checks = [], []
    for i, (s, bgra, matte, want) in enumerate(jobs_np):
        h, w = bgra.shape[:2]
        ts, win, fs = _padded(rng, bgra, i % 3, 1, 2 + i % 5, 1)
        checks.append((ts, fs))
        planes = []
        for k, p in enumerate(want):
            tp, pw, fp = _padded(rng, np.zeros_like(p), (i + 3 * k) % 7, 1 + k, 1 + (i + k) % 9, 2)
            exp = fp.copy()
            exp[1 + k:1 + k + p.shape[0], (i + 3 * k) % 7:(i + 3 * k) % 7 + p.shape[1]] = p
            planes.append(pw)
            checks.append((tp, exp))
        recs.append(ifb.BgraToYcbcr(ifb.BitmapWindow.from_torch(win, alpha_meaningful=matte is not None), s, *planes,
                                    matte_bgra=matte or (255, 255, 255, 255)))
    b.bgra_to_ycbcr(recs, stream=stream)
    return b, checks


def _verify(checks, what=""):
    for k, (t, want) in enumerate(checks):
        got = t.cpu().numpy()
        assert np.array_equal(got, want), (what, k, np.argwhere(got != want)[:4].tolist())


def test_the_libjpeg_turbo_fixture_in_one_launch():
    rng = np.random.default_rng(1)
    b0 = _ifb().Batch(0)
    n0 = b0.kernel_launches
    jobs = []
    for name in CASES:
        s, src, y, cb, cr, matte = golden_case(name)
        jobs.append((s, src, MATTE if matte else None, (y, cb, cr)))
    b, checks = _run(jobs, rng, b=b0)
    b.sync()
    assert b.kernel_launches == n0 + 1
    _verify(checks, "golden")


@pytest.mark.parametrize("s", eo.SAMPLINGS)
@pytest.mark.parametrize("size", [(4032, 3024), (3840, 2160), (4031, 3023), (1, 3001), (3001, 1), (517, 389)])
def test_seeded_frames_against_the_oracle(s, size):
    w, h = size
    rng = np.random.default_rng(w * 7 + h + s)
    bgra = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    b, checks = _run([(s, bgra, None, eo.convert(s, bgra))], rng)
    b.sync()
    _verify(checks, (s, size))


@pytest.mark.parametrize("s", eo.SAMPLINGS)
@pytest.mark.parametrize("matte", [(255, 255, 255, 255), (40, 200, 90, 255), (10, 120, 250, 128)])
def test_cut_out_alpha_equals_apply_matte_then_an_opaque_conversion(s, matte):
    """a cut-out (alpha 0, 255 and values between): the fused planes equal ifb200_batch_apply_matte on a copy followed by the opaque
    conversion, and the oracle's; the source is only read"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(sum(matte) + s)
    w, h = 1031, 517
    bgra = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    a = bgra[..., 3]
    a[rng.random(a.shape) < 0.3] = 0
    a[rng.random(a.shape) < 0.3] = 255
    src = torch.from_numpy(bgra).cuda()
    b = ifb.Batch(0)
    fused = b.to_ycbcr(ifb.BitmapWindow.from_torch(src, alpha_meaningful=True), s, matte_bgra=matte, stream="own")
    flat = src.clone()
    err = C.create_string_buffer(512)
    st = b._stream("own")
    assert ifb.lib().ifb200_batch_apply_matte(b._h, flat.data_ptr(), w, h, w * 4, (C.c_uint8 * 4)(*matte), 1, st, err, 512) == 0, err.value
    two_step = b.to_ycbcr(flat, s, stream="own")
    b.sync()
    assert torch.equal(src.cpu(), torch.from_numpy(bgra))
    want = eo.convert_matte(s, bgra, matte, True)
    for f, t, o in zip(fused, two_step, want):
        assert np.array_equal(f.cpu().numpy(), t.cpu().numpy()) and np.array_equal(f.cpu().numpy(), o)


def test_a_1024_job_mixed_call_is_one_launch():
    rng = np.random.default_rng(1024)
    jobs = []
    for i in range(1024):
        s = int(rng.choice(eo.SAMPLINGS))
        w, h = int(rng.integers(1, 70)), int(rng.integers(1, 50))
        bgra = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        matte = rye.MATTES[i % 4] if i % 3 == 0 else None
        jobs.append((s, bgra, matte, eo.convert_matte(s, bgra, matte, True) if matte else eo.convert(s, bgra)))
    b0 = _ifb().Batch(0)
    n0 = b0.kernel_launches
    b, checks = _run(jobs, rng, b=b0)
    b.sync()
    assert b.kernel_launches == n0 + 1
    _verify(checks, "1024 jobs")


def test_back_to_back_calls_on_two_streams():
    import torch
    rng = np.random.default_rng(2)
    b = _ifb().Batch(0)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    all_checks = []
    for k in range(8):
        st = streams[k % 2]
        jobs = []
        for s in eo.SAMPLINGS:
            bgra = rng.integers(0, 256, (int(rng.integers(100, 600)), int(rng.integers(200, 900)), 4), dtype=np.uint8)
            jobs.append((s, bgra, None, eo.convert(s, bgra)))
        with torch.cuda.stream(st):
            _, checks = _run(jobs, rng, stream=st.cuda_stream, b=b)
        all_checks.append(checks)
    torch.cuda.synchronize()
    for k, checks in enumerate(all_checks):
        _verify(checks, ("call", k))


def test_the_emulation_launches_on_the_device():
    """the multi-job launches of the CPU emulation (every source and plane phase, widths 1..40, mattes, items whose CTA boundaries
    fall inside a band)"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(11)
    b = ifb.Batch(0)
    for jobs in rye.fixed_launches(rng) + [[rye.make_job(rng, matte=rye.MATTES[k % 4] if k % 2 else None) for k in range(8)]
                                           for _ in range(20)]:
        dev = {id(r): torch.from_numpy(r.buf.copy()).cuda() for _, rs, _, _ in jobs for r in rs}
        recs = []
        for d, rs, _, _ in jobs:
            ptr = lambda r, p: dev[id(r)].data_ptr() + (p - r.buf.ctypes.data)
            s, py, pb, pr = rs
            ch, cw = eo.chroma_shape(d["sampling"], d["w"], d["h"])
            recs.append(ifb.BgraToYcbcr(ifb.PixelRows(ptr(s, d["src"]), d["w"], d["h"], d["src_stride"], 4, dev[id(s)]), d["sampling"],
                                        ifb.PixelRows(ptr(py, d["y"]), d["w"], d["h"], d["y_stride"], 1, dev[id(py)]),
                                        ifb.PixelRows(ptr(pb, d["cb"]), cw, ch, d["cb_stride"], 1, dev[id(pb)]),
                                        ifb.PixelRows(ptr(pr, d["cr"]), cw, ch, d["cr_stride"], 1, dev[id(pr)]),
                                        bool(d["alpha_meaningful"]), d["matte_bgra"]))
        b.bgra_to_ycbcr(recs, stream="own")
        b.sync()
        for _, rs, _, _ in jobs:
            for r in rs:
                got = dev[id(r)].cpu().numpy()
                assert np.array_equal(got, r.exp), ([j[0] for j in jobs], np.nonzero(got != r.exp)[0][:4].tolist())


def test_nothing_to_write_launches_nothing_and_a_bad_descriptor_changes_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    z = torch.zeros((0, 4), dtype=torch.uint8, device="cuda")
    b.bgra_to_ycbcr([], stream="own")
    b.bgra_to_ycbcr([ifb.BgraToYcbcr(torch.zeros((0, 4, 4), dtype=torch.uint8, device="cuda"), ifb.YCBCR_420, z, z[:, :2], z[:, :2])],
                    stream="own")
    src = torch.full((8, 8, 4), 5, dtype=torch.uint8, device="cuda")
    y = torch.full((8, 8), 7, dtype=torch.uint8, device="cuda")
    c = torch.full((8, 4), 9, dtype=torch.uint8, device="cuda")
    with pytest.raises(ifb.FlowError) as e:         # the second job's Cr plane is its Cb plane
        b.bgra_to_ycbcr([ifb.BgraToYcbcr(src, ifb.YCBCR_420, y, c[:4], c[4:]),
                         ifb.BgraToYcbcr(src, ifb.YCBCR_420, y, c[:4], c[:4])], stream="own")
    b.sync()
    assert e.value.kind == ifb.ErrorKind.InvalidArgument and "bgra_to_ycbcr job 1: the Cr plane overlaps the Cb plane" in str(e.value)
    assert b.kernel_launches == n0 and bool((y == 7).all()) and bool((c == 9).all()) and bool((src == 5).all())


@pytest.mark.parametrize("s", [eo.S420, eo.S444])
def test_a_frame_whose_source_passes_2_32_bytes(s):
    """32 768 x 33 000: the BGRA source is 4.33 GB, so rows past 32 768 lie beyond byte 2^32 of it.  The source is seeded on the
    device; rows around the seam, the first rows and the last rows of every plane are checked against the oracle."""
    import torch
    ifb = _ifb()
    W, H = 32768, 33000
    free, _ = torch.cuda.mem_get_info(0)
    if free < 8 << 30:
        pytest.skip(f"the {W} x {H} frame and its planes take 6.5 GB; {free / 2**30:.1f} GiB of device memory is free, 8 GiB wanted")
    g = torch.Generator(device="cuda").manual_seed(32 + s)
    src = torch.randint(0, 256, (H, W, 4), dtype=torch.uint8, device="cuda", generator=g)
    assert src.numel() > 1 << 32
    b = ifb.Batch(0)
    y, cb, cr = b.to_ycbcr(src, s, stream="own")
    b.sync()
    seam = (1 << 32) // (W * 4)                                 # the first source row at or past byte 2^32
    for y0, y1 in ((0, 4), (seam - 4, seam + 4), (H - 4, H)):   # even bounds: whole 4:2:0 row pairs
        want = eo.convert(s, src[y0:y1].cpu().numpy())
        c0, c1 = (y0 // 2, y1 // 2) if s == eo.S420 else (y0, y1)
        for got, w_ in zip((y[y0:y1], cb[c0:c1], cr[c0:c1]), want):
            assert np.array_equal(got.cpu().numpy(), w_), (s, y0, y1)
    del src, y, cb, cr
    torch.cuda.empty_cache()

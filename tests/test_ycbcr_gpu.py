"""JPEG colour stages on the GPU (ycbcr_to_bgra_kernel through Batch.ycbcr_to_bgra), byte for byte: libjpeg-turbo's own output on every
case of tests/golden/ycbcr_golden.npz; tests/ycbcr_oracle.py on seeded frames up to 4032 x 3024 at every sampling; a 1024-job call of
mixed samplings and sizes as one launch; back-to-back calls on two streams; the emulation's multi-job launches at every phase; and one
4:2:0 frame whose BGRA output passes 2^32 bytes, checked on rows around the 2^32 seam and at its edges.  Every plane and destination is
a sub-window of a padded tensor, with sentinel bytes around it that must come back unchanged."""
import numpy as np
import pytest

from tests import ycbcr_oracle as yo
from tests.cpu_emu import run_ycbcr_cases as ryc
from tests.test_ycbcr_oracle import CASES, golden_case

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


def _random_frame(rng, s, w, h):
    ch, cw = yo.chroma_shape(s, w, h)
    return (rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (ch, cw), dtype=np.uint8),
            rng.integers(0, 256, (ch, cw), dtype=np.uint8))


def _run(jobs_np, rng, stream="own", b=None):
    """one call of ycbcr_to_bgra over [(sampling, y, cb, cr)] with every plane and destination a padded sub-window; -> (batch,
    [(destination tensor, expected full destination, [(plane tensor, its host copy)])])"""
    ifb = _ifb()
    b = b or ifb.Batch(0)
    jobs, checks = [], []
    for i, (s, y, cb, cr) in enumerate(jobs_np):
        h, w = y.shape
        planes = [_padded(rng, p, 1 + (i + k) % 5, 1 + k, 3 + i % 7, 2) for k, p in enumerate((y, cb, cr))]
        dst0 = np.zeros((h, w, 4), np.uint8)
        td, win, full = _padded(rng, dst0, 1 + i % 3, 2, 5, 1)
        want = full.copy()
        want[2:2 + h, 1 + i % 3:1 + i % 3 + w] = yo.convert(s, y, cb, cr)
        jobs.append((planes[0][1], planes[1][1], planes[2][1], s, ifb.BitmapWindow.from_torch(win)))
        checks.append((td, want, [(t, f) for t, _, f in planes]))
    b.ycbcr_to_bgra(jobs, stream=stream)
    return b, checks


def _verify(checks, what=""):
    for k, (td, want, planes) in enumerate(checks):
        got = td.cpu().numpy()
        assert np.array_equal(got, want), (what, k, np.argwhere(np.any(got != want, axis=-1))[:4].tolist())
        for t, f in planes:
            assert np.array_equal(t.cpu().numpy(), f), (what, k, "a plane changed")


def test_the_libjpeg_turbo_fixture_in_one_launch():
    rng = np.random.default_rng(1)
    b0 = _ifb().Batch(0)
    n0 = b0.kernel_launches
    b, checks = _run([(s, y, cb, cr) for s, y, cb, cr, _ in map(golden_case, CASES)], rng, b=b0)
    b.sync()
    assert b.kernel_launches == n0 + 1
    for name, (td, want, _) in zip(CASES, checks):
        assert np.array_equal(yo.convert(*golden_case(name)[:4]), golden_case(name)[4])
    _verify(checks, "golden")


@pytest.mark.parametrize("s", yo.SAMPLINGS)
@pytest.mark.parametrize("size", [(4032, 3024), (3840, 2160), (4031, 3023), (1, 3001), (3001, 1), (517, 389)])
def test_seeded_frames_against_the_oracle(s, size):
    w, h = size
    rng = np.random.default_rng(w * 7 + h + s)
    b, checks = _run([(s,) + _random_frame(rng, s, w, h)], rng)
    b.sync()
    _verify(checks, (s, size))


def test_a_1024_job_mixed_call_is_one_launch():
    rng = np.random.default_rng(1024)
    jobs = []
    for i in range(1024):
        s = int(rng.choice(yo.SAMPLINGS))
        w, h = int(rng.integers(1, 70)), int(rng.integers(1, 50))
        jobs.append((s,) + _random_frame(rng, s, w, h))
    b0 = _ifb().Batch(0)
    n0 = b0.kernel_launches
    b, checks = _run(jobs, rng, b=b0)
    b.sync()
    assert b.kernel_launches == n0 + 1
    _verify(checks, "1024 jobs")


def test_back_to_back_calls_on_two_streams():
    import torch
    rng = np.random.default_rng(2)
    ifb = _ifb()
    b = ifb.Batch(0)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    all_checks = []
    for k in range(8):
        st = streams[k % 2]
        jobs = [(s,) + _random_frame(rng, s, int(rng.integers(200, 900)), int(rng.integers(100, 600))) for s in yo.SAMPLINGS]
        with torch.cuda.stream(st):
            _, checks = _run(jobs, rng, stream=st.cuda_stream, b=b)
        all_checks.append(checks)
    torch.cuda.synchronize()
    for k, checks in enumerate(all_checks):
        _verify(checks, ("call", k))


def test_the_emulation_launches_on_the_device():
    """the multi-job launches of the CPU emulation (every plane phase modulo 16, every destination phase, widths 1..40, items whose
    CTA boundaries fall inside a band)"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(11)
    b = ifb.Batch(0)
    for jobs in ryc.fixed_launches(rng) + [[ryc.make_job(rng) for _ in range(8)] for _ in range(20)]:
        dev = {id(r): torch.from_numpy(r.buf.copy()).cuda() for _, rs, _, _ in jobs for r in rs}
        recs = []
        for d, rs, _, _ in jobs:
            ptr = lambda r, p: dev[id(r)].data_ptr() + (p - r.buf.ctypes.data)
            py, pb, pr, t = rs
            ch, cw = yo.chroma_shape(d["sampling"], d["w"], d["h"])
            recs.append((ifb.PixelRows(ptr(py, d["y"]), d["w"], d["h"], d["y_stride"], 1, dev[id(py)]),
                         ifb.PixelRows(ptr(pb, d["cb"]), cw, ch, d["cb_stride"], 1, dev[id(pb)]),
                         ifb.PixelRows(ptr(pr, d["cr"]), cw, ch, d["cr_stride"], 1, dev[id(pr)]), d["sampling"],
                         ifb.PixelRows(ptr(t, d["dst"]), d["w"], d["h"], d["dst_stride"], 4, dev[id(t)])))
        b.ycbcr_to_bgra(recs, stream="own")
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
    b.ycbcr_to_bgra([], stream="own")
    b.ycbcr_to_bgra([(z, z[:, :2], z[:, :2], ifb.YCBCR_420, torch.zeros((0, 4, 4), dtype=torch.uint8, device="cuda"))], stream="own")
    y = torch.full((8, 8), 7, dtype=torch.uint8, device="cuda")
    c = torch.full((4, 4), 9, dtype=torch.uint8, device="cuda")
    dst = torch.full((8, 8, 4), 5, dtype=torch.uint8, device="cuda")
    big = torch.full((16, 64), 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ifb.FlowError) as e:         # the second job's destination overlaps its own Y plane
        b.ycbcr_to_bgra([(y, c, c, ifb.YCBCR_420, dst),
                         (big[8:16, :8], c, c, ifb.YCBCR_420, big.view(16, 16, 4)[8:16, 0:8])], stream="own")
    b.sync()
    assert e.value.kind == ifb.ErrorKind.InvalidArgument and "ycbcr job 1: destination overlaps the Y plane" in str(e.value)
    assert b.kernel_launches == n0 and bool((dst == 5).all()) and bool((big == 3).all())


def _oracle_rows(s, y, cb, cr, y0, y1, W, H):
    """the oracle's output rows [y0, y1) of a W x H frame from host copies of the rows it needs: y = luma rows [y0, y1), cb / cr =
    chroma rows [a, b) as returned by _chroma_band"""
    a, _ = _chroma_band(s, y0, y1, H)
    band_h = cb.shape[0] * (2 if s == yo.S420 else 1)
    off = (y0 - 2 * a) if s == yo.S420 else (y0 - a)
    up_b = yo.upsample(s, cb, W, band_h)[off:off + (y1 - y0)]
    up_r = yo.upsample(s, cr, W, band_h)[off:off + (y1 - y0)]
    return yo.ycc_to_bgra(y, up_b, up_r)


def _chroma_band(s, y0, y1, H):
    """chroma rows [a, b) that output rows [y0, y1) read, with the halo rows of 4:2:0"""
    if s != yo.S420:
        return y0, y1
    ch = (H + 1) // 2
    return max(y0 // 2 - 1, 0), min((y1 + 1) // 2 + 1, ch)


def test_a_420_frame_past_2_32_output_bytes():
    """32 768 x 33 000 at 4:2:0: the BGRA output is 4.33 GB, so rows past 32 768 lie beyond byte 2^32 of the destination.  Planes are
    seeded on the device; rows around the seam, the first rows and the last rows are checked against the oracle."""
    import torch
    ifb = _ifb()
    W, H = 32768, 33000
    ch, cw = yo.chroma_shape(yo.S420, W, H)
    g = torch.Generator(device="cuda").manual_seed(32)
    y = torch.randint(0, 256, (H, W), dtype=torch.uint8, device="cuda", generator=g)
    cb = torch.randint(0, 256, (ch, cw), dtype=torch.uint8, device="cuda", generator=g)
    cr = torch.randint(0, 256, (ch, cw), dtype=torch.uint8, device="cuda", generator=g)
    out = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    assert out.numel() > 1 << 32
    b = ifb.Batch(0)
    b.ycbcr_to_bgra([(y, cb, cr, ifb.YCBCR_420, ifb.BitmapWindow.from_torch(out))], stream="own")
    b.sync()
    seam = (1 << 32) // (W * 4)                                 # the first row at or past byte 2^32
    for y0, y1 in ((0, 5), (seam - 3, seam + 3), (seam + 1, seam + 6), (H - 5, H)):
        a, bnd = _chroma_band(yo.S420, y0, y1, H)
        want = _oracle_rows(yo.S420, y[y0:y1].cpu().numpy(), cb[a:bnd].cpu().numpy(), cr[a:bnd].cpu().numpy(), y0, y1, W, H)
        got = out[y0:y1].cpu().numpy()
        assert np.array_equal(got, want), (y0, y1, np.argwhere(np.any(got != want, axis=-1))[:4].tolist())
    del y, cb, cr, out
    torch.cuda.empty_cache()

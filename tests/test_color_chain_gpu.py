"""Colour chains on the GPU (the colour kernels through Batch.color_chain), bit for bit against the node-by-node oracle: every preset
alone on Bgra32 and Bgr32 windows; the full RIAPI chain on 4K and 8K frames, also against the expansion run on the device with the
existing single-window calls; padded strides and sub-windows with sentinel bytes around them; batches of 1, 7 and 64 jobs as one
launch (three with white balance); a call with nothing to write as none; a bad descriptor that changes nothing; and the config-2
resample followed by s.saturation=-0.5&s.contrast=0.2&a.balancewhite=true against the oracle; and the window metadata (format,
compositing) each chain leaves behind, as the nodes leave it."""
import numpy as np
import pytest

import oracle
from tests import color_oracle as co
from tests.cpu_emu import run_color_cases as rcc

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _product_steps(chain):
    """the product's step records of an oracle chain"""
    ifb = _ifb()
    out = []
    for s in chain:
        if s[0] == "matrix":
            out.append(ifb.ColorMatrixSrgb(s[1]))
        elif s[0] == "enable_transparency":
            out.append(ifb.EnableTransparency())
        else:
            out.append(ifb.WhiteBalanceHistogramAreaThresholdSrgb(s[1]))
    return out


def _upload(jobs):
    import torch
    return {id(bm): torch.from_numpy(bm.buf.copy()).cuda() for _, bm, _, _, _ in jobs}


def _jobs_of(jobs, dev):
    ifb = _ifb()
    return [(ifb.BitmapWindow(dev[id(bm)].data_ptr() + (d["ptr"] - bm.buf.ctypes.data), d["w"], d["h"], d["stride"], d["am"],
                              _keep=dev[id(bm)]), _product_steps(chain)) for d, bm, _, chain, _ in jobs]


def _check(jobs, dev, what):
    for _, bm, _, _, _ in jobs:
        got = dev[id(bm)].cpu().numpy()
        assert np.array_equal(got, bm.exp), (what, np.nonzero(got != bm.exp)[0][:4].tolist())


def test_every_preset_alone_on_bgra32_and_bgr32():
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(21)
    for p in (-0.7, 0.3):
        jobs = [rcc.make_job(rng, co.preset(k, p), (67, 13), am) for k in range(10) for am in (False, True)]
        dev = _upload(jobs)
        wins = b.color_chain(_jobs_of(jobs, dev), stream="own")
        b.sync()
        _check(jobs, dev, p)
        for (d, _, _, chain, _), w in zip(jobs, wins):
            assert w.alpha_meaningful == (d["am"] or chain[0][0] == "enable_transparency")


def test_padded_strides_and_sub_windows_with_random_chains():
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(22)
    for rep in range(6):
        jobs = [rcc.make_job(rng) for _ in range(9)]
        dev = _upload(jobs)
        b.color_chain(_jobs_of(jobs, dev), stream="own")
        b.sync()
        _check(jobs, dev, rep)


def test_batches_are_one_launch_or_three_with_white_balance():
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(23)
    for n in (1, 7, 64):
        for wb in (False, True):
            first = rcc.make_job(rng, co.preset(co.INVERT) + ([("white_balance", None)] if wb else []))
            jobs = [first] + [rcc.make_job(rng, wb=False) for _ in range(n - 1)]
            dev = _upload(jobs)
            before = b.kernel_launches
            b.color_chain(_jobs_of(jobs, dev), stream="own")
            b.sync()
            assert b.kernel_launches == before + (3 if wb else 1), (n, wb)
            _check(jobs, dev, (n, wb))


def test_call_with_nothing_to_write_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    t = torch.full((8, 8, 4), 7, dtype=torch.uint8, device="cuda")
    win = ifb.BitmapWindow.from_torch(t, alpha_meaningful=True)
    before = b.kernel_launches
    b.color_chain([(win, []), (win, [ifb.EnableTransparency()]), (ifb.BitmapWindow(0, 0, 5, 0), ifb.ColorFilterSrgb.sepia())], stream="own")
    b.color_chain([], stream="own")
    b.sync()
    assert b.kernel_launches == before and (t.cpu().numpy() == 7).all()


def test_a_bad_descriptor_changes_nothing_and_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(24)
    jobs = [rcc.make_job(rng) for _ in range(7)]
    dev = _upload(jobs)
    good = _jobs_of(jobs, dev)
    sq = ifb.BitmapWindow.from_torch(torch.zeros((6, 6, 4), dtype=torch.uint8, device="cuda"))
    wb = ifb.WhiteBalanceHistogramAreaThresholdSrgb()
    for bad, kind in (((ifb.BitmapWindow(sq.ptr + 2, 5, 6, 24, _keep=sq._keep), ifb.ColorFilterSrgb.invert()), ifb.ErrorKind.InvalidArgument),
                      ((sq, [ifb.WhiteBalanceHistogramAreaThresholdSrgb(float("nan"))]), ifb.ErrorKind.InvalidArgument),
                      ((sq, [wb, wb]), ifb.ErrorKind.MethodNotImplemented)):
        before = b.kernel_launches
        with pytest.raises(ifb.FlowError) as e:
            b.color_chain(good[:3] + [bad] + good[3:], stream="own")
        b.sync()
        assert e.value.kind == kind and "color job 3" in str(e.value)
        assert b.kernel_launches == before
        for _, bm, _, _, _ in jobs:
            assert np.array_equal(dev[id(bm)].cpu().numpy(), bm.buf)


ALL_KEYS = dict(alpha=0.6, brightness=0.1, contrast=0.2, saturation=-0.3, sepia=True, grayscale="flat", balance_white=True)


def _expansion_on_device(b, t, chain, am):
    """the chain node by node on the device with the existing single-window calls"""
    ifb = _ifb()
    win = ifb.BitmapWindow.from_torch(t, alpha_meaningful=am)
    for s in chain:
        if s[0] == "matrix":
            b.color_matrix(win.ptr, win.w, win.h, win.stride, s[1], stream="own")
        elif s[0] == "enable_transparency":
            if not win.alpha_meaningful:
                b.canvas([ifb.EnableTransparency(win)], stream="own")
        else:
            b.white_balance(win, s[1], stream="own")
    b.sync()


@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)])
@pytest.mark.parametrize("am", [False, True])
def test_the_full_riapi_chain_on_4k_and_8k_frames(w, h, am):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    host = oracle.synth_noise(w, h, seed=w + am, alpha_mode="mixed")
    chain = co.riapi_steps(**ALL_KEYS)
    want, want_am, _ = co.run_chain(host, chain, am)
    src = torch.from_numpy(host).cuda()
    exp_dev = src.clone()
    _expansion_on_device(b, exp_dev, chain, am)
    before = b.kernel_launches
    out = b.color_chain([(ifb.BitmapWindow.from_torch(src, alpha_meaningful=am), ifb.riapi_color_steps(**ALL_KEYS))], stream="own")[0]
    b.sync()
    assert b.kernel_launches == before + 3 and out.alpha_meaningful == want_am
    assert torch.equal(src, exp_dev)
    assert np.array_equal(src.cpu().numpy(), want)


def test_config2_resample_then_the_chain_equals_the_oracle():
    """3840x2160 -> 512x288 Robidoux in linear light (config 2), then s.saturation=-0.5&s.contrast=0.2&a.balancewhite=true as one
    chain call, against the oracle's scale_and_render followed by the node-by-node expansion"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    inp = oracle.synth_noise(3840, 2160, seed=12, alpha_mode="mixed")
    mid = np.zeros((288, 512, 4), np.uint8)
    oracle.scale_and_render(inp, mid, filter=2, linear=True, alpha_meaningful=True)
    kw = dict(saturation=-0.5, contrast=0.2, balance_white=True)
    want, _, _ = co.run_chain(mid, co.riapi_steps(**kw), True)
    src = torch.from_numpy(inp).cuda()
    out = torch.zeros((288, 512, 4), dtype=torch.uint8, device="cuda")
    win = ifb.BitmapWindow.from_torch(out, alpha_meaningful=True)
    b.scale_and_render_many([(ifb.BitmapWindow.from_torch(src, alpha_meaningful=True), win, ifb.ScaleAndRenderParams(w=512, h=288))], stream="own")
    before = b.kernel_launches
    b.color_chain([(win, ifb.riapi_color_steps(**kw))], stream="own")
    b.sync()
    assert b.kernel_launches == before + 3
    got = out.cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()


def test_window_metadata_after_the_chain_is_what_the_nodes_leave():
    """ColorMatrixSrgbMutDef sets BlendWithSelf after every matrix whatever the format (flow/nodes/color.rs:29); EnableTransparency on
    Bgr32 makes the window Bgra32 with BlendWithSelf, on Bgra32 it does nothing; the white balance leaves the metadata alone.  Zero-area
    windows get the same metadata: the nodes still run there."""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    BC = ifb.BitmapCompositing
    chains = {"none": [], "enable_transparency": [ifb.EnableTransparency()], "brightness": ifb.ColorFilterSrgb.brightness(0.1),
              "sepia": ifb.ColorFilterSrgb.sepia(), "white_balance": [ifb.WhiteBalanceHistogramAreaThresholdSrgb()],
              "alpha": ifb.ColorFilterSrgb.alpha(0.5), "white_balance_then_invert": [ifb.WhiteBalanceHistogramAreaThresholdSrgb()] + ifb.ColorFilterSrgb.invert()}
    t = torch.zeros((len(chains) * 8, 16, 16, 4), dtype=torch.uint8, device="cuda")
    jobs, want = [], []
    i = 0
    for name, steps in chains.items():
        matrix = any(isinstance(s, ifb.ColorMatrixSrgb) for s in steps)
        et = any(isinstance(s, ifb.EnableTransparency) for s in steps)
        for am in (False, True):
            for compose in (BC.ReplaceSelf, BC.BlendWithMatte):
                for empty in (False, True):
                    w = ifb.BitmapWindow.from_torch(t[i], alpha_meaningful=am, compose=compose)
                    if empty:
                        w = ifb.BitmapWindow(w.ptr, 0, 16, w.stride, am, compose, _keep=w._keep)
                    i += 1
                    jobs.append((w, steps))
                    want.append((name, am, compose, empty, am or et, BC.BlendWithSelf if matrix or (et and not am) else compose))
    out = b.color_chain(jobs, stream="own")
    b.sync()
    for w, (name, am, compose, empty, am_after, compose_after) in zip(out, want):
        assert (bool(w.alpha_meaningful), w.compose) == (am_after, compose_after), (name, am, compose, empty)

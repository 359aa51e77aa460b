"""python -m tests.cpu_emu.run_hv_cases <libhv_emu.so> [n_cases]: the emulated hv_ring_kernel against the oracle.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded)."""
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from imageflow_b200 import synth
from tests import cpu_emu, util

# (in_w, in_h, out_w, out_h, filter, kwargs of run_hv)
CASES = [
    (640, 480, 200, 150, 2, dict()),                                         # config-1 shape
    (960, 540, 128, 128, 2, dict(n_bands=3, jobs_repeat=2)),                 # config-2 ratios (7.5 x 4.2), bands
    (960, 540, 128, 128, 6, dict(alpha=True, n_bands=2)),                    # Lanczos3: ring depth 6
    (800, 600, 400, 300, 2, dict(alpha=True, compose=1, cm="sepia")),        # 2x, composite over the canvas, colour matrix
    (1280, 96, 320, 24, 2, dict(strip_cols=16, alpha=True, compose=2)),      # many strips, matte
    (260, 250, 61, 59, 2, dict(in_xoff=4, n_bands=4)),                       # ragged sizes, unaligned window origin, short bands
    (33, 17, 7, 5, 2, dict(alpha=True, in_xoff=8)),                          # smaller than one TMA box
    (8, 8, 1, 1, 2, dict(alpha=True)),
    (256, 256, 256, 256, 2, dict(strip_cols=32, sb_low16=0x1400)),           # 1:1, another shared-memory origin
    (512, 384, 128, 96, 14, dict(linear=False, n_bands=2)),                  # Mitchell in sRGB space
    (1024, 64, 96, 17, 13, dict(alpha=True, sharpen=50.0)),                  # CatmullRom, sharpen
    (128, 128, 37, 41, 24, dict()),                                          # Box
    (400, 300, 100, 75, 4, dict(alpha=True, linear=False, strip_cols=16)),   # Ginseng (ring depth 6), sRGB space
    # cut-out content (synth.cutout_np over synth.cutout_canvas_np): alpha exactly 0, negative, tiny, above 1 and next to 0.994
    # before the store, fa == 0 and fa < 0 in BlendWithSelf (tests/test_alpha_edges_oracle.py checks that these are reached)
    (640, 480, 200, 150, 2, dict(content="cutout", alpha=True)),
    (640, 480, 200, 150, 2, dict(content="cutout", alpha=True, compose=1)),
    (640, 480, 200, 150, 2, dict(content="cutout", alpha=True, compose=2, linear=False, cm="sepia")),
    (960, 540, 128, 128, 6, dict(content="cutout", alpha=True, compose=1, linear=False)),       # Lanczos3: ring depth 6
    (960, 540, 128, 128, 6, dict(content="cutout", alpha=True, compose=2)),
    (512, 384, 128, 96, 2, dict(content="cutout", alpha=True, compose=1, cm="sepia", n_bands=2)),
    (512, 384, 128, 96, 2, dict(content="cutout", alpha=False, compose=1, linear=False)),
]


def run(so, limit=None):
    L = cpu_emu.load_hv(so)
    n = 0
    for (iw, ih, ow, oh, flt, kw) in CASES:
        kw = dict(kw)
        alpha = kw.pop("alpha", False)
        cm = kw.pop("cm", None)
        cm = ifb.color_filter_matrix(0) if cm == "sepia" else None
        common = dict(filter=flt, alpha_meaningful=alpha, linear=kw.pop("linear", True), compose=kw.pop("compose", 0), matte=(40, 120, 250, 200),
                      color_matrix=cm, sharpen=kw.pop("sharpen", 0.0))
        if kw.pop("content", "noise") == "cutout":
            inp, canvas = synth.cutout_np(iw, ih, seed=iw + oh), synth.cutout_canvas_np(ow + 5, oh + 3, seed=3)
        else:
            inp = util.noise(iw, ih, seed=iw + oh, alpha_mode="mixed" if alpha else "opaque")
            canvas = util.noise(ow + 5, oh + 3, seed=3, alpha_mode="mixed")
        exp = canvas.copy()
        oracle.scale_and_render(inp, exp, x=2, y=1, w=ow, h=oh, **common)
        outs = cpu_emu.run_hv(L, ifb, inp, canvas, x=2, y=1, w=ow, h=oh, **common, **kw)
        assert outs is not None, ("not a ring geometry", iw, ih, ow, oh, flt)
        for o in outs:
            d = np.abs(o.astype(np.int16) - exp.astype(np.int16))
            assert d.max() == 0, (iw, ih, ow, oh, flt, kw, int(d.max()), int((d > 0).sum()))
        n += 1
        if limit and n >= limit:
            return n
    return n


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else None))

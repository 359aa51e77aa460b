"""python -m tests.cpu_emu.run_tile2_cases <libtile2_emu.so> [n_cases]: the emulated fused_tile2_kernel against the oracle.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded)."""
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from imageflow_b200 import synth
from tests import cpu_emu, util

GEOMETRIES = [(64, 64, 128, 128, 14), (33, 17, 70, 50, 2), (5, 3, 200, 100, 14), (100, 60, 333, 200, 4), (256, 256, 256, 256, 2), (300, 40, 310, 47, 13)]
# cut-out content (synth.cutout_np over synth.cutout_canvas_np), every variant: alpha exactly 0, negative, tiny, above 1 and next
# to 0.994 before the store, fa == 0 and fa < 0 in BlendWithSelf (tests/test_alpha_edges_oracle.py checks that these are reached)
CUTOUT_GEOMETRIES = [(100, 60, 333, 200, 14), (300, 200, 300, 200, 2)]


def variants():
    sepia, general = ifb.color_filter_matrix(0), ifb.color_filter_matrix(6, 0.5)
    general[4, 0] = 0.1
    return [(True, True, 1, sepia), (False, False, 0, None), (True, False, 2, None), (False, True, 1, general),
            (True, True, 0, general), (True, False, 1, None), (False, True, 2, sepia), (True, True, 2, sepia)]


def run(so, limit=None):
    L = cpu_emu.load_tile2(so)
    n = 0
    for gi, (iw, ih, ow, oh, flt) in enumerate(GEOMETRIES):
        for vi, (alpha, linear, compose, cm) in enumerate(variants()):
            if (gi + vi) % 2:                      # half of the grid: every geometry and every variant still occur
                continue
            inp = util.noise(iw, ih, seed=iw + oh + vi, alpha_mode="mixed" if alpha else "opaque")
            canvas = util.noise(ow + 5, oh + 3, seed=2 + vi, alpha_mode="mixed")
            kw = dict(x=2, y=1, w=ow, h=oh, filter=flt, alpha_meaningful=alpha, linear=linear, compose=compose, matte=(40, 120, 250, 200), color_matrix=cm)
            exp = canvas.copy()
            oracle.scale_and_render(inp, exp, **kw)
            for o in cpu_emu.run_tile2(L, ifb, inp, canvas, grid=2, jobs_repeat=2, **kw):   # 2 persistent CTAs walk the tiles of 2 jobs
                assert np.array_equal(o, exp), (iw, ih, ow, oh, flt, alpha, linear, compose, cm is not None)
            n += 1
            if limit and n >= limit:
                return n
    for (iw, ih, ow, oh, flt) in CUTOUT_GEOMETRIES:
        for vi, (alpha, linear, compose, cm) in enumerate(variants()):
            inp, canvas = synth.cutout_np(iw, ih, seed=iw + oh + vi), synth.cutout_canvas_np(ow + 5, oh + 3, seed=2 + vi)
            kw = dict(x=2, y=1, w=ow, h=oh, filter=flt, alpha_meaningful=alpha, linear=linear, compose=compose, matte=(40, 120, 250, 200), color_matrix=cm)
            exp = canvas.copy()
            oracle.scale_and_render(inp, exp, **kw)
            for o in cpu_emu.run_tile2(L, ifb, inp, canvas, grid=2, **kw):
                assert np.array_equal(o, exp), ("cutout", iw, ih, ow, oh, flt, alpha, linear, compose, cm is not None)
            n += 1
            if limit and n >= limit:
                return n
    return n


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else None))

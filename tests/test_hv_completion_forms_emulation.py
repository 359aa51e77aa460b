"""hv_ring_kernel's one-completion chunk forms, executed on the CPU (tests/cpu_emu/hv_kernel_emu.cc) against the oracle.  A chunk
of four source columns with exactly one completion runs the form compiled for the ring slot of the completing column, in either
chunk of a pair, with a predicated park behind each of its four columns.  Ratios near 7.5 : 1 and 4 : 1 that are not whole
numbers move the completing column through every slot and every column of the chunk; together these cases reach each (slot,
column) of both chunks at ring depths 4 and 6, with three and with four channels, for the stored-frame kernel (the case list of
tests/test_hv_emulation.py never reaches a one-completion chunk at ring depth 6 with three channels), bit-exact."""
import numpy as np
import pytest

import imageflow_b200 as ifb
import oracle
from tests import cpu_emu, util

# (in_w, in_h, out_w, out_h, filter, alpha_meaningful)
CASES = [
    (960, 540, 128, 72, 2, False),      # 7.5 : 1, ring depth 4, three channels
    (960, 540, 128, 72, 6, False),      # Lanczos3: ring depth 6
    (960, 540, 131, 75, 2, True),       # 7.3 : 1, four channels
    (960, 540, 233, 131, 2, True),      # 4.1 : 1
    (960, 540, 131, 75, 6, True),
    (960, 540, 233, 131, 6, True),
]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return cpu_emu.load_hv(cpu_emu.build(str(tmp_path_factory.mktemp("hv_forms")), "hv_kernel_emu.cc"))


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%dx%d-%dx%d-f%d-a%d" % c)
def test_one_completion_forms_are_bit_exact(emu, case):
    iw, ih, ow, oh, flt, alpha = case
    inp = util.noise(iw, ih, seed=iw + ow, alpha_mode="mixed" if alpha else "opaque")
    canvas = util.noise(ow + 5, oh + 3, seed=3, alpha_mode="mixed")
    common = dict(filter=flt, alpha_meaningful=alpha, linear=True, compose=0, matte=(40, 120, 250, 200), color_matrix=None, sharpen=0.0)
    exp = canvas.copy()
    oracle.scale_and_render(inp, exp, x=2, y=1, w=ow, h=oh, **common)
    outs = cpu_emu.run_hv(emu, ifb, inp, canvas, x=2, y=1, w=ow, h=oh, **common)
    assert outs is not None, "not a ring geometry"
    for o in outs:
        d = np.abs(o.astype(np.int16) - exp.astype(np.int16))
        assert d.max() == 0, (case, int(d.max()), int((d > 0).sum()))

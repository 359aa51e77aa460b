"""hv_ring_kernel's H accumulators in register order, executed on the CPU (tests/cpu_emu/hv_kernel_emu.cc) against the oracle.

At the start of every chunk (four source columns) register 0 holds the oldest open output column.  A chunk with exactly one
completion parks register 0 (register AV - 1 when the completion is on the chunk's last column) and rotates the registers by one;
a general chunk rotates behind each of its completions; the CTA stages each weight record in the register order that walk gives.
The cases below are checked, from the planner's own completion table, to reach a one-completion chunk with its completion on every
column of both chunks of a pair under every rotation phase (the rotations so far, mod AV), at ring depths 4 and 6 with three and with
four channels, and a general chunk with two or more completions right behind a one-completion chunk; then each case runs bit-exact."""
import numpy as np
import pytest

import imageflow_b200 as ifb
import oracle
from tests import cpu_emu, util

# (in_w, in_h, out_w, out_h, filter, alpha_meaningful): ratios that are not whole numbers move the completing column through every
# column of a chunk; one strip's rotations then move it through every phase
CASES = [
    (960, 540, 131, 75, 2, False),      # 7.3 : 1, ring depth 4, three channels
    (960, 540, 233, 131, 2, False),     # 4.1 : 1
    (960, 540, 131, 75, 2, True),       # four channels
    (960, 540, 233, 131, 2, True),
    (960, 540, 131, 75, 6, False),      # Lanczos3: ring depth 6
    (960, 540, 233, 131, 6, False),
    (960, 540, 131, 75, 6, True),
    (960, 540, 233, 131, 6, True),
    (960, 540, 347, 195, 2, False),     # 2.8 : 1: general chunks, some right behind a one-completion chunk
    (960, 540, 347, 195, 6, True),
]


def chunk_walk(iw, ih, ow, oh, flt, alpha):
    """(av, {(chunk of the pair, completing column, rotation phase)} of the one-completion chunks, number of general chunks with two
    or more completions right behind a one-completion chunk), from the strips' completion tables"""
    info, blob = cpu_emu.hv_plan(ifb, iw, ih, ow, oh, flt, alpha=alpha)
    assert info.ok and blob is not None, "not a ring geometry"
    av = info.av
    hw_stride = (info.o_hdone - info.o_hw) // (info.n_strips * info.avp * 4)
    hd_stride = hw_stride + 64
    one, gen_after_one = set(), 0
    for s in range(info.n_strips):
        hd = blob[info.o_hdone + s * hd_stride:info.o_hdone + s * hd_stride + hw_stride].astype(np.int64) & 0x7f
        rot, prev_one = 0, False
        for c4 in range(0, hw_stride, 4):
            d = hd[c4:c4 + 4]
            n1, n2 = int((d >= 1).sum()), int((d >= 2).sum())
            is_one = n1 == 1 and n2 == 0
            if is_one:
                one.add(((c4 // 4) & 1, int(np.flatnonzero(d)[0]), rot % av))
                rot += 1
            else:
                if prev_one and int(d.sum()) >= 2:
                    gen_after_one += 1
                rot += int(d.sum())
            prev_one = is_one
    return av, one, gen_after_one


def test_cases_reach_every_column_and_phase():
    reach = {}
    gen = {}
    for iw, ih, ow, oh, flt, alpha in CASES:
        av, one, g = chunk_walk(iw, ih, ow, oh, flt, alpha)
        key = (av, 4 if alpha else 3)
        reach.setdefault(key, set()).update(one)
        gen[key] = gen.get(key, 0) + g
    for av in (4, 6):
        for ch in (3, 4):
            want = {(h, col, ph) for h in (0, 1) for col in range(4) for ph in range(av)}
            missing = sorted(want - reach.get((av, ch), set()))
            assert not missing, ((av, ch), missing)
    assert gen[(4, 3)] > 0 and gen[(6, 4)] > 0, gen


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return cpu_emu.load_hv(cpu_emu.build(str(tmp_path_factory.mktemp("hv_regs")), "hv_kernel_emu.cc"))


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%dx%d-%dx%d-f%d-a%d" % c)
def test_register_order_is_bit_exact(emu, case):
    iw, ih, ow, oh, flt, alpha = case
    inp = util.noise(iw, ih, seed=iw + ow + flt, alpha_mode="mixed" if alpha else "opaque")
    canvas = util.noise(ow + 5, oh + 3, seed=4, alpha_mode="mixed")
    common = dict(filter=flt, alpha_meaningful=alpha, linear=True, compose=0, matte=(40, 120, 250, 200), color_matrix=None, sharpen=0.0)
    exp = canvas.copy()
    oracle.scale_and_render(inp, exp, x=2, y=1, w=ow, h=oh, **common)
    outs = cpu_emu.run_hv(emu, ifb, inp, canvas, x=2, y=1, w=ow, h=oh, **common)
    assert outs is not None, "not a ring geometry"
    for o in outs:
        d = np.abs(o.astype(np.int16) - exp.astype(np.int16))
        assert d.max() == 0, (case, int(d.max()), int((d > 0).sum()))

"""python -m tests.cpu_emu.run_color_cases <libcolor_emu.so> [n_launches]: the emulated colour-chain kernels
(tests/cpu_emu/color_kernel_emu.cc, with the product's planner) against the node-by-node chain of tests/color_oracle.py.  Also the body
of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every launch holds several jobs, each a sub-window of an exactly sized bitmap of random sentinel bytes (no byte after the last pixel of
the last row) at a random origin, with a row pitch that is often not a multiple of 16, so that rows start at every 4-byte phase modulo
16.  Chains mix the presets with random parameters, random sparse matrices with signed zeros, NaN and infinite coefficients,
EnableTransparency on Bgr32 and Bgra32 windows, and white balance.  Per launch:
  - jobs that share one step array (and so their planned tables) are as right as the others;
  - every bitmap equals the expected one (the chain's result in the window; every other byte, stride padding included, unchanged);
  - no pixel is stored twice, and the pixels stored are exactly the windows';
  - every load is in a window, each pixel loaded once per pass (twice for a job that white-balances);
  - the counters of each white balance equal the oracle's histograms of the frame as the chain leaves it before the white balance."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import ColorDesc, ColorStep
from tests import color_oracle as co
from tests.cpu_emu.run_orient_cases import window_in

SOURCES = ("color_kernel_emu.cc", "ifb_color.cc", "ifb_orient.cc")          # of tests.cpu_emu.build
SIZES = [(1, 1), (1, 7), (7, 1), (5, 3), (31, 5), (33, 9), (64, 3), (65, 2), (2, 65), (129, 17)]
MATRIX, ENABLE_TRANSPARENCY, WHITE_BALANCE = 0, 1, 2


def load(so):
    L = C.CDLL(so)
    L.emu_color.restype = C.c_long
    L.emu_color.argtypes = [C.POINTER(ColorDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                            C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int), C.c_char_p,
                            C.c_size_t, C.c_int]
    L.emu_color_plan.restype = C.c_long
    L.emu_color_plan.argtypes = [C.POINTER(ColorDesc), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t,
                                 C.POINTER(C.c_size_t)]
    L.emu_color_tables.restype = C.c_long
    L.emu_color_tables.argtypes = [C.POINTER(ColorDesc), C.c_size_t, C.c_void_p, C.c_size_t]
    return L


def steps_array(chain):
    """the ifb200_color_step array of an oracle chain"""
    arr = (ColorStep * max(len(chain), 1))()
    for s, c in zip(arr, chain):
        if c[0] == "matrix":
            s.kind = MATRIX
            s.matrix = (C.c_float * 25)(*np.asarray(c[1], np.float32).reshape(25).tolist())
        elif c[0] == "enable_transparency":
            s.kind = ENABLE_TRANSPARENCY
        else:
            s.kind = WHITE_BALANCE
            s.threshold = -1.0 if c[1] is None else float(c[1])
    return arr


def desc(ptr, w, h, stride, am, chain, keep, shared=None):
    """the descriptor of one job; jobs with the same chain object share one step array when `shared` (a dict) is given, as the
    Python mirror passes them (the planner then shares their tables)"""
    d = ColorDesc()
    if shared is not None and id(chain) in shared:
        arr = shared[id(chain)]
    else:
        arr = steps_array(chain)
        if shared is not None:
            shared[id(chain)] = arr
    keep.append(arr)
    d.px = ptr; d.w = w; d.h = h; d.stride = stride; d.alpha_meaningful = int(am)
    d.steps = C.cast(arr, C.c_void_p).value; d.n_steps = len(chain)
    return d


def sparse_matrix(rng):
    """a random 5x5 with many zeros of either sign, sometimes separable, sometimes NaN / infinite / out-of-range coefficients"""
    m = rng.normal(0, 0.8, (5, 5)).astype(np.float32)
    m[rng.random((5, 5)) < 0.6] = 0.0
    m[rng.random((5, 5)) < 0.15] = np.float32(-0.0)
    if rng.random() < 0.5:                                     # separable: off-diagonal zeros of the 4x4 part
        for k in range(4):
            for c in range(4):
                if k != c:
                    m[k, c] = np.float32(-0.0) if rng.random() < 0.3 else np.float32(0.0)
    if rng.random() < 0.2:
        m[rng.integers(0, 5), rng.integers(0, 4)] = rng.choice([np.nan, np.inf, -np.inf, 300.0, -7.5])
    return m


def random_step(rng):
    r = rng.random()
    if r < 0.45:
        which = int(rng.integers(0, 10))
        return co.preset(which, float(rng.choice([-1.5, -1.0, -0.5, -0.2, 0.0, 0.1, 0.3, 0.5, 1.0, 2.0]) + rng.normal(0, 0.05)))
    if r < 0.75:
        return [("matrix", sparse_matrix(rng))]
    if r < 0.9:
        return [("enable_transparency",)]
    return [("white_balance", float(rng.choice([-1.0, 0.0, 0.006, 0.05, 0.3, 0.6])))]


def random_chain(rng, wb=None):
    chain = []
    for _ in range(int(rng.integers(1, 7))):
        chain += [s for s in random_step(rng) if s[0] != "white_balance"]
    chain = chain[:15]
    if wb if wb is not None else rng.random() < 0.35:
        chain.insert(int(rng.integers(0, len(chain) + 1)), ("white_balance", float(rng.choice([-1.0, 0.0, 0.01, 0.2]))))
    return chain


def make_job(rng, chain=None, size=None, am=None, wb=None):
    """-> (desc, bitmap, window pixel addresses, chain, expected pre-WB histogram or None); the bitmap's `exp` holds the result"""
    w, h = size or (SIZES[int(rng.integers(0, len(SIZES)))] if rng.random() < 0.6 else (int(rng.integers(1, 90)), int(rng.integers(1, 30))))
    chain = random_chain(rng, wb) if chain is None else chain
    am = bool(rng.random() < 0.5) if am is None else am
    bm, x, y = window_in(rng, w, h)
    want, _, hist = co.run_chain(bm.view(bm.buf, x, y, w, h).copy(), chain, am)
    bm.view(bm.exp, x, y, w, h)[...] = want
    return {"ptr": bm.buf.ctypes.data + y * bm.pitch + x * 4, "w": w, "h": h, "stride": bm.pitch, "am": am}, bm, bm.addrs(x, y, w, h), chain, hist


def launch(L, jobs, sabotage=0):
    """runs one call on the emulator -> (ctas, loads, stores, histograms (n_wb, 768), launches, error message)"""
    keep, shared = [], {}
    arr = (ColorDesc * max(len(jobs), 1))(*[desc(d["ptr"], d["w"], d["h"], d["stride"], d["am"], ch, keep, shared) for d, _, _, ch, _ in jobs])
    cap = 2 * sum(len(a) for _, _, a, _, _ in jobs) + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    hist = np.zeros(768 * max(len(jobs), 1), np.uint64)
    nl, ns, nwb, nlaunch = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_int()
    err = C.create_string_buffer(256)
    ctas = L.emu_color(arr, len(jobs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), hist.ctypes.data, hist.size,
                       C.byref(nwb), C.byref(nlaunch), err, 256, sabotage)
    assert nl.value <= cap and ns.value <= cap
    return ctas, loads[:nl.value].tolist(), stores[:ns.value].tolist(), hist[:768 * nwb.value].reshape(-1, 768), nlaunch.value, err.value.decode()


def check(jobs, ctas, ld, st, hist, launches):
    """the properties of the module docstring; raises AssertionError"""
    assert ctas >= 0, ctas
    writing = [j for j in jobs if j[3] and any(s[0] != "enable_transparency" or not j[0]["am"] for s in j[3])]
    want_st, want_ld = set(), []
    for d, _, addrs, chain, h in writing:
        want_st |= addrs
        want_ld += list(addrs) * (2 if h is not None else 1)
    assert launches == (0 if not writing else 3 if any(j[4] is not None for j in writing) else 1), launches
    assert len(set(st)) == len(st), "a pixel stored twice"
    assert set(st) == want_st, "stored set differs from the windows"
    assert sorted(ld) == sorted(want_ld), "loads differ from one per pixel and pass"
    wants = [j[4] for j in writing if j[4] is not None]
    assert len(hist) == len(wants)
    for got, want in zip(hist, wants):
        assert np.array_equal(got, want.reshape(768)), "histogram differs from the oracle's"
    for _, bm, _, _, _ in jobs:
        diff = np.nonzero(bm.buf != bm.exp)[0]
        assert diff.size == 0, ("bytes differ", diff[:4].tolist())


def run(so, n_launches=150, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    fixed = [[make_job(rng, co.preset(k, p), s, am) for k in range(10) for p in (-0.5, 0.3) for am in (False, True)] for s in SIZES[:5]]
    shared = [[make_job(rng, chain, None, am) for am in (False, True, True, False) for _ in range(2)]
              for chain in (co.preset(co.ALPHA, 0.5) + co.preset(co.CONTRAST, 0.2), co.preset(co.SEPIA) + [("white_balance", None)])]
    for it, jobs in enumerate(fixed + shared + [[make_job(rng) for _ in range(int(rng.integers(1, 7)))] for _ in range(n_launches)]):
        ctas, ld, st, hist, launches, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st, hist, launches)
        except AssertionError as e:
            raise AssertionError((it, [(j[0], j[3]) for j in jobs], e.args))
        cases += len(jobs)
    return cases


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (color_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    chain = co.preset(co.BRIGHTNESS, 0.1) + co.preset(co.SEPIA) + [("white_balance", None)] + co.preset(co.CONTRAST, 0.2)
    jobs = [make_job(rng, chain, (300, 21), True) for _ in range(3)]
    ctas, ld, st, hist, launches, err = launch(L, jobs, sabotage=kind)
    try:
        check(jobs, ctas, ld, st, hist, launches)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 150))

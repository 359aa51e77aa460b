"""python -m tests.cpu_emu.run_round_corners_cases <libround_corners_emu.so> [n_launches]: the emulated round_corners_kernel
(tests/cpu_emu/round_corners_kernel_emu.cc) against the oracle.  Also the body of the AddressSanitizer run (the test starts it in a
subprocess with libasan preloaded).

Every launch holds several jobs, each a sub-window of one larger bitmap filled with random sentinel bytes.  Per launch:
  - the whole bitmap equals the oracle applied to each window in turn (results, and every byte outside the windows unchanged);
  - no pixel is stored twice (every pixel belongs to at most one thread);
  - the pixels stored are exactly the pixels the oracle writes (its touch mask);
  - the pixels loaded are pixels the oracle writes too (only blended pixels are read), each at most once."""
import ctypes as C
import sys

import numpy as np

import oracle
from tests import round_corners_oracle as rco
from imageflow_b200._lib import RoundCornersDesc

SOURCES = ("round_corners_kernel_emu.cc", "ifb_round_corners.cc")          # of tests.cpu_emu.build


def load(so):
    L = C.CDLL(so)
    L.emu_round_corners.restype = C.c_long
    L.emu_round_corners.argtypes = [C.POINTER(RoundCornersDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    return L


RADII = [0.0, 0.3, 1.0, 2.5, 3.7, 7.0, 12.5, 19.5, 100.0, -2.0, float("nan"), float("inf"), float("-inf")]


def _job(rng):
    w, h = int(rng.integers(1, 41)), int(rng.integers(1, 41))
    mode = int(rng.integers(0, 5))
    radius = [float(rng.choice(RADII)) if rng.random() < 0.4 else float(rng.uniform(0, 22)) for _ in range(4)]
    if mode in (0, 3) and rng.random() < 0.5:
        radius = [float(rng.choice([0.0, 12.0, 50.0, 100.0, 175.0])) for _ in range(4)]
    matte = [int(v) for v in rng.integers(0, 256, 4)]
    if rng.random() < 0.2:
        matte = [0, 0, 0, 0]
    return w, h, mode, radius, matte


def run(so, n_launches=600, seed=1):
    L = load(so)
    t_lin = oracle.byte_to_float_table(True)
    lut = oracle.linear_to_srgb_table()
    cases = 0
    rng = np.random.default_rng(seed)
    for it in range(n_launches):
        jobs = [_job(rng) for _ in range(int(rng.integers(1, 8)))]
        if it % 97 == 0:
            jobs.append((int(rng.integers(150, 420)), int(rng.integers(150, 420)), int(rng.integers(0, 5)), [float(rng.uniform(0, 220))] * 4, [9, 8, 7, 200]))
        # windows stacked vertically inside one bitmap, each with a random left margin and a gap row, padded pitch
        bw = max(w for w, *_ in jobs) + 8
        pitch = bw * 4 + int(rng.integers(0, 3)) * 4 + 16
        rows = sum(h + 2 for _, h, *_ in jobs) + 1
        buf = rng.integers(0, 256, (rows, pitch), dtype=np.uint8)
        buf.reshape(-1)[3::4][rng.random(buf.size // 4) < 0.2] = 0
        exp = buf.copy()
        descs = (RoundCornersDesc * len(jobs))()
        want_stores, y = set(), 1
        for d, (w, h, mode, radius, matte) in zip(descs, jobs):
            x0 = int(rng.integers(0, bw - w + 1))
            off = y * pitch + x0 * 4
            view = np.lib.stride_tricks.as_strided(exp.reshape(-1)[off:], (h, w, 4), (pitch, 4, 1))
            mask = rco.round_corners(view, mode, radius, matte, want_mask=True)
            ys, xs = np.nonzero(mask)
            want_stores.update((buf.ctypes.data + off + ys * pitch + xs * 4).tolist())
            d.px = buf.ctypes.data + off; d.w = w; d.h = h; d.stride = pitch; d.mode = mode
            d.radius = (C.c_float * 4)(*radius); d.matte_bgra = (C.c_uint8 * 4)(*matte)
            y += h + 2
        cap = sum(w * h for w, h, *_ in jobs) * 2 + 16
        loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
        nl, ns = C.c_size_t(), C.c_size_t()
        err = C.create_string_buffer(256)
        ctas = L.emu_round_corners(descs, len(jobs), t_lin.ctypes.data, lut.ctypes.data, loads.ctypes.data, stores.ctypes.data, cap,
                                   C.byref(nl), C.byref(ns), err, 256)
        assert ctas >= 0, err.value.decode()
        assert nl.value <= cap and ns.value <= cap
        st, ld = stores[:ns.value].tolist(), loads[:nl.value].tolist()
        assert len(set(st)) == len(st), ("a pixel stored twice", jobs)
        assert set(st) == want_stores, ("stored set differs from the oracle's touch mask", jobs)
        assert len(set(ld)) == len(ld) and set(ld) <= want_stores, ("unexpected loads", jobs)
        bad = np.argwhere(buf != exp)
        assert bad.size == 0, ("bytes differ", jobs, bad[:4].tolist())
        cases += len(jobs)
    return cases


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 600))

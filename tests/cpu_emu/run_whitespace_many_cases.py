"""python -m tests.cpu_emu.run_whitespace_many_cases <libwhitespace_many_emu.so> [n_launches]: the emulated whitespace_segments_kernel
and whitespace_walk_kernel (tests/cpu_emu/whitespace_many_emu.cc, with the product's planner) against oracle.detect_content.  Also the
body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Each launch holds several frames of the _images corpora of tests/test_whitespace_product.py and of the geometries of
tests/test_whitespace_plan.py, at thresholds 0, 1, 80 and 255 and both alpha modes, each frame in a bitmap of its own whose row pitch
is often wider than the frame.  Per launch: every rectangle and every count of window-interior pixels visited equals the oracle's;
two launches at most; no frame's walk met a window the summaries cannot replay (a window whose columns would depend on the box); the
sentinel words around the summaries are intact and every summary byte was written."""
import ctypes as C
import sys

import numpy as np

import oracle
from imageflow_b200._lib import DetectContentDesc
from tests.test_whitespace_product import _images

SOURCES = ("whitespace_many_emu.cc", "ifb_whitespace.cc")     # of tests.cpu_emu.build
THRESHOLDS = (0, 1, 80, 255)


def load(so):
    L = C.CDLL(so)
    L.emu_detect_content_many.restype = C.c_long
    L.emu_detect_content_many.argtypes = [C.POINTER(DetectContentDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(C.c_int),
                                          C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.emu_detect_content_plan.restype = C.c_long
    L.emu_detect_content_plan.argtypes = [C.POINTER(DetectContentDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    return L


def geometry_frames(rng):
    """frames of the planner's geometries with a few random blobs: w, h in 3..10, every (w - 1) mod 290 in {0..3}, tall narrow and
    wide short frames"""
    sizes = [(w, h) for w in range(3, 11) for h in range(3, 11)]
    sizes += [(290 * k + 1 + r, int(rng.integers(3, 40))) for k in (1, 2) for r in range(4)]
    sizes += [(int(rng.integers(3, 41)), int(rng.integers(200, 2001))) for _ in range(12)]
    sizes += [(int(rng.integers(600, 2000)), int(rng.integers(3, 12))) for _ in range(8)]
    for w, h in sizes:
        a = np.full((h, w, 4), 255, np.uint8)
        for _ in range(int(rng.integers(0, 4))):
            x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
            a[y:y + int(rng.integers(1, 6)), x:x + int(rng.integers(1, 6))] = rng.integers(0, 256, 4)
        yield a


def corpus(rng, n_images):
    """(frame, threshold, alpha_meaningful): the corpora of the product walk's tests at the thresholds above, then the geometries"""
    for seed in (11, 23, 5):
        for a, _, _ in _images(n_images, seed):
            yield a, int(rng.choice(THRESHOLDS)), bool(rng.integers(0, 2))
    for a in geometry_frames(rng):
        yield a, int(rng.choice(THRESHOLDS)), bool(rng.integers(0, 2))


def padded(rng, a):
    """a in a bitmap of its own with a row pitch of at least its width, often wider"""
    h, w = a.shape[:2]
    pitch = w * 4 + 4 * int(rng.choice([0, 0, 1, 3, 16]))
    buf = np.full((h, pitch), 0x77, np.uint8)
    v = np.lib.stride_tricks.as_strided(buf, (h, w, 4), (pitch, 4, 1))
    v[...] = a
    return buf, v


def launch(L, frames):
    """one emulated call over [(bitmap view, threshold, alpha_meaningful)] -> (rects, visited, launches, bad, guards_ok, unwritten, err)"""
    n = len(frames)
    arr = (DetectContentDesc * n)()
    for d, (v, thr, am) in zip(arr, frames):
        d.px, d.w, d.h, d.stride, d.alpha_meaningful, d.threshold = v.ctypes.data, v.shape[1], v.shape[0], v.strides[0], int(am), thr
    rects, visited = np.zeros((n, 4), np.uint32), np.zeros(n, np.uint64)
    la, bad, ok, unw = C.c_int(), C.c_int(), C.c_int(), C.c_uint64()
    err = C.create_string_buffer(256)
    r = L.emu_detect_content_many(arr, n, rects.ctypes.data, visited.ctypes.data, C.byref(la), C.byref(bad), C.byref(ok), C.byref(unw), err, 256)
    return r, rects, visited, la.value, bad.value, ok.value, unw.value, err.value.decode()


def run(so, n_launches=10**9, seed=1, n_images=400):
    L = load(so)
    rng = np.random.default_rng(seed)
    frames, launches, cases = [], 0, 0

    def flush():
        nonlocal frames, launches, cases
        if not frames:
            return
        r, rects, visited, la, bad, ok, unw, err = launch(L, [(v, t, am) for _, v, t, am in frames])
        assert r >= 0 and not err, err
        assert la <= 2 and bad == 0 and ok == 1 and unw == 0, (la, bad, ok, unw)
        for (a, _, thr, am), got, n in zip(frames, rects, visited):
            want, wn = oracle.detect_content(np.ascontiguousarray(a), thr, am)
            assert tuple(int(x) for x in got) == want and int(n) == wn, (a.shape, thr, am, tuple(got), want, int(n), wn)
        cases += len(frames)
        launches += 1
        frames = []

    for a, thr, am in corpus(rng, n_images):
        buf, v = padded(rng, a)
        frames.append((a, v, thr, am))
        if len(frames) >= int(rng.integers(1, 12)):
            flush()
            if launches >= n_launches:
                return cases
    flush()
    return cases


if __name__ == "__main__":
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 10**9
    print("cases exact:", run(sys.argv[1], n, n_images=400 if n > 10**6 else 60))

"""Host half of the product's detect_content (imageflow_b200/csrc/ifb_whitespace.cc): the reference's window walk
(graphics/whitespace.rs:333-421) over a per-pixel code map, checked on the CPU against the oracle -- rectangle and number of
pixels visited -- with the code map taken from the oracle (on a GPU box the map comes from whitespace_codes_kernel)."""
import numpy as np
import pytest

import oracle


def _images(n, seed):
    rng = np.random.default_rng(seed)
    for it in range(n):
        w, h = [(int(rng.integers(3, 1200)), int(rng.integers(3, 40))), (int(rng.integers(3, 40)), int(rng.integers(3, 1200))),
                (int(rng.integers(3, 400)), int(rng.integers(3, 400))), (int(rng.integers(280, 700)), int(rng.integers(3, 30)))][it % 4]
        if it % 50 == 0:
            w, h = int(rng.integers(1, 4)), int(rng.integers(1, 9))              # below 3 pixels: the whole bitmap (whitespace.rs:288-290)
        a = np.zeros((h, w, 4), np.uint8)
        if rng.random() < 0.3:
            a[...] = rng.integers(0, 256, 4)
        for _ in range(int(rng.integers(0, 8))):
            x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
            if rng.random() < 0.5:
                a[y:y + int(rng.integers(1, 4)), x:x + int(rng.integers(1, 4))] = rng.integers(0, 256, 4)
            else:
                x2, y2 = int(rng.integers(x, w)) + 1, int(rng.integers(y, h)) + 1
                a[y:y2, x:x2] = rng.integers(0, 256, (y2 - y, x2 - x, 4))
        yield a, int(rng.choice([0, 1, 5, 30, 80])), bool(rng.integers(0, 2))


def test_window_walk_matches_the_oracle():
    import imageflow_b200 as ifb
    for a, thr, am in _images(800, 11):
        assert ifb.detect_content_from_codes(oracle.whitespace_codes(a, thr, am)) == oracle.detect_content(a, thr, am), (a.shape, thr, am)


def test_reference_known_answers_through_the_product_walk():               # smoke.rs:420-475 and a slice of :477-592
    import imageflow_b200 as ifb
    red = (0, 0, 255, 255)
    a = np.zeros((10, 10, 4), np.uint8); a[1:9, 1:9] = red
    assert ifb.detect_content_from_codes(oracle.whitespace_codes(a, 1))[0] == (1, 1, 9, 9)
    b = np.zeros((100, 100, 4), np.uint8); b[3:70, 2:70] = red
    assert ifb.detect_content_from_codes(oracle.whitespace_codes(b, 1))[0] == (2, 3, 70, 70)
    for (w, h) in [(3, 3), (7, 11), (11, 4)]:                               # every dot position of the small canvases
        for x in range(w):
            for y in range(h):
                for (sw, sh) in [(1, 1), (2, 2), (2, 1)]:
                    if (w, h, x, y) == (3, 3, 1, 1) or x + sw > w or y + sh > h:
                        continue
                    c = np.zeros((h, w, 4), np.uint8); c[y:y + sh, x:x + sw] = red
                    assert ifb.detect_content_from_codes(oracle.whitespace_codes(c, 1))[0] == (x, y, x + sw, y + sh), (w, h, x, y, sw, sh)
    for (x, y, rw, rh) in [(67, 0, 1, 1), (881, 881, 1, 1), (0, 1, 1, 1), (1, 67, 1896, 1370)]:   # the large canvases of the reference test
        if x + rw <= 3000 and y + rh <= 2000:
            c = np.zeros((2000, 3000, 4), np.uint8); c[y:y + rh, x:x + rw] = red
            assert ifb.detect_content_from_codes(oracle.whitespace_codes(c, 1))[0] == (x, y, x + rw, y + rh), (x, y, rw, rh)


def test_kernel_source_under_cpu_emulation_matches_the_oracle(tmp_path):
    """tests/cpu_emu/whitespace_kernel_emu.cc compiles the product's CUDA source of whitespace_codes_kernel (unmodified) with
    g++ under a sequential emulation of threadIdx / blockIdx / __shared__ / __syncthreads and runs it with the launch geometry
    the engine uses: every code byte must equal the oracle's, for ragged sizes, padded pitches, both grayscale formulas."""
    import ctypes as C
    from tests import cpu_emu
    L = C.CDLL(cpu_emu.build(str(tmp_path), "whitespace_kernel_emu.cc"))
    L.emu_whitespace_codes.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p]
    for a, thr, am in _images(200, 5):
        h, w = a.shape[:2]
        pitch = (w * 4 + 63) // 64 * 64                                   # like the engine's device copies
        buf = np.zeros((h, pitch), np.uint8)
        np.lib.stride_tricks.as_strided(buf, (h, w, 4), (pitch, 4, 1))[...] = a
        codes = np.full((h, w), 7, np.uint8)
        L.emu_whitespace_codes(buf.ctypes.data, w, h, pitch, int(am), thr, codes.ctypes.data)
        assert np.array_equal(codes, oracle.whitespace_codes(a, thr, am)), (a.shape, thr, am)


def test_bad_code_maps_are_rejected():
    import imageflow_b200 as ifb
    with pytest.raises(ifb.FlowError):
        ifb.detect_content_from_codes(np.zeros((0, 5), np.uint8))

"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/ifb200.h declares,
its host logic (weights, tables, colour-filter matrices, argument validation) matches the reference's golden vectors,
and the product never routes through the oracle.  No GPU compute is called here."""
import ctypes as C
import glob
import gzip
import json
import os
import re
import subprocess

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(os.path.dirname(__file__), "golden")


def test_library_loads_and_exports_every_declared_symbol():
    L = ifb.lib()
    hdr = open(os.path.join(ROOT, "include", "ifb200.h")).read()
    declared = sorted(set(re.findall(r"^(?:uint32_t|uint64_t|const char\*|int|void)\s+(ifb200_[a-z0-9_]+)\s*\(", hdr, re.M)))
    assert declared, "no declarations found in include/ifb200.h"
    for name in declared:
        assert hasattr(L, name), f"{name} declared in ifb200.h but not exported by libifb200.so"
    assert sorted(_lib.SYMBOLS) == declared
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (ifb200_[a-z0-9_]+)", out))
    assert exported == set(declared)
    assert L.ifb200_abi_version() == (1 << 16) | 2


def test_desc_struct_layout_matches_header():
    # field order/sizes of ifb200_resample_desc (include/ifb200.h) on LP64
    d = _lib.ResampleDesc
    offs = {n: getattr(d, n).offset for n, _ in d._fields_}
    assert offs["in_"] == 0 and offs["in_w"] == 8 and offs["in_stride"] == 16 and offs["canvas"] == 24
    assert offs["cv_w"] == 32 and offs["x"] == 44 and offs["filter"] == 60 and offs["sharpen_percent"] == 64
    assert offs["linear"] == 68 and offs["alpha_meaningful"] == 72 and offs["compose"] == 76 and offs["matte_bgra"] == 80
    assert offs["color_matrix"] == 88 and C.sizeof(d) == 96


def test_product_weights_match_reference_golden_tables():
    """The product's own populate_weights (csrc/ifb_weights.cc) against weights.txt / weights_params.txt."""
    with gzip.open(os.path.join(G, "weights_golden.json.gz"), "rt") as f:
        g = json.load(f)

    def cmp(got, exp):
        assert len(got) == len(exp)
        for (l, r, w), e in zip(got, exp):
            assert len(w) == len(e) == r - l + 1
            assert np.max(np.abs(w.astype(np.float64) - np.array(e))) <= 1e-6

    for r in g["weights"]:
        cmp(ifb.populate_weights(r["filter"], r["out"], r["in"]), r["w"])
    errors = 0
    for r in g["params"]:
        if r.get("error"):
            with pytest.raises(ifb.FlowError) as e:
                ifb.populate_weights(r["filter"], r["out"], r["in"], r["kernel_scale"], r["lobe_mode"], r["lobe_value"])
            assert e.value.kind == ifb.ErrorKind.TotalWeightZero
            errors += 1
        else:
            cmp(ifb.populate_weights(r["filter"], r["out"], r["in"], r["kernel_scale"], r["lobe_mode"], r["lobe_value"]), r["w"])
    assert errors == 6


def test_product_and_oracle_weights_are_bit_identical():
    import oracle
    for f in (1, 2, 3, 4, 6, 8, 10, 13, 14, 16, 17, 22, 24, 27, 29, 31):
        for (i, o) in ((3840, 512), (2160, 512), (1080, 2160), (640, 200), (7, 3), (33, 7), (5, 9)):
            a = ifb.populate_weights(f, o, i)
            b = oracle.weights(f, o, i)
            for (l1, r1, w1), (l2, r2, w2) in zip(a, b):
                assert (l1, r1) == (l2, r2) and np.array_equal(w1.view(np.uint32), w2.view(np.uint32))
    a = ifb.populate_weights(2, 512, 3840, 1.0, 2, 50.0)
    b = oracle.weights(2, 512, 3840, 1.0, 2, 50.0)
    assert all(np.array_equal(x[2].view(np.uint32), y[2].view(np.uint32)) for x, y in zip(a, b))


def test_product_tables_match_reference_and_oracle():
    import oracle
    L = ifb.lib()
    lut = np.zeros(16384, np.uint8)
    L.ifb200_linear_to_srgb_table(lut.ctypes.data_as(C.POINTER(C.c_uint8)))
    with gzip.open(os.path.join(G, "lut16k_golden.bin.gz"), "rb") as f:
        assert np.array_equal(lut, np.frombuffer(f.read(), np.uint8))          # lut.rs:14
    for linear in (0, 1):
        t = np.zeros(256, np.float32)
        L.ifb200_byte_to_float_table(linear, t.ctypes.data_as(C.POINTER(C.c_float)))
        assert np.array_equal(t.view(np.uint32), oracle.byte_to_float_table(bool(linear)).view(np.uint32))
    for which, p in ((0, 0), (1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (6, .25), (7, .5), (8, -.1), (9, 2.0)):
        assert np.array_equal(ifb.color_filter_matrix(which, p), oracle.color_filter_matrix(which, p))
    with pytest.raises(ifb.FlowError):
        ifb.color_filter_matrix(99)


def test_no_cuda_device_fails_loudly_not_silently():
    """In the CPU container every compute entry point must report NoDevice -- there is no CPU fallback."""
    if ifb.device_count() > 0:
        pytest.skip("a CUDA device is present")
    a = np.zeros((8, 8, 4), np.uint8)
    c = np.zeros((4, 4, 4), np.uint8)
    with pytest.raises(ifb.FlowError) as e:
        ifb.scale_and_render(ifb.BitmapWindow.from_numpy(a), ifb.BitmapWindow.from_numpy(c), ifb.ScaleAndRenderParams(w=4, h=4))
    assert e.value.kind == ifb.ErrorKind.NoDevice and "no CPU fallback" in str(e.value)
    with pytest.raises(ifb.FlowError) as e:
        ifb.window_bgra32_apply_color_matrix(ifb.BitmapWindow.from_numpy(a), ifb.color_filter_matrix(0))
    assert e.value.kind == ifb.ErrorKind.NoDevice
    with pytest.raises(ifb.FlowError) as e:
        ifb.Batch(0)
    assert e.value.kind == ifb.ErrorKind.NoDevice


def test_argument_validation_precedes_device_use():
    a = np.zeros((8, 8, 4), np.uint8)
    c = np.zeros((4, 4, 4), np.uint8)
    wi, wc = ifb.BitmapWindow.from_numpy(a), ifb.BitmapWindow.from_numpy(c)
    with pytest.raises(ifb.FlowError) as e:                                   # scaling.rs:24-29
        ifb.scale_and_render(wi, wc, ifb.ScaleAndRenderParams(x=3, y=0, w=2, h=4))
    assert e.value.kind == ifb.ErrorKind.InvalidArgument and "out of bounds" in str(e.value)
    with pytest.raises(ifb.FlowError) as e:
        ifb.scale_and_render(wi, wc, ifb.ScaleAndRenderParams(w=4, h=4, interpolation_filter=99))
    assert e.value.kind == ifb.ErrorKind.BadFilter
    wi.pixel_layout = "BGR"
    with pytest.raises(ifb.FlowError) as e:                                   # scaling.rs:43-48
        ifb.scale_and_render(wi, wc, ifb.ScaleAndRenderParams(w=4, h=4))
    assert e.value.kind == ifb.ErrorKind.MethodNotImplemented
    assert wc.window(0, 0, 5, 4) is None and wc.window(1, 1, 3, 4).w == 2     # bitmaps.rs:413-431


def test_plan_tables_build_on_the_host_for_any_geometry():
    """Host half of the engine (no CUDA call): plans -- weights as weights.rs, ring/tile tables -- for ordinary, ragged, tiny,
    up-scaling and extreme geometries.  A down-scale whose H windows are wider than a ring-kernel strip (3000 -> 1 columns)
    must not fail: it is planned for the generic pair.  The tables do not depend on the number of builder threads."""
    import imageflow_b200 as ifb
    geos = [(3840, 2160, 512, 512, 2), (3840, 2160, 512, 512, 6), (7680, 4320, 1920, 1080, 2, 50.0), (1920, 1080, 3840, 2160, 14),
            (33, 17, 7, 5, 2), (8, 8, 1, 1, 2), (4, 4, 4, 1, 17), (1, 1, 1, 1, 2), (1, 1, 300, 200, 14),
            (3000, 8, 1, 1, 2), (2500, 6, 2, 3, 6), (16, 4000, 3, 1, 2), (4097, 3, 1030, 2, 13)]
    one = ifb.plan_probe(geos, threads=1, want_hash=True)
    four = ifb.plan_probe(geos, threads=4, want_hash=True)
    assert one["table_hash"] == four["table_hash"] and one["table_bytes"] == four["table_bytes"] > 0
    assert ifb.plan_probe([], threads=2)["table_bytes"] == 0
    # regression pins (cubic filters only: polynomial f64 arithmetic, no libm): the kernel tables of the benchmark geometries
    # as the build whose kernel source passes tests/test_hv_emulation.py lays them out (round 2: streaming H-then-V ring kernel).
    # A deliberate change of the table layout updates these constants.
    pins = {((3840, 2160, 512, 512, 2),): (0xf4276ae5577da3e2, 354480),
            ((7680, 4320, 1920, 1080, 2, 50.0),): (0x4d5a0cc2c88695c1, 224000),
            ((1920, 1080, 3840, 2160, 14),): (0xe0ce1caa7adbc55b, 0),            # up-scale: tile kernel, no ring tables
            ((640, 480, 200, 150, 2), (33, 17, 7, 5, 2)): (0x5175ec0383b3940b, 82835)}
    for geo, (h, nbytes) in pins.items():
        r = ifb.plan_probe(list(geo), threads=1, want_hash=True)
        assert (r["table_hash"], r["table_bytes"]) == (h, nbytes), geo
    for bad in [(0, 4, 1, 1, 2), (4, 4, 0, 1, 2), (4, 4, 1, 1, 77)]:
        with pytest.raises(ifb.FlowError):
            ifb.plan_probe([bad])


def test_descriptor_arrays_are_filled_in_place_like_single_descriptors():
    """Batch.make_descs writes into the array elements directly; every field must come out as in the one-job path"""
    import ctypes as C
    import imageflow_b200 as ifb
    from imageflow_b200 import graphics
    rng = np.random.default_rng(3)
    jobs = []
    for i in range(200):
        a = ifb.BitmapWindow(int(rng.integers(1, 1 << 47)), int(rng.integers(1, 9000)), int(rng.integers(1, 9000)), int(rng.integers(4, 9000)) * 4,
                             alpha_meaningful=bool(rng.integers(0, 2)))
        b = ifb.BitmapWindow(int(rng.integers(1, 1 << 47)), int(rng.integers(1, 9000)), int(rng.integers(1, 9000)), int(rng.integers(4, 9000)) * 4,
                             compose=ifb.BitmapCompositing(int(rng.integers(0, 3))),
                             matte_bgra=tuple(int(v) for v in rng.integers(0, 256, 4)) if i % 2 else (0, 0, 0, 0))
        p = ifb.ScaleAndRenderParams(x=int(rng.integers(0, 50)), y=int(rng.integers(0, 50)), w=int(rng.integers(1, 4000)), h=int(rng.integers(1, 4000)),
                                     sharpen_percent_goal=float(rng.choice([0.0, 25.0])), interpolation_filter=ifb.Filter(int(rng.integers(1, 32))),
                                     scale_in_colorspace=ifb.WorkingFloatspace(int(rng.integers(0, 2))))
        jobs.append((a, b, p, ifb.color_filter_matrix(0)) if i % 5 == 0 else (a, b, p))
    arr, keep = ifb.Batch.make_descs(ifb.Batch.__new__(ifb.Batch), jobs)
    assert len(keep) == 41                                    # 40 colour matrices + the list that keeps the bitmaps alive
    sz, off = C.sizeof(ifb.ResampleDesc), ifb.ResampleDesc.color_matrix.offset
    for i, j in enumerate(jobs):
        one = bytearray(bytes(graphics._desc(*j)))
        got = bytearray(bytes(arr)[i * sz:(i + 1) * sz])
        for blob in (one, got):                               # the matrix pointer differs per call: compare what it points at
            ptr = int.from_bytes(blob[off:off + 8], "little")
            assert (ptr != 0) == (len(j) > 3)
            if ptr:
                assert np.array_equal(np.ctypeslib.as_array((C.c_float * 25).from_address(ptr)), ifb.color_filter_matrix(0).reshape(25))
            blob[off:off + 8] = bytes(8)
        assert one == got, i


def test_tile_kernel_float_quotients_are_exact():
    """fused_tile2_kernel starts a thread's items at (t / ic, t % ic) and advances by 256 / ic without an integer division:
    q = (int)((t + 0.5f) * (1.0f / ic)) and (int)(256.5f * (1.0f / ic)).  Exact for every t < 256 and every tile width."""
    t = np.arange(256, dtype=np.float32)
    for ic in range(1, 40000):
        ric = np.float32(1.0) / np.float32(ic)
        assert np.array_equal(((t + np.float32(0.5)) * ric).astype(np.int32), np.arange(256) // ic), ic
        assert int(np.float32(256.5) * ric) == 256 // ic, ic


def test_product_never_touches_the_oracle():
    """The oracle is test infrastructure: nothing under imageflow_b200/ or include/ may import, link or name it."""
    # functional references only (comments may mention that the oracle exists)
    pat = re.compile(r"^\s*(import|from)\s+oracle|#\s*include\s*[<\"][^>\"]*oracle|\bifo_[a-z_]+\s*\(|libifb_oracle|-lifb_oracle|oracle/")
    offenders = []
    for path in glob.glob(os.path.join(ROOT, "imageflow_b200", "**", "*"), recursive=True) + glob.glob(os.path.join(ROOT, "include", "*")):
        if os.path.isdir(path) or path.endswith((".so", ".o", ".pyc", ".log")):
            continue
        txt = open(path, errors="replace").read()
        for ln, line in enumerate(txt.splitlines(), 1):
            if pat.search(line) and "identical in every kernel here and in oracle/" not in line and "anything from oracle/" not in line:
                offenders.append(f"{os.path.relpath(path, ROOT)}:{ln}: {line.strip()[:100]}")
    assert not offenders, "\n".join(offenders)
    out = subprocess.run(["ldd", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in out
    syms = subprocess.run(["nm", "-D", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "ifo_" not in syms


def test_synthetic_generators_are_seed_stable():
    from imageflow_b200 import synth
    import torch
    a = synth.noise_np(64, 48, 3, "mixed")
    assert np.array_equal(a, synth.noise_torch(64, 48, 3, "mixed", device="cpu").numpy())
    assert int(a.astype(np.uint64).sum()) == int(synth.noise_np(64, 48, 3, "mixed").astype(np.uint64).sum())
    g = synth.gradient_np(300, 270)
    assert g[5, 7].tolist() == [7, 5, 12, 255] and g[269, 299].tolist() == [299 % 256, 269 % 256, (299 + 269) % 256, 255]
    assert np.array_equal(g, synth.gradient_torch(300, 270, device="cpu").numpy())

"""ctypes loader of libifb_units.so (TEST INFRASTRUCTURE): units_probe.cu, the product's store-epilogue device functions compiled
with the product's flags and called on arrays.  __graft_entry__.build() builds it next to this file; a GPU test that needs it
fails when it is missing (there is nothing to fall back to)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("IFB_UNITS_LIB") or os.path.join(_HERE, "libifb_units.so")   # IFB_UNITS_LIB: A/B builds during development

REPORT_WORDS = 72                  # struct Report in units_probe.cu

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(LIB_PATH)
    p, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.ifbu_rcp.argtypes = [p, p]
    L.ifbu_div3.argtypes = [i32, p, u64, p, p]
    L.ifbu_div3_edges.argtypes = [p, p, u32, p, u32]
    L.ifbu_clamp.argtypes = [p, p]
    L.ifbu_encode.argtypes = [p, p, p, p]
    L.ifbu_epilogue.argtypes = [i32, i32, i32, i32, i32, p, p, u32, u32, p, p, p, p, p]
    for f in ("ifbu_rcp", "ifbu_div3", "ifbu_div3_edges", "ifbu_clamp", "ifbu_encode", "ifbu_epilogue"):
        getattr(L, f).restype = i32
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    assert rc == 0, f"{what}: CUDA error {rc}"


class Reports:
    """n device-side reports (trials, mismatches, the first 16 counterexamples) in one int32 CUDA tensor"""

    def __init__(self, torch, n: int):
        self.t = torch.zeros(n * REPORT_WORDS, dtype=torch.int32, device="cuda")
        self.n = n

    def ptr(self, k: int = 0) -> int:
        return self.t.data_ptr() + k * REPORT_WORDS * 4

    def read(self):
        """-> [(trials, mismatches, [(a, b, got, expected), ...])] as raw 32-bit words"""
        w = self.t.cpu().numpy().view(np.uint32).reshape(self.n, REPORT_WORDS).astype(np.uint64)
        out = []
        for r in w:
            trials = int(r[0] | (r[1] << np.uint64(32)))
            bad = int(r[2] | (r[3] << np.uint64(32)))
            n_ex = min(int(r[4]), 16)
            out.append((trials, bad, [tuple(int(v) for v in r[8 + 4 * k:12 + 4 * k]) for k in range(n_ex)]))
        return out

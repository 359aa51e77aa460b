"""Seed-stable synthetic BGRA frames (SURVEY.md §8d), numpy and torch flavours producing identical bytes.

gradient: B=x%256, G=y%256, R=(x+y)%256, A=255   (reference bench: benches/bench_graphics.rs:405-414)
noise   : counter hash of (0x1F2E3D4C+seed, x, y), uniform u8 per channel; alpha 'opaque' or 'mixed'
          (25 % exactly 0, 25 % exactly 255, rest uniform) -- worst case for the LUT gathers.
cutout  : a transparent PNG (logo / cut-out): opaque shapes, one-pixel lines and ~1 % isolated opaque pixels on an alpha-0 field
          whose colour bytes are non-zero; patches of alpha 253 / 254 (filtered, they straddle BlendWithSelf's 0.994); 0/255
          colour checkerboards inside the opaque disc.  A down-scale of it reaches every alpha edge of the store epilogue
          (a == 0, a < 0, a tiny, a > 1, a near 0.994), which noise averages away.
cutout_canvas: a canvas for BlendWithSelf with alpha-0, opaque and partial-alpha blocks (fa == 0 and fa < 0 over it).
"""
from __future__ import annotations

import numpy as np

_M = 0xFFFFFFFF


def gradient_np(w: int, h: int, alpha: int = 255) -> np.ndarray:
    x = np.arange(w, dtype=np.uint32)[None, :]
    y = np.arange(h, dtype=np.uint32)[:, None]
    a = np.empty((h, w, 4), np.uint8)
    a[..., 0] = (x % 256).astype(np.uint8)
    a[..., 1] = (y % 256).astype(np.uint8)
    a[..., 2] = ((x + y) % 256).astype(np.uint8)
    a[..., 3] = alpha
    return a


def _mix_np(v):
    v = v.astype(np.uint64)
    v ^= v >> np.uint64(16)
    v = (v * np.uint64(0x7FEB352D)) & np.uint64(_M)
    v ^= v >> np.uint64(15)
    v = (v * np.uint64(0x846CA68B)) & np.uint64(_M)
    v ^= v >> np.uint64(16)
    return v


def noise_np(w: int, h: int, seed: int = 0, alpha_mode: str = "opaque") -> np.ndarray:
    x = np.arange(w, dtype=np.uint64)[None, :]
    y = np.arange(h, dtype=np.uint64)[:, None]
    k = ((x * np.uint64(0x9E3779B1)) & np.uint64(_M)) ^ ((y * np.uint64(0x85EBCA77)) & np.uint64(_M)) ^ np.uint64((0x1F2E3D4C + seed) & _M)
    base = _mix_np(k)
    a = np.empty((h, w, 4), np.uint8)
    a[..., 0] = (base & np.uint64(0xFF)).astype(np.uint8)
    a[..., 1] = ((base >> np.uint64(8)) & np.uint64(0xFF)).astype(np.uint8)
    a[..., 2] = ((base >> np.uint64(16)) & np.uint64(0xFF)).astype(np.uint8)
    if alpha_mode == "opaque":
        a[..., 3] = 255
    else:
        h2 = _mix_np(base ^ np.uint64(0xA5A5A5A5))
        sel = (h2 >> np.uint64(24)) & np.uint64(3)
        al = ((h2 >> np.uint64(8)) & np.uint64(0xFF))
        a[..., 3] = np.where(sel == 0, 0, np.where(sel == 1, 255, al)).astype(np.uint8)
    return a


def _mix_t(v):
    v = v ^ (v >> 16)
    v = (v * 0x7FEB352D) & _M
    v = v ^ (v >> 15)
    v = (v * 0x846CA68B) & _M
    v = v ^ (v >> 16)
    return v


def noise_torch(w: int, h: int, seed: int = 0, alpha_mode: str = "opaque", device="cuda", out=None):
    """Same bytes as noise_np, computed on `device` (int64 arithmetic masked to 32 bits)."""
    import torch
    x = torch.arange(w, dtype=torch.int64, device=device)[None, :]
    y = torch.arange(h, dtype=torch.int64, device=device)[:, None]
    k = ((x * 0x9E3779B1) & _M) ^ ((y * 0x85EBCA77) & _M) ^ ((0x1F2E3D4C + seed) & _M)
    base = _mix_t(k)
    if out is None:
        out = torch.empty((h, w, 4), dtype=torch.uint8, device=device)
    out[..., 0] = (base & 0xFF).to(torch.uint8)
    out[..., 1] = ((base >> 8) & 0xFF).to(torch.uint8)
    out[..., 2] = ((base >> 16) & 0xFF).to(torch.uint8)
    if alpha_mode == "opaque":
        out[..., 3] = 255
    else:
        h2 = _mix_t(base ^ 0xA5A5A5A5)
        sel = (h2 >> 24) & 3
        al = (h2 >> 8) & 0xFF
        al = torch.where(sel == 0, torch.zeros_like(al), torch.where(sel == 1, torch.full_like(al, 255), al))
        out[..., 3] = al.to(torch.uint8)
    return out


def _cutout_planes(x, y, w: int, h: int, seed: int, where):
    """(b, g, r, a) of the cut-out frame from int64 coordinate grids; only operators and `where`, so numpy and torch compute
    the same integers (a product that leaves int64 wraps, and the mask to 32 bits keeps the low bits either way)."""
    k = ((x * 0x9E3779B1) & _M) ^ ((y * 0x85EBCA77) & _M) ^ ((0x6C8E9CF5 + seed) & _M)
    base = _mix_t(k)
    h2 = _mix_t(base ^ 0xA5A5A5A5)
    b, g, r = (base & 0xFF) | 1, ((base >> 8) & 0xFF) | 1, ((base >> 16) & 0xFF) | 1        # never 0, also under alpha 0
    zero = x * 0 + y * 0
    a = zero
    s = min(w, h)
    # opaque disc, with 0/255 checkerboards of 1-pixel cells (upper half) and 4-pixel cells (lower half) in every channel
    disc = (2 * x - w) ** 2 + (2 * y - h) ** 2 < (2 * s // 3) ** 2
    cell = where(2 * y < h, (x + y) & 1, ((x >> 2) + (y >> 2)) & 1)
    checker = disc & ((2 * x - w) ** 2 + (2 * y - h) ** 2 < (s // 2) ** 2)
    a = where(disc, zero + 255, a)
    cb = cell * 255
    b, g, r = where(checker, cb, b), where(checker, 255 - cb, g), where(checker, cb, r)
    # opaque bar at the left edge
    a = where((x >= w // 16) & (x < w // 8) & (y >= h // 8) & (y < (7 * h) // 8), zero + 255, a)
    # alpha 254 and 253 patches side by side, and one where they alternate (filtered to ~0.9941)
    band = (y >= h // 10) & (y < (4 * h) // 10)
    a = where(band & (x >= (6 * w) // 8) & (x < (7 * w) // 8), zero + 254, a)
    a = where(band & (x >= (7 * w) // 8) & (x < (15 * w) // 16), zero + 253, a)
    a = where((y >= (6 * h) // 10) & (y < (9 * h) // 10) & (x >= (6 * w) // 8) & (x < (15 * w) // 16), 253 + ((x + y) & 1), a)
    # one-pixel lines: a row, a column, a diagonal
    line = (y == h // 5) | (x == (5 * w) // 7) | ((x == y) & (x < s // 2))
    a = where(line, zero + 255, a)
    # ~1 % isolated opaque pixels
    a = where(((h2 >> 8) & 0xFFFF) < 655, zero + 255, a)
    return b, g, r, a


def cutout_np(w: int, h: int, seed: int = 0) -> np.ndarray:
    x = np.arange(w, dtype=np.int64)[None, :]
    y = np.arange(h, dtype=np.int64)[:, None]
    with np.errstate(over="ignore"):
        planes = _cutout_planes(x, y, w, h, seed, np.where)
    a = np.empty((h, w, 4), np.uint8)
    for c, p in enumerate(planes):
        a[..., c] = np.broadcast_to(p, (h, w)).astype(np.uint8)
    return a


def cutout_torch(w: int, h: int, seed: int = 0, device="cuda", out=None):
    """Same bytes as cutout_np, computed on `device`."""
    import torch
    x = torch.arange(w, dtype=torch.int64, device=device)[None, :]
    y = torch.arange(h, dtype=torch.int64, device=device)[:, None]
    planes = _cutout_planes(x, y, w, h, seed, torch.where)
    if out is None:
        out = torch.empty((h, w, 4), dtype=torch.uint8, device=device)
    for c, p in enumerate(planes):
        out[..., c] = p.expand(h, w).to(torch.uint8)
    return out


def _cutout_canvas_planes(x, y, seed: int, where):
    k = ((x * 0x9E3779B1) & _M) ^ ((y * 0x85EBCA77) & _M) ^ ((0x2B7E1516 + seed) & _M)
    base = _mix_t(k)
    blk = ((x >> 3) + (y >> 3)) % 3                         # 8x8 blocks: alpha 0, alpha 255, partial alpha
    a = where(blk == 0, base * 0, where(blk == 1, base * 0 + 255, (base >> 24) & 0xFF))
    return (base & 0xFF) | 1, ((base >> 8) & 0xFF) | 1, ((base >> 16) & 0xFF) | 1, a


def cutout_canvas_np(w: int, h: int, seed: int = 0) -> np.ndarray:
    x = np.arange(w, dtype=np.int64)[None, :]
    y = np.arange(h, dtype=np.int64)[:, None]
    with np.errstate(over="ignore"):
        planes = _cutout_canvas_planes(x, y, seed, np.where)
    a = np.empty((h, w, 4), np.uint8)
    for c, p in enumerate(planes):
        a[..., c] = np.broadcast_to(p, (h, w)).astype(np.uint8)
    return a


def cutout_canvas_torch(w: int, h: int, seed: int = 0, device="cuda"):
    import torch
    x = torch.arange(w, dtype=torch.int64, device=device)[None, :]
    y = torch.arange(h, dtype=torch.int64, device=device)[:, None]
    out = torch.empty((h, w, 4), dtype=torch.uint8, device=device)
    for c, p in enumerate(_cutout_canvas_planes(x, y, seed, torch.where)):
        out[..., c] = p.expand(h, w).to(torch.uint8)
    return out


def gradient_torch(w: int, h: int, alpha: int = 255, device="cuda", out=None):
    import torch
    x = torch.arange(w, dtype=torch.int64, device=device)[None, :]
    y = torch.arange(h, dtype=torch.int64, device=device)[:, None]
    if out is None:
        out = torch.empty((h, w, 4), dtype=torch.uint8, device=device)
    out[..., 0] = (x % 256).to(torch.uint8).expand(h, w)
    out[..., 1] = (y % 256).to(torch.uint8).expand(h, w)
    out[..., 2] = ((x + y) % 256).to(torch.uint8)
    out[..., 3] = alpha
    return out

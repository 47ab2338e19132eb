"""Seeded full-resolution gray sequences for the dense-flow tests (tests/test_farneback_*.py, tools/make_flow_golden.py):
what Flow::ComputeMask receives before its pyrDown (perfect/src/Flow.cc:26).

  room       consecutive frames of synth.RoomStream (camera moving inside a textured room)
  blobs      static texture with textured discs moving by several pixels per frame
  flat       one grey level everywhere (the solve's 1e-3 term dominates)
  identical  the same textured frame repeated (zero motion, noise included)
  border     a texture sliding diagonally, so content leaves and enters through the image borders
"""
from __future__ import annotations

import numpy as np

from orb_slam2_ssd_semantic_b200 import synth

SCENES = ("room", "blobs", "flat", "identical", "border")

# half-resolution (rows, cols): the live frame's 320 x 240, odd sides, an exact halving with a row tail of 1 (162 -> 81),
# both sides of the pyramid-level cut-offs (min side 63 | 64: 0 | 1 coarser level, 255 | 256: 2 | 3), the smallest size
# the device accepts
HALF_SIZES = ((240, 320), (97, 161), (98, 162), (63, 80), (64, 80), (255, 320), (256, 320), (16, 16))

_ROOMS: dict = {}


def frames(scene: str, rows: int, cols: int, n: int = 2, seed: int = 7, t0: int = 0) -> np.ndarray:
    """-> n x rows x cols uint8, frames t0 .. t0 + n - 1 of the scene."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if scene == "room":
        key = (seed, rows, cols)
        if key not in _ROOMS:
            _ROOMS[key] = synth.RoomStream(seed=seed, h=rows, w=cols, ppm=60.0)
        return np.stack([_ROOMS[key].frame(t0 + t)[0] for t in range(n)])
    if scene == "flat":
        return np.full((n, rows, cols), 128, np.uint8)
    if scene == "identical":
        f = synth.texture(seed, rows, cols, nrect=60, nline=30)
        return np.repeat(np.clip(np.rint(f), 0, 255).astype(np.uint8)[None], n, axis=0)
    if scene == "border":
        pad = 6 * (n + t0) + 8
        big = synth.texture(seed, rows + pad, cols + pad, nrect=80, nline=40)
        out = [big[pad - 6 * (t0 + t) - 4:pad - 6 * (t0 + t) - 4 + rows, pad - 6 * (t0 + t) - 4:pad - 6 * (t0 + t) - 4 + cols]
               for t in range(n)]
        return np.clip(np.rint(np.stack(out)), 0, 255).astype(np.uint8)
    if scene == "blobs":
        base = synth.texture(seed, rows, cols, nrect=60, nline=30)
        tex = synth.texture(seed + 1, rows, cols, nrect=60, nline=30)
        yy, xx = np.mgrid[0:rows, 0:cols]
        nb = 4
        c = rng.uniform(0.2, 0.8, (nb, 2)) * (rows, cols)
        r = rng.uniform(0.08, 0.2, nb) * min(rows, cols) + 3
        v = rng.normal(0, 4.0, (nb, 2))
        out = []
        for t in range(t0, t0 + n):
            img = base.copy()
            for b in range(nb):
                cy, cx = c[b] + v[b] * t
                m = (yy - cy) ** 2 + (xx - cx) ** 2 < r[b] ** 2
                sy, sx = int(round(v[b, 0] * t)), int(round(v[b, 1] * t))
                img[m] = np.roll(tex, (sy, sx), axis=(0, 1))[m]
            out.append(img + np.random.Generator(np.random.PCG64(seed * 1000 + t)).normal(0, 1.5, img.shape))
        return np.clip(np.rint(np.stack(out)), 0, 255).astype(np.uint8)
    raise ValueError(scene)

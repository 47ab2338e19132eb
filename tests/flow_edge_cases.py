"""Crafted half-resolution (prev, cur) u8 pairs for calcOpticalFlowFarneback(prev, cur, None, 0.5, 3, 15, 3, 5, 1.2, 0),
each named after the edges of OpenCV 4.13's code (and so of csrc/flow.cu) it must reach.  `cases()` -> list of Case;
tests/test_farneback_edges_cpu.py checks that every case reaches each edge it declares and that the restatement
(oracle/farneback_py.py) equals cv2 on it, tools/make_farneback_edges_golden.py stores cv2's flow, and
tests/test_farneback_edges_gpu.py runs the device on every case.

Edges a case may declare (axis: "rows" or "cols"; level k: 0 = the half-resolution image, k = 1..3 coarser):
  ("levels", ((h0, w0), (h1, w1), ...))  the pyramid's level sizes, finest first (so also the level count)
  ("resize", (path0, path1, ...))        the image resize at each level: "copy", "area" (INTER_AREA's fast path for an
                                         exact halving of both sides) or "linear"
  ("area_tail", r)                       level 1 takes the area path with a width of r (mod 8), so its 4-wide SIMD
                                         loop leaves a row tail of r % 4 outputs, and a tail cut at 8 would leave r
  ("halves", axis)                      level 1 halves `axis` exactly and not the other side (mixed parity)
  ("round", k, axis, "up" | "down")      side * 0.5^k ends in exactly .5 and cvRound (half to even) goes up / down
  ("cut_below", axis, k)                 level k is not added, and only `axis` stops it: side * 0.5^k lies in
                                         [32 - 0.5^k, 32), one half-resolution pixel short of the cut
  ("cut_at", axis, k)                    level k is added with `axis` exactly at the minimum: side * 0.5^k == 32
  ("side", axis, n)                      the side equals n, an end of the accepted range [16, 2048]
  ("upsample_clamps",)                   the flow upsample into every level below the top takes the left (sx < 0)
                                         and the right (sx + 1 >= SW) clamp
  ("sample", where)                      some UpdateMatrices sample has x1 == -1, y1 == -1, x1 == w-2, y1 == h-2,
                                         x1 == w-1, y1 == h-1 (where = "x=-1", "y=-1", "x=w-2", ...) or lies more than
                                         one pixel outside (where = "far": x1 < -1, x1 >= w, y1 < -1 or y1 >= h)
  ("det_small",)                         some solve has g11*g22 - g12^2 < 1e-3 (the +1e-3 dominates) while h != 0
  ("det_zero",)                          some solve has g11*g22 - g12^2 == 0 exactly
  ("saturated",)                         every pixel of both images is 0 or 255
  ("same",)                              prev == cur
  ("m_max",)                             max |M| over every UpdateMatrices exceeds that of every flow_scenes scene
  ("one_dim",)                           both images are constant along each row (content varies in y only)
  ("impulse",)                           each image has exactly one nonzero pixel
  ("inverted",)                          cur == 255 - prev (a 4-px checkerboard shifted by half its period)
  ("brightness", d)                      cur == prev + d wherever prev + d <= 255
  ("beyond_reach", dx, dy)               cur is prev's texture translated by (dx, dy), and the flow at the centre
                                         recovers less than half of it
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from orb_slam2_ssd_semantic_b200 import synth

U8 = np.uint8
SAMPLES = tuple(("sample", where) for where in ("x=-1", "y=-1", "x=w-2", "y=h-2", "x=w-1", "y=h-1", "far"))


@dataclass(frozen=True)
class Case:
    name: str
    prev: np.ndarray
    cur: np.ndarray
    edges: tuple


def _u8(a) -> np.ndarray:
    return np.clip(np.rint(a), 0, 255).astype(U8)


def sequence(rows: int, cols: int, n: int, dy: int = 1, dx: int = 2, seed: int = 11) -> np.ndarray:
    """-> n x rows x cols u8: a texture translated by (dx, dy) from each frame to the next.  Every frame is a crop of
    one larger texture, so content enters and leaves through the borders (no wrap-around seam); seeded per-frame noise
    keeps every pixel changing."""
    pad = 2 * (n - 1) * max(abs(dy), abs(dx)) + 2
    big = synth.texture(seed, rows + pad, cols + pad, nrect=max(8, rows * cols // 800), nline=max(4, rows * cols // 1600))
    oy = ox = pad // 2
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for t in range(n):
        f = big[oy - t * dy:oy - t * dy + rows, ox - t * dx:ox - t * dx + cols]
        out.append(_u8(f + rng.normal(0, 1.5, f.shape)))
    return np.stack(out)


def moving(rows: int, cols: int, dy: int = 1, dx: int = 2, seed: int = 11) -> tuple:
    """(prev, cur) of `sequence`: cur(x) == prev(x - (dx, dy)) up to the noise."""
    prev, cur = sequence(rows, cols, 2, dy, dx, seed)
    return prev, cur


def _levels(*sizes):
    return ("levels", tuple(sizes))


def _geometry_cases():
    out = []
    # level 1's area path at every width residue mod 8 (tails 0..3 of the 4-wide loop; 84..87 separate ~3 from ~7)
    for w in range(80, 88):
        out.append(("area_w%d" % w, 120, 2 * w, (_levels((120, 2 * w), (60, w)), ("resize", ("copy", "area")),
                                                ("area_tail", w % 8), ("upsample_clamps",))))
    # one side halves exactly, the other does not: linear at level 1
    linear1 = ("resize", ("copy", "linear"))
    out.append(("parity_98x161", 98, 161, (_levels((98, 161), (49, 80)), linear1, ("halves", "rows"),
                                           ("round", 1, "cols", "down"))))
    out.append(("parity_97x162", 97, 162, (_levels((97, 162), (48, 81)), linear1, ("halves", "cols"),
                                           ("round", 1, "rows", "down"))))
    out.append(("parity_161x98", 161, 98, (_levels((161, 98), (80, 49)), linear1, ("halves", "cols"),
                                           ("round", 1, "rows", "down"))))
    # cvRound's half to even on each side, up and down, at levels 1, 2 and 3
    out.append(("round_99x163", 99, 163, (_levels((99, 163), (50, 82)), ("resize", ("copy", "linear")),
                                          ("round", 1, "rows", "up"), ("round", 1, "cols", "up"))))
    out.append(("round_163x99", 163, 99, (_levels((163, 99), (82, 50)), ("resize", ("copy", "linear")),
                                          ("round", 1, "rows", "up"), ("round", 1, "cols", "up"))))
    out.append(("round_270x206", 270, 206, (_levels((270, 206), (135, 103), (68, 52)),
                                            ("resize", ("copy", "area", "linear")),
                                            ("round", 2, "rows", "up"), ("round", 2, "cols", "up"))))
    out.append(("round_130x134", 130, 134, (_levels((130, 134), (65, 67), (32, 34)),
                                            ("resize", ("copy", "area", "linear")),
                                            ("round", 2, "rows", "down"), ("round", 2, "cols", "up"))))
    out.append(("round_134x130", 134, 130, (_levels((134, 130), (67, 65), (34, 32)),
                                            ("resize", ("copy", "area", "linear")),
                                            ("round", 2, "rows", "up"), ("round", 2, "cols", "down"))))
    out.append(("round_260x268", 260, 268, (_levels((260, 268), (130, 134), (65, 67), (32, 34)),
                                            ("resize", ("copy", "area", "linear", "linear")),
                                            ("round", 3, "rows", "down"), ("round", 3, "cols", "up"))))
    out.append(("round_268x260", 268, 260, (_levels((268, 260), (134, 130), (67, 65), (34, 32)),
                                            ("resize", ("copy", "area", "linear", "linear")),
                                            ("round", 3, "rows", "up"), ("round", 3, "cols", "down"))))
    # every level cut, one pixel short of it and exactly at it, with the rows limiting and with the columns limiting
    cuts = ((63, 200, (63, 200)), (64, 200, (64, 200), (32, 100)),
            (127, 200, (127, 200), (64, 100)), (128, 200, (128, 200), (64, 100), (32, 50)),
            (255, 300, (255, 300), (128, 150), (64, 75)), (256, 300, (256, 300), (128, 150), (64, 75), (32, 38)))
    for r, c, *sizes in cuts:
        k = {63: 1, 64: 1, 127: 2, 128: 2, 255: 3, 256: 3}[r]
        edge = "cut_below" if r % 2 else "cut_at"
        out.append(("cut_%dx%d" % (r, c), r, c, (_levels(*sizes), (edge, "rows", k))))
        out.append(("cut_%dx%d" % (c, r), c, r, (_levels(*[(w, h) for h, w in sizes]), (edge, "cols", k))))
    # the accepted range of half-resolution sides
    out.append(("range_16x16", 16, 16, (_levels((16, 16)), ("side", "rows", 16), ("side", "cols", 16))))
    out.append(("range_16x33", 16, 33, (_levels((16, 33)), ("side", "rows", 16))))
    out.append(("range_16x2048", 16, 2048, (_levels((16, 2048)), ("side", "rows", 16), ("side", "cols", 2048))))
    out.append(("range_2048x16", 2048, 16, (_levels((2048, 16)), ("side", "rows", 2048), ("side", "cols", 16))))
    out.append(("range_63x2048", 63, 2048, (_levels((63, 2048)), ("side", "cols", 2048), ("cut_below", "rows", 1))))
    out.append(("range_2048x63", 2048, 63, (_levels((2048, 63)), ("side", "rows", 2048), ("cut_below", "cols", 1))))
    out.append(("range_2048x2048", 2048, 2048, (_levels((2048, 2048), (1024, 1024), (512, 512), (256, 256)),
                                                ("resize", ("copy", "area", "linear", "linear")),
                                                ("side", "rows", 2048), ("side", "cols", 2048), ("upsample_clamps",))))
    return [Case(name, *moving(r, c, seed=100 + i), edges) for i, (name, r, c, edges) in enumerate(out)]


def _checker(rows, cols, cell):
    yy, xx = np.mgrid[0:rows, 0:cols]
    return ((yy // cell + xx // cell) % 2 * 255).astype(U8)


def _content_cases():
    rng = np.random.Generator(np.random.PCG64(2024))
    out = []
    noise = lambda: (rng.integers(0, 2, (256, 256)) * 255).astype(U8)
    a, b = noise(), noise()
    out.append(Case("binary_noise", a, b, (("saturated",), ("m_max",), ("det_small",)) + SAMPLES))
    out.append(Case("binary_noise_same", a, a.copy(), (("saturated",), ("same",))))
    chk = _checker(96, 128, 4)
    out.append(Case("checker_shift1", chk, np.roll(chk, 1, 1), (("saturated",),)))
    out.append(Case("checker_shift4", chk, np.roll(chk, 4, 1), (("saturated",), ("inverted",))))
    imp0 = np.zeros((64, 64), U8)
    imp1 = imp0.copy()
    imp0[32, 32] = 255
    imp1[33, 34] = 255
    out.append(Case("impulse", imp0, imp1, (("impulse",), ("det_zero",))))
    stripes = np.repeat(((np.arange(96) // 3) % 2 * 200 + 20).astype(U8)[:, None], 128, 1)
    out.append(Case("stripes_shift_y", stripes, np.roll(stripes, 1, 0), (("one_dim",), ("det_small",))))
    ramp = np.repeat((np.arange(128) * 2).astype(U8)[None], 64, 0)
    out.append(Case("ramp_shift", ramp, np.roll(ramp, 3, 1), (("det_small",),)))
    out.append(Case("ramp_plus1", ramp, np.minimum(ramp.astype(np.int64) + 1, 255).astype(U8),
                    (("brightness", 1), ("det_small",))))
    out.append(Case("black_to_white", np.zeros((64, 64), U8), np.full((64, 64), 255, U8), (("saturated",),)))
    for dx, dy in ((30, -25), (-60, 0)):
        p, c = moving(160, 200, dy=dy, dx=dx, seed=300 + dx)
        out.append(Case("translate_%d_%d" % (dx, dy), p, c, (("beyond_reach", dx, dy),) + SAMPLES))
    return out


def cases() -> list:
    return _geometry_cases() + _content_cases()

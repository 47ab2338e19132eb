"""Deterministic crafted inputs for the extractor's front half: the pyramid (k_resize / k_resize_g), FAST with its per-cell
NMS and threshold fallback (k_fast_cells) and the 7x7 blur (k_blur7_strip / k_blur7_edges), all in csrc/orbx_kernels.cuh.
Each case names the branch it pins; tests/test_extractor_stages_cpu.py checks on the oracle that it really reaches it, and
tests/test_extractor_stages_gpu.py compares every stage of the device with the oracle on it, bit for bit.

Families:
  fast/*    rings whose only qualifying 9-arc has min |d| exactly t (no corner) and t + 1 (a corner) for all 16 arc starts
            (arcs from 8 on wrap from ring index 15 to 0) and both polarities, at the initial and at the fallback
            threshold; every arc holds a compass pair with one pixel only in the arc, and that pixel sits at exactly
            t + 1.  m = 1 and 2 at t = 0, m = 255 (score 254).
  nms/*     equal-score neighbours in each of the 8 directions (both suppressed) and a neighbour one score lower (the
            centre survives).
  fallback/ a cell holding only a 255/255 pair and a dot of 15: NMS empties it at iniTh 20, the fallback at minTh 7 keeps
            the dot; iniTh == minTh, minTh = 0, and the pair alone.
  cells/*   dots on the first and last detection row and column of every cell (neighbouring cells' dots straddle the
            boundary, one pixel apart, and per-cell NMS keeps both), the clamped last row and column of cells, the 6-px
            ROI overlaps, all byte phases x0 & 3, both FAST tile pitches, and the two dots at (49, 100) and (50, 100).
  blur/*    level sizes with w % 4 in {0..3}, w % 128 leaving the last strip tile 0, 1 or 2 interior groups, h % 35 in
            {0, 1, 6, 7, 8, 34}; 128 impulses on black whose (+-1, +-1) taps are exact rounding ties (4.5 -> 5), at the
            first and last three rows and columns, in interior strips, tail rows and edge groups; all-255; noise.
  resize/*  column and row ramps, 1-px checkers and all-255 at scale 1.2 and at the factors near 2 where the pyramid
            switches from k_resize_g to k_resize."""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field

import numpy as np

from tests.test_boundaries_gpu import _levels_with_cells, _width_with_widest_roi, level_sizes  # noqa: F401

EDGE_THRESHOLD, FAST_BORDER = 19, 16
# FAST's Bresenham circle of radius 3 as (dx, dy), ring index 0..15 (cv::FAST's pixel order, k_fast_cells' v[0..15])
RING = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0),
        (-3, 1), (-2, 2), (-1, 3)]
K7 = np.array([18, 34, 48, 56, 48, 34, 18], np.int64)   # GaussianBlur 7x7 sigma 2, 8-bit fixed point per pass
BLS_ROWS = 35                                           # k_blur7_strip's strip height
DEFAULT = (1000, 1.2, 1, 20, 7)                         # nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST


@dataclass
class Case:
    name: str
    img: np.ndarray
    params: tuple = DEFAULT
    want: list = field(default_factory=list)     # (level, x, y, score) that must be a FAST candidate
    absent: list = field(default_factory=list)   # (level, x, y) that must not be
    cell_counts: dict = field(default_factory=dict)   # (level, x0, y0) of a cell -> its exact candidate count


# ---- geometry (orbx.cu ensure_geometry, in float32 like the C++; level sizes and the tile-pitch and resize-kernel
# choices are test_boundaries_gpu's) -----------------------------------------------------------------------------------
f32 = np.float32


def cells(lh, lw):
    """The FAST cells of one level as (x0, y0, rw, rh), in the order vToDistributeKeys collects them."""
    maxbx, maxby = lw - EDGE_THRESHOLD + 3, lh - EDGE_THRESHOLD + 3
    width, height = f32(maxbx - FAST_BORDER), f32(maxby - FAST_BORDER)
    ncols, nrows = int(width / f32(30)), int(height / f32(30))
    wcell, hcell = int(math.ceil(f32(width / f32(ncols)))), int(math.ceil(f32(height / f32(nrows))))
    out = []
    for i in range(nrows):
        iniy = FAST_BORDER + i * hcell
        if iniy >= maxby - 3:
            continue
        maxy = min(iniy + hcell + 6, maxby)
        for j in range(ncols):
            inix = FAST_BORDER + j * wcell
            if inix >= maxbx - 6:
                continue
            maxx = min(inix + wcell + 6, maxbx)
            out.append((inix, iniy, maxx - inix, maxy - iniy))
    return out


def cell_of(cs, x, y):
    """The cell whose detection range [x0 + 3, x0 + rw - 3) x [y0 + 3, y0 + rh - 3) holds (x, y)."""
    for c in cs:
        x0, y0, rw, rh = c
        if x0 + 3 <= x < x0 + rw - 3 and y0 + 3 <= y < y0 + rh - 3:
            return c
    return None


# ---- numpy restatements used to check that a case reaches its edge ---------------------------------------------------
def fast_m(img, x, y):
    """m(p) = max over the 16 9-arcs of max(min d, min -d), d = ring - centre: a corner at t iff m > t, score m - 1."""
    c = int(img[y, x])
    d = [int(img[y + dy, x + dx]) - c for dx, dy in RING]
    best = 0
    for s in range(16):
        arc = [d[(s + i) % 16] for i in range(9)]
        best = max(best, min(arc), min(-v for v in arc))
    return best


def blur_sum(img):
    """The exact integer 7x7 sum of GaussianBlur's two fixed-point passes with REFLECT_101 padding; the blurred pixel is
    (sum + 32768) >> 16, a rounding tie where sum % 65536 == 32768."""
    p = np.pad(img.astype(np.int64), 3, mode="reflect")   # numpy's "reflect" is REFLECT_101
    h, w = img.shape
    hs = sum(K7[k] * p[:, k:k + w] for k in range(7))
    return sum(K7[k] * hs[k:k + h, :] for k in range(7))


def blur_exact(img):
    return ((blur_sum(img) + 32768) >> 16).astype(np.uint8)


def blur_path(h, w, y, x):
    """Which code writes blurred pixel (y, x): ("edge" | "strip", "full" | "tail")."""
    x0 = x & ~3
    kern = "edge" if (x0 < 4 or x0 + 8 > w) else "strip"
    s0 = (y // BLS_ROWS) * BLS_ROWS
    s1 = min(h, s0 + BLS_ROWS)
    yb = s0 + ((y - s0) // 7) * 7
    return kern, ("tail" if yb + 7 > s1 else "full")


# ---- painters --------------------------------------------------------------------------------------------------------
def paint_arc(img, x, y, start, d, sign, dip=False):
    """A ring around (x, y) whose 9-arc from `start` differs from the centre by exactly sign * d and whose other 7 pixels
    equal it: m = d, the arc's compass pixels at exactly d.  With `dip`, one non-compass pixel of the arc sits at d - 1:
    m = d - 1 while the compass test still sees d."""
    c = int(img[y, x])
    low = (2 if start % 4 == 3 else 1) if dip else -1
    for i in range(9):
        dx, dy = RING[(start + i) % 16]
        img[y + dy, x + dx] = c + sign * (d - (i == low))


# level 0 of 480 x 640: 20 x 14 cells of 37 x 38 px at x0 = 16 + 31 j, y0 = 16 + 32 i (the last column 19 px wide, the
# last row 32 px high); (34 + 31 j, 35 + 32 i) is well inside cell (i, j)'s detection range, x = 614 in the last column's
# [608, 621)
def _centre(n):
    i, j = divmod(n, 20)
    return (34 + 31 * j if j < 19 else 614), 35 + 32 * i


def fast_threshold_case(params, name):
    """16 arc starts x 2 polarities x {corner at iniTh, exactly iniTh, exactly iniTh behind a compass pair at iniTh + 1,
    and the same three at minTh}, one per cell on a flat 100 background (minTh + 1 <= iniTh: the minTh cells are empty at
    iniTh and fall back).  The exactly-iniTh cells also hold a dark dot of m = 60 so that they do not fall back to minTh.
    The compass test passes the pixels of the third kind, so only the exact m > t decides them."""
    _, _, _, ini, mn = params
    assert mn + 1 <= ini < 60
    img = np.full((480, 640), 100, np.uint8)
    case = Case(name, img, params)
    n = 0
    for start in range(16):
        for sign in (1, -1):
            for d, corner, companion, dip in ((ini + 1, True, False, False), (ini, False, True, False), (ini + 1, False, True, True),
                                              (mn + 1, True, False, False), (mn, False, False, False), (mn + 1, False, False, True)):
                x, y = _centre(n)
                n += 1
                paint_arc(img, x, y, start, d, sign, dip)
                if companion:   # in the cell's detection range, away from the ring (the last column is 13 px wide)
                    img[y - 11, x + 5 if x == 614 else x - 11] = 40
                if corner:
                    case.want.append((0, x, y, d - 1))
                else:
                    case.absent.append((0, x, y))
    return case


def low_threshold_case():
    """t = 0: dots of contrast 1 (m = 1: a corner whose score 0 never survives NMS) and 2 (score 1) of both polarities."""
    img = np.full((480, 640), 100, np.uint8)
    case = Case("fast/m1_m2_at_t0", img, (1000, 1.2, 1, 0, 0))
    for n, v in enumerate((101, 99, 102, 98)):
        x, y = _centre(2 * n + 41)
        img[y, x] = v
        if abs(v - 100) == 2:
            case.want.append((0, x, y, 1))
        else:
            case.absent.append((0, x, y))
    return case


def m255_case():
    """White dots on black and black dots on white: m = 255, score 254, the largest the 8-bit packing holds."""
    img = np.zeros((480, 640), np.uint8)
    img[:, 320:] = 255
    case = Case("fast/m255", img, (1000, 1.2, 1, 254, 254))
    for n in range(280):
        x, y = _centre(n)
        if abs(x - 320) < 8 or n % 3:
            continue
        img[y, x] = 0 if x > 320 else 255
        case.want.append((0, x, y, 254))
    return case


DIRS = [(-1, -1), (0, -1), (1, -1), (-1, 0), (1, 0), (-1, 1), (0, 1), (1, 1)]


def nms_case():
    """A bright dot (m = 50) next to another in each of the 8 directions: of equal m both go, one lower keeps the centre."""
    img = np.full((480, 640), 100, np.uint8)
    case = Case("nms/eight_directions", img)
    for n, (dx, dy) in enumerate(DIRS):
        for k, lower in enumerate((False, True)):
            x, y = _centre(2 * (2 * n + k) + 20)
            img[y, x] = 150
            img[y + dy, x + dx] = 149 if lower else 150
            if lower:
                case.want.append((0, x, y, 49))
            else:
                case.absent.append((0, x, y))
            case.absent.append((0, x + dx, y + dy))
    return case


def fallback_cases():
    """Cell 0 of 480 x 640 holds only the 255/255 pair at (25, 25), (26, 25) and a dot of 15 at (40, 40); cell 1 the pair
    alone.  At iniTh 20 NMS removes the pair: the cell is empty after NMS, not before, and the fallback keeps the dot."""
    img = np.zeros((480, 640), np.uint8)
    img[25, 25] = img[25, 26] = 255
    img[40, 40] = 15
    img[25, 56] = img[25, 57] = 255
    c0, c1 = (16, 16), (47, 16)
    out = []
    for params, tag, dot in (((1000, 1.2, 1, 20, 7), "ini20_min7", True), ((1000, 1.2, 1, 20, 20), "ini_eq_min", False),
                             ((1000, 1.2, 1, 20, 0), "min0", True)):
        case = Case("fallback/" + tag, img, params, cell_counts={(0,) + c0: int(dot), (0,) + c1: 0})
        (case.want if dot else case.absent).append((0, 40, 40, 14) if dot else (0, 40, 40))
        case.absent += [(0, 25, 25), (0, 26, 25), (0, 56, 25), (0, 57, 25)]
        out.append(case)
    return out


def edge_dots(rows, cols, nlevels, name):
    """Dots on black at the first and last detection column (same row) and the first and last detection row (same
    column) of every level-0 cell, values varying by cell: neighbouring cells' dots are one pixel apart across the
    boundary."""
    img = np.zeros((rows, cols), np.uint8)
    case = Case(name, img, (1000, 1.2, nlevels, 20, 7))
    cs = cells(rows, cols)
    for n, (x0, y0, rw, rh) in enumerate(cs):
        v = 40 + (n * 37) % 200
        ya = y0 + 3 + (rh - 6) // 3
        xc = x0 + 3 + (rw - 6) // 2
        for k, (x, y) in enumerate(((x0 + 3, ya), (x0 + rw - 4, ya), (xc, y0 + 3), (xc, y0 + rh - 4))):
            img[y, x] = v + k
            case.want.append((0, x, y, v + k - 1))
    return case


def straddle_case():
    img = np.zeros((480, 640), np.uint8)
    img[100, 49] = img[100, 50] = 200
    return Case("cells/straddle_49_50", img, want=[(0, 49, 100, 199), (0, 50, 100, 199)],
                cell_counts={(0, 16, 80): 1, (0, 47, 80): 1})


def pitch_widths():
    """480-row widths whose widest FAST ROI over 8 levels is 45 px (FAST_TP_SMALL, the last it serves) and 46 px
    (FAST_TP_BIG)."""
    return (("small_pitch", _width_with_widest_roi(45)), ("big_pitch", _width_with_widest_roi(46)))


def fast_cases():
    out = [fast_threshold_case(DEFAULT, "fast/arcs_ini20_min7"), fast_threshold_case((1000, 1.2, 1, 40, 1), "fast/arcs_ini40_min1"),
           low_threshold_case(), m255_case(), nms_case()] + fallback_cases()
    out += [straddle_case(), edge_dots(480, 640, 1, "cells/edges_480x640"), edge_dots(480, 640, 8, "cells/edges_480x640_8lv"),
            edge_dots(333, 517, 1, "cells/edges_333x517")]
    for tag, cols in pitch_widths():
        out.append(edge_dots(480, cols, 8, "cells/edges_480x%d_%s" % (cols, tag)))
    return out


# ---- blur ------------------------------------------------------------------------------------------------------------
# (h, w): w % 4 = 0, 1, 2, 3; w % 128 = 0 (last strip tile 0 interior groups), 8 (1), 12 (2), 124, 127; h % 35 = 0, 1, 6,
# 7, 8, 34
BLUR_SIZES = [(70, 128), (71, 129), (76, 130), (77, 131), (78, 252), (104, 255), (139, 264), (105, 268), (141, 256),
              (106, 385)]


def impulses(h, w):
    """128 on black every 8 px from (1, 1), plus the last three rows and columns: each (+-1, +-1) tap of an isolated
    impulse is 128 * 48 * 48 / 65536 = 4.5, a rounding tie."""
    img = np.zeros((h, w), np.uint8)
    ys = sorted(set(range(1, h - 1, 8)) | {0, 2, h - 3, h - 1})
    xs = sorted(set(range(1, w - 1, 8)) | {0, 2, w - 3, w - 1})
    img[np.ix_(range(1, h - 1, 8), range(1, w - 1, 8))] = 128
    img[np.ix_(ys[:3] + ys[-3:], [w // 2])] = 128
    img[np.ix_([h // 2], xs[:3] + xs[-3:])] = 128
    img[h - 2, 1:w - 1:8] = 128
    img[1:h - 1:8, w - 2] = 128
    return img


def blur_cases():
    rng = np.random.default_rng(7)
    out = []
    for h, w in BLUR_SIZES:
        out.append(Case("blur/impulses_%dx%d" % (h, w), impulses(h, w)))
        out.append(Case("blur/full255_%dx%d" % (h, w), np.full((h, w), 255, np.uint8)))
        out.append(Case("blur/noise_%dx%d" % (h, w), rng.integers(0, 256, (h, w), dtype=np.uint8)))
    out.append(Case("blur/impulses_480x640_8lv", impulses(480, 640), (1000, 1.2, 8, 20, 7)))
    out.append(Case("blur/noise_480x640_8lv", rng.integers(0, 256, (480, 640), dtype=np.uint8), (1000, 1.2, 8, 20, 7)))
    return out


# ---- resize ----------------------------------------------------------------------------------------------------------
RESIZE_SCALES = [1.2, 1.99, 2.0, 2.01, 2.2, 2.34]


def resize_images(h=480, w=640):
    y, x = np.mgrid[0:h, 0:w]
    return {"colramp": ((x * 37) & 255).astype(np.uint8), "rowramp": ((y * 53) & 255).astype(np.uint8),
            "checker1": (((x + y) & 1) * 255).astype(np.uint8), "full255": np.full((h, w), 255, np.uint8)}


def resize_cases():
    out = []
    for s in RESIZE_SCALES:
        for tag, img in resize_images().items():
            out.append(Case("resize/%s_%s" % (tag, s), img, (1000, s, _levels_with_cells(s), 20, 7)))
    return out


@functools.lru_cache(maxsize=None)
def all_cases():
    return fast_cases() + blur_cases() + resize_cases()

"""Deterministic crafted cases for the dynamic mask (csrc/dynm_plane.cuh, csrc/dynm.cu, csrc/flow.cu) and the masked
batch tracker's upload chunks (csrc/orbs.cu).  Each case is named after the edge it makes observable and lists it in
`edges`; tests/test_dynmask_edges_cpu.py checks on the oracle's intermediate results that the case really reaches it.

Masks are built through the flow, as the product receives them: a step of a piecewise-constant half-resolution flow comes
out of pyrUp as 1/8, 1/2 and 7/8 of its value on consecutive full-resolution pixels, so the value V of each side of a
step, against the threshold, puts a full-resolution edge of the static region (mask 1) at any column or row
(`profile_for`).  Isolated dynamic pixels and 3 x 3 blocks come from one to four half-resolution pixels of a larger V
(`spot_flow`).

Families:
  phase/*      static bands 40, 41, 42 px wide: two erosions by the radius-10 ellipse leave 0, 1, 2 columns; the
               surviving column of the 41-px band at every bit phase 0..31 of a middle word, in the first and last word
  hband/*      the same with horizontal bands (rows of the element outside the image are skipped)
  side/*       static bands 10..42 px wide touching each image side (outside pixels never erode), at W % 32 in {0, 1, 23,
               31}: 20 and 21..30 px against the right side are where the padding bits beyond W decide the result
  zero/*       isolated dynamic pixels and 3 x 3 blocks: bit 31 and bit 0 of adjacent words, first / last rows and
               columns, corners
  narrow/*     W % 32 in {0, 1, 31} with one or two words per row; heights below 11 and below 21; odd gray shapes whose
               last row / column lies beyond the 2h x 2w the flow covers and stays 1
  tie/*        thr equal to a pixel's float32 x*x + y*y and one ulp above, pairs where a fused multiply-add rounds
               differently, thresholds just below / at / above the floor of 40, NaN in either channel
Keypoint-filter cases (`lookup_cases`): truncation at k, k - ulp, k + 0.5 on both sides of mask transitions at every bit
phase, the last row and column, coordinates outside the mask (clamped by the per-stage entry), counts around the
512-keypoint chunks of the in-place compaction with three keep patterns.
Farneback cases (`flow_cases`): the size limits 16 and 2048 (2049 refused), level sizes that are exact .5 ties at levels
2 and 3, translations whose displaced fetches leave every image side, a checkerboard against its inverse."""
from __future__ import annotations

import functools
from fractions import Fraction

import numpy as np

from oracle import dynmask_py as O

f32 = np.float32
THR = 100.0
# V of a step side, and where its edge lands at THR = 100 (first static / first dynamic pixel relative to the step):
# 100: 1/8 V is already dynamic; 40: 1/8 static, 1/2 dynamic; 16: 1/2 static, 7/8 dynamic; 11: 7/8 static, V dynamic
STEP_V = (100.0, 40.0, 16.0, 11.0)


def up(x, n=1):
    for _ in range(n):
        x = np.nextafter(f32(x), f32(np.inf))
    return f32(x)


def down(x, n=1):
    for _ in range(n):
        x = np.nextafter(f32(x), f32(-np.inf))
    return f32(x)


def threshold_mask(flow, thr, shape):
    """Flow.cc:24-41 as the oracle computes it, before the morphology: pixels beyond 2h x 2w stay 1."""
    f2 = O.pyr_up(flow)
    m = np.ones(shape, np.uint8)
    m[:f2.shape[0], :f2.shape[1]] = O.flow_mask(f2, thr)
    return m


def stages(flow, thr, shape):
    """-> (threshold mask, after one erosion, after two erosions, final mask) of the oracle."""
    el = O.ellipse(21)
    m0 = threshold_mask(flow, thr, shape)
    e1 = O.morph(m0, el, True)
    e2 = O.morph(e1, el, True)
    return m0, e1, e2, O.morph(e2, el, False)


class MaskCase:
    def __init__(self, name, flow, thr, shape, edges):
        self.name, self.flow, self.thr, self.shape, self.edges = name, np.ascontiguousarray(flow, f32), float(thr), \
            tuple(shape), edges

    def __repr__(self):
        return self.name


# --------------------------------------------------------------------------------------------------------------------
# 1-D step profiles

def _profile_mask(p, n_full):
    """The threshold mask along one axis of a flow that varies along that axis only (value p[x] in channel 0)."""
    fl = np.zeros((2, len(p), 2), f32)
    fl[:, :, 0] = p
    return O.flow_mask(O.pyr_up(fl), THR)[0, :n_full]


def _runs(static):
    """-> [(start, end)] of the maximal runs of 0 (dynamic) in a 0/1 vector."""
    out, x, n = [], 0, len(static)
    while x < n:
        if static[x]:
            x += 1
            continue
        s = x
        while x < n and not static[x]:
            x += 1
        out.append((s, x))
    return out


def profile_for(static, n):
    """A half-resolution profile (n values) whose threshold mask at THR along the 2n covered pixels is exactly `static`
    (0/1 vector of length 2n).  Each dynamic run gets a V region whose left and right halves may take different values
    of STEP_V, so that each of its two edges lands where asked."""
    static = np.asarray(static, np.uint8)
    assert len(static) == 2 * n
    p = np.zeros(n, f32)
    for s, e in _runs(static):
        best = None
        for vl in STEP_V:
            for vr in STEP_V:
                for b in ((s - 2) // 2, (s - 1) // 2, s // 2, (s + 1) // 2, (s + 2) // 2) if s else (0,):
                    for a in ((e - 1) // 2, e // 2, (e + 1) // 2, (e + 2) // 2, (e + 3) // 2) if e < 2 * n else (n,):
                        if not 0 <= b < a <= n:
                            continue
                        q = p.copy()
                        mid = (a + b + 1) // 2
                        q[b:mid], q[mid:a] = vl, vr
                        got = _profile_mask(q, 2 * n)
                        lo, hi = max(s - 4, 0), min(e + 4, 2 * n)
                        if (got[lo:hi] == static[lo:hi]).all():
                            best = q
                            break
                    if best is not None:
                        break
                if best is not None:
                    break
            if best is not None:
                break
        assert best is not None, ("no step profile", s, e)
        p = best
    assert (_profile_mask(p, 2 * n) == static).all()
    return p


def band_flow(h, w, axis, static):
    """Flow h x w x 2 whose threshold mask is `static` (0/1 over 2w columns for axis 1, 2h rows for axis 0) on every row
    (column); the profile rides on channel 1 for vertical variation, channel 0 for horizontal."""
    fl = np.zeros((h, w, 2), f32)
    if axis == 1:
        fl[:, :, 0] = profile_for(static, w)[None, :]
    else:
        fl[:, :, 1] = profile_for(static, h)[:, None]
    return fl


def _interval(n, s, e):
    v = np.zeros(n, np.uint8)
    v[max(s, 0):min(e, n)] = 1
    return v


# --------------------------------------------------------------------------------------------------------------------
# mask families

def _phase_cases():
    out = []
    h, w = 24, 64                   # 48 x 128 mask: four words per row
    W = 2 * w
    for word, phases in ((1, range(32)), (0, range(21, 32)), (3, range(0, 11))):
        for p in phases:
            c = 32 * word + p       # the column the 41-px band leaves
            for width in (40, 41, 42):
                s = c - 20
                if s + width > W - 1:   # the band must not touch the right side
                    continue
                st = _interval(W, s, s + width)
                survive = list(range(s + 20, s + width - 20))
                out.append(MaskCase("phase/w%d/word%d/bit%02d" % (width, word, p), band_flow(h, w, 1, st), THR, (2 * h, W),
                                    [("band", 1, s, s + width), ("survive", 1, survive)]
                                    + ([("phase", p)] if width == 41 else []) + ([("word", word, 4)] if width == 41 else [])))
    return out


def _hband_cases():
    out = []
    h, w = 40, 24                   # 80 x 48 mask
    H = 2 * h
    for r in (21, 22, 31, 32, 40, 57, 58):
        for width in (40, 41, 42):
            s = r - 20
            if s + width > H - 1:       # the band must not touch the bottom
                continue
            st = _interval(H, s, s + width)
            out.append(MaskCase("hband/w%d/row%d" % (width, r), band_flow(h, w, 0, st), THR, (H, 2 * w),
                                [("band", 0, s, s + width), ("survive", 0, list(range(s + 20, s + width - 20)))]))
    return out


def _side_cases():
    out = []
    widths = (10, 20, 21, 25, 30, 31, 40, 41, 42)
    for W in (96, 97, 95, 87):          # W % 32 = 0, 1, 31, 23; the odd ones have a last column beyond the flow
        w, h = W // 2, 24
        for side in ("left", "right") if W % 2 == 0 else ("right",):   # an odd W's last column is static anyway
            for width in widths:
                if side == "left":
                    st = _interval(2 * w, 0, width)
                    s, e = 0, width
                else:
                    st = _interval(2 * w, W - width, W)
                    s, e = W - width, W
                out.append(MaskCase("side/%s/W%d/w%d" % (side, W, width), band_flow(h, w, 1, st), THR, (2 * h, W),
                                    [("band", 1, s, e), ("side", side), ("wmod", W % 32)]))
    for H in (48, 49):
        h, w = H // 2, 40
        for side in ("top", "bottom") if H % 2 == 0 else ("bottom",):
            for width in widths:
                if side == "top":
                    st, s, e = _interval(2 * h, 0, width), 0, width
                else:
                    st, s, e = _interval(2 * h, H - width, H), H - width, H
                out.append(MaskCase("side/%s/H%d/w%d" % (side, H, width), band_flow(h, w, 0, st), THR, (H, 2 * w),
                                    [("band", 0, s, e), ("side", side)]))
    return out


def spot_flow(h, w, targets, shape):
    """(flow, thr): a zero flow with one small patch of a single V whose threshold mask is 0 exactly on `targets` (a set of
    (Y, X) full-resolution pixels inside the 2h x 2w the flow covers) and 1 everywhere else."""
    ys = sorted({y for y, _ in targets})
    xs = sorted({x for _, x in targets})

    def spans(lo, hi, n):
        c = {(max(a, 0), min(b, n - 1)) for a in ((lo - 1) // 2, lo // 2, (lo + 1) // 2)
             for b in ((hi - 1) // 2, hi // 2, (hi + 1) // 2)}
        return sorted((a, b) for a, b in c if a <= b)

    want = np.ones(shape, np.uint8)
    for y, x in targets:
        want[y, x] = 0
    for ry in spans(ys[0], ys[-1], h):
        for rx in spans(xs[0], xs[-1], w):
            for v in (11.0, 13.0, 16.0, 20.0, 25.0, 30.0, 40.0, 50.0, 60.0, 80.0):
                for thr in (100.0, 120.0, 150.0):
                    fl = np.zeros((h, w, 2), f32)
                    fl[ry[0]:ry[1] + 1, rx[0]:rx[1] + 1, 0] = v
                    if (threshold_mask(fl, thr, shape) == want).all():
                        return fl, thr
    raise AssertionError("no spot flow for %s" % (targets,))


def _zero_cases():
    out = []
    for H, W in ((48, 96), (49, 97)):
        h, w = H // 2, W // 2
        Yl, Xl = 2 * h - 1, 2 * w - 1          # last covered row / column
        spots = {"bit31": [(24, 31)], "bit0": [(24, 32)], "bit31b": [(25, 63)], "bit0b": [(23, 64)],
                 "row0": [(0, 40)], "row0b": [(0, 41)], "rowlast": [(Yl, 50)], "rowlast-b": [(Yl, 51)],
                 "col0": [(20, 0)], "col0b": [(21, 0)], "collast": [(22, Xl)], "collast-b": [(23, Xl)],
                 "corner-tl": [(0, 0)], "corner-tr": [(0, Xl)], "corner-bl": [(Yl, 0)], "corner-br": [(Yl, Xl)]}
        for name, t in list(spots.items()):
            (y, x), = t
            spots["block-" + name] = [(y + dy, x + dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)
                                      if 0 <= y + dy <= Yl and 0 <= x + dx <= Xl]
        for name, t in spots.items():
            fl, thr = spot_flow(h, w, t, (H, W))
            edges = [("zeros", sorted(t))]
            if name.startswith(("bit", "block-bit")):
                edges.append(("bits", sorted({x & 31 for _, x in t})))
            if any(y in (0, Yl) for y, _ in t) and any(x in (0, Xl) for _, x in t):
                edges.append(("corner",))
            out.append(MaskCase("zero/%dx%d/%s" % (H, W, name), fl, thr, (H, W), edges))
    return out


def _random_blocks(seed, h, w, p=0.3, v=40.0):
    rng = np.random.Generator(np.random.PCG64(seed))
    fl = np.zeros((h, w, 2), f32)
    fl[..., 0] = np.where(rng.random((h, w)) < p, f32(v), f32(0))
    return fl


def _narrow_cases():
    out = []
    shapes = [(48, 32), (48, 33), (48, 31), (48, 63), (48, 64), (48, 65), (48, 4), (48, 5),   # W % 32 in {0, 1, 31}
              (4, 64), (5, 65), (10, 33), (11, 31), (11, 64), (20, 64), (21, 63), (4, 4), (5, 5), (10, 10), (20, 20)]
    for i, (H, W) in enumerate(shapes):
        h, w = H // 2, W // 2
        edges = [("words", (W + 31) // 32, W % 32)]
        if H < 21:
            edges.append(("short", H))
        if H % 2 or W % 2:
            edges.append(("beyond", H % 2, W % 2))
        for j, (p, v) in enumerate(((0.3, 40.0), (0.08, 100.0))):
            seed = 1000 + 100 * i + 10 * j
            while not 0 < threshold_mask(_random_blocks(seed, h, w, p, v), THR, (H, W)).mean() < 1:
                seed += 1
            out.append(MaskCase("narrow/%dx%d/blocks%d" % (H, W, j), _random_blocks(seed, h, w, p, v), THR, (H, W),
                                edges + [("mixed",)]))
        if W >= 8:                              # a static column band with a 1-px dynamic gap at a word edge, if any
            c = min(2 * w - 4, 30) & ~1
            st = np.ones(2 * w, np.uint8)
            st[c] = 0
            out.append(MaskCase("narrow/%dx%d/gap%d" % (H, W, c), band_flow(h, w, 1, st), THR, (H, W),
                                edges + [("gap", c), ("mixed",)]))
    return out


def round32(q: Fraction) -> np.float32:
    """The float32 nearest the exact rational q (ties to even)."""
    f = f32(float(q))
    cands = [down(f), f, up(f)]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))
    return f32(best)


def fma32(a, b, c) -> np.float32:
    return round32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def sum32(x, y) -> np.float32:
    return f32(f32(x * x) + f32(y * y))


def _value_band(h, w, values, x0=6, bw=8, gap=8):
    """Zero flow with vertical half-resolution bands x0 + k (bw + gap) .. + bw of constant (x, y) = values[k] -> (flow,
    [(Y, X) of a pixel deep inside band k])."""
    fl = np.zeros((h, w, 2), f32)
    centres = []
    for k, (x, y) in enumerate(values):
        a = x0 + k * (bw + gap)
        fl[2:h - 2, a:a + bw] = (x, y)
        centres.append((h, 2 * a + bw))
    return fl, centres


def produced(fl, yx):
    f2 = O.pyr_up(fl)
    return f2[yx][0], f2[yx][1]


@functools.lru_cache(maxsize=None)
def fma_pairs():
    """(x, y) flow values whose pyrUp'd centre (fx, fy) has fmaf(fx, fx, fy*fy) below and above (and fmaf(fy, fy, fx*fx)
    below and above) the two-rounding sum, with that sum >= 40."""
    rng = np.random.Generator(np.random.PCG64(4242))
    found = {}
    while len(found) < 4:
        x, y = f32(rng.uniform(3.0, 9.0)), f32(rng.uniform(3.0, 9.0))
        fl, (c,) = _value_band(16, 32, [(x, y)])
        fx, fy = produced(fl, c)
        s = sum32(fx, fy)
        if s < 40:
            continue
        for key, v in (("xx_below", fma32(fx, fx, f32(fy * fy))), ("yy_below", fma32(fy, fy, f32(fx * fx)))):
            kk = key if v < s else key.replace("below", "above") if v > s else None
            if kk and kk not in found:
                found[kk] = (x, y)
    return found


def _tie_cases():
    out = []
    h, w = 16, 64
    H, W = 2 * h, 2 * w
    # integer tie: 6*6 + 8*8 = 100
    pairs = [("int", (f32(6), f32(8)))] + sorted(fma_pairs().items())
    for name, (x, y) in pairs:
        fl, (c,) = _value_band(h, w, [(x, y)])
        fx, fy = produced(fl, c)
        t2 = sum32(fx, fy)
        kinds = [("tie", c, "at")]
        if name != "int":
            kinds.append(("fma", c, name))
        out.append(MaskCase("tie/%s/at" % name, fl, t2, (H, W), kinds))
        out.append(MaskCase("tie/%s/ulp" % name, fl, up(t2), (H, W), [("tie", c, "ulp")]))
    # the floor: pixels at 40 - ulp, 40, 40 + ulp (searched near (6, 2)) and 39.61 against thresholds around 40
    vals, k = {}, 1
    while len(vals) < 3 and k < 4096:
        for yy in (f32(2) - f32(k) * f32(2 ** -23), f32(2) + f32(k) * f32(2 ** -22)):
            fl, (c,) = _value_band(h, w, [(f32(6), yy)])
            t = sum32(*produced(fl, c))
            for key, want in (("below", down(40)), ("at", f32(40)), ("above", up(40))):
                if t == want and key not in vals:
                    vals[key] = yy
        k += 1
    assert len(vals) == 3, vals
    values = [(f32(6), vals["below"]), (f32(6), vals["at"]), (f32(6), vals["above"]), (f32(6), f32(1.9))]
    fl, cs = _value_band(h, w, values, x0=3, bw=6, gap=8)
    for tname, thr in (("1", 1.0), ("0", 0.0), ("neg", -5.0), ("40-ulp", down(40)), ("40", 40.0), ("40+ulp", up(40)),
                       ("40+2ulp", up(40, 2))):
        out.append(MaskCase("tie/floor/thr%s" % tname, fl, thr, (H, W), [("floor", cs, float(thr))]))
    # NaN in either channel (and both), next to finite static pixels
    fl = np.zeros((h, w, 2), f32)
    fl[5, 10, 0] = np.nan
    fl[9, 30, 1] = np.nan
    fl[3, 50] = (np.nan, np.nan)
    fl[12, 60, 1] = -np.inf
    out.append(MaskCase("tie/nan", fl, THR, (H, W), [("nan", [(10, 20, 0), (18, 60, 1), (6, 100, 0)])]))
    return out


@functools.lru_cache(maxsize=None)
def mask_cases():
    return _phase_cases() + _hband_cases() + _side_cases() + _zero_cases() + _narrow_cases() + _tie_cases()


# --------------------------------------------------------------------------------------------------------------------
# tracker flows: band edges at word boundaries and the right-side widths the padding bits decide

TRACKER_SHAPES = ((480, 640), (481, 641), (480, 663), (481, 671))   # W % 32 = 0, 1, 23, 31


def tracker_flows(rows, cols):
    """Three frames: zero flow; vertical dynamic bands starting at bit 31 / bit 0 and a static band of 25 px against the
    right side; horizontal bands plus a static band of 20 px against the right side and 25 px against the bottom."""
    h, w = rows // 2, cols // 2
    W, Hc = 2 * w, 2 * h
    st = np.ones(W, np.uint8)
    st[63:96] = 0                        # dynamic from bit 31 of word 1 to bit 31 of word 2
    st[160:161 + 64] = 0                 # from bit 0 of word 5 through bit 0 of word 7
    st[cols - 45:cols - 25] = 0          # static again on the last 25 columns
    f1 = band_flow(h, w, 1, st)
    f2 = np.zeros((h, w, 2), f32)
    sr = np.ones(Hc, np.uint8)
    sr[31:64] = 0
    sr[rows - 60:rows - 25] = 0
    f2[..., 1] = profile_for(sr, h)[:, None]
    sc = np.ones(W, np.uint8)
    sc[cols - 41:cols - 20] = 0
    f2[..., 0] = profile_for(sc[:W], w)[None, :]
    return np.stack([np.zeros((h, w, 2), f32), f1, f2])


# --------------------------------------------------------------------------------------------------------------------
# keypoint lookups

def _kps(xy, tag0=0):
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    xy = np.asarray(xy, f32).reshape(-1, 2)
    n = len(xy)
    k = np.zeros(n, KP_DTYPE)
    k["x"], k["y"] = xy[:, 0], xy[:, 1]
    k["angle"] = np.arange(n, dtype=f32) * f32(0.5)
    k["octave"] = np.arange(n) % 8
    k["response"] = np.arange(n, dtype=f32) + f32(7)
    d = np.random.Generator(np.random.PCG64(n)).integers(0, 256, (n, 32)).astype(np.uint8)
    d[:, :4] = np.arange(tag0, tag0 + n, dtype=np.uint32).view(np.uint8).reshape(n, 4)   # the index, to find it again
    return k, d


class LookupCase:
    def __init__(self, name, mask, kps, desc, edges, clamped=False):
        self.name, self.mask, self.kps, self.desc, self.edges, self.clamped = name, mask, kps, desc, edges, clamped

    def __repr__(self):
        return self.name

    def lookup_kps(self):
        """The keypoints at the pixel the per-stage entry reads (truncated, then clamped into the mask)."""
        k = self.kps.copy()
        rows, cols = self.mask.shape
        k["x"] = np.clip(np.trunc(k["x"].astype(np.float64)), 0, cols - 1).astype(f32)
        k["y"] = np.clip(np.trunc(k["y"].astype(np.float64)), 0, rows - 1).astype(f32)
        return k

    def expected(self):
        """-> (kps, desc) kept, by the oracle's rule on the pixel each keypoint reads."""
        _, dk = O.filter_keypoints(self.mask, self.lookup_kps(), self.desc)
        idx = dk[:, :4].copy().view(np.uint32).ravel()
        return self.kps[idx].copy(), self.desc[idx].copy()


def _transition_case():
    rows, cols = 112, 160                       # five words per row
    m = np.ones((rows, cols), np.uint8)
    xy, edges = [], []
    for p in range(32):
        y = 2 + 3 * p
        x0 = 32 + p                             # 1 -> 0 at bit p of word 1, 0 -> 1 at bit p + 3 (word 1 or 2)
        m[y, x0:x0 + 3] = 0
        for X in (x0, x0 + 3):
            fX = f32(X)
            for x in (fX, down(fX), fX + f32(0.5), fX - f32(0.5), up(fX)):
                for yy in (f32(y), down(f32(y)), f32(y) + f32(0.5), down(f32(y + 1)), f32(y + 1)):
                    xy.append((x, yy))
        edges.append(("phase", p))
    k, d = _kps(xy)
    return LookupCase("lookup/transitions", m, k, d, edges + [("trunc",)])


def _last_row_col_case():
    rows, cols = 96, 130
    m = np.ones((rows, cols), np.uint8)
    m[rows - 1, ::3] = 0
    m[::3, cols - 1] = 0
    xy = [(f32(x) + f32(dx), down(f32(rows))) for x in range(0, cols, 2) for dx in (0.0, 0.5)]
    xy += [(down(f32(cols)), f32(y) + f32(dy)) for y in range(0, rows, 2) for dy in (0.0, 0.75)]
    xy += [(f32(cols - 1), f32(rows - 1)), (down(f32(cols)), down(f32(rows)))]
    k, d = _kps(xy)
    return LookupCase("lookup/last-row-col", m, k, d, [("last",), ("trunc",)])


def _outside_case():
    rows, cols = 64, 96
    m = np.ones((rows, cols), np.uint8)
    m[0, 0] = m[rows - 1, cols - 1] = m[0, 40] = m[30, 0] = m[rows - 1, 50] = m[20, cols - 1] = 0
    xs = (-0.5, -3.7, -1.0, 0.0, 40.2, float(cols), cols + 5.2, float(cols - 1))
    ys = (-0.25, -7.5, 0.0, 20.0, 30.9, float(rows), rows + 2.5, float(rows - 1))
    xy = [(x, y) for x in xs for y in ys]
    k, d = _kps(xy)
    return LookupCase("lookup/outside", m, k, d, [("outside",)], clamped=True)


def _count_cases():
    out = []
    rows, cols = 64, 128
    m = np.ones((rows, cols), np.uint8)
    m[:, 100:110] = 0
    for n in (511, 512, 513, 1024, 1025):
        for pat in ("all-but-first", "alternate", "last-of-chunk"):
            i = np.arange(n)
            keep = {"all-but-first": i > 0, "alternate": i % 2 == 1,
                    "last-of-chunk": (i % 512 == 511) | (i == n - 1)}[pat]
            x = np.where(keep, f32(10.5) + f32(80.0) * (i % 97) / f32(97), f32(100.5) + (i % 9))
            y = f32(0.5) + (i % 63).astype(f32)
            k, d = _kps(np.stack([x, y], 1).astype(f32))
            out.append(LookupCase("lookup/count%d/%s" % (n, pat), m, k, d, [("count", n, pat, int(keep.sum()))]))
    return out


@functools.lru_cache(maxsize=None)
def lookup_cases():
    return [_transition_case(), _last_row_col_case(), _outside_case()] + _count_cases()


# --------------------------------------------------------------------------------------------------------------------
# Farneback

def texture(seed, rows, cols, cell=6):
    """Smooth deterministic u8 texture: random cell values bilinearly interpolated, plus fine noise."""
    rng = np.random.Generator(np.random.PCG64(seed))
    ch, cw = rows // cell + 3, cols // cell + 3
    g = rng.uniform(0, 255, (ch, cw)).astype(f32)
    yy = np.arange(rows, dtype=f32) / f32(cell)
    xx = np.arange(cols, dtype=f32) / f32(cell)
    y0, x0 = yy.astype(int), xx.astype(int)
    fy, fx = (yy - y0)[:, None], (xx - x0)[None, :]
    v = g[y0][:, x0] * (1 - fy) * (1 - fx)
    v += g[y0 + 1][:, x0] * fy * (1 - fx)
    v += g[y0][:, x0 + 1] * (1 - fy) * fx
    v += g[y0 + 1][:, x0 + 1] * fy * fx
    v += rng.normal(0, 3.0, (rows, cols)).astype(f32)
    return np.clip(np.rint(v), 0, 255).astype(np.uint8)


class FlowCase:
    def __init__(self, name, gray, edges, refused=False):
        self.name, self.gray, self.edges, self.refused = name, gray, edges, refused   # gray: 2 x 2h x 2w full resolution

    def __repr__(self):
        return self.name

    @property
    def half(self):
        return self.gray.shape[1] // 2, self.gray.shape[2] // 2

    def pair(self):
        from oracle import farneback_py as FB
        h, w = self.half
        return FB.pyr_down(self.gray[0], h, w), FB.pyr_down(self.gray[1], h, w)


def _shifted(seed, h, w, dy, dx):
    """Two 2h x 2w frames of one texture, the second moved by (dy, dx) pixels (dy / 2, dx / 2 at half resolution)."""
    P = max(abs(dy), abs(dx)) + 4
    big = texture(seed, 2 * h + 2 * P, 2 * w + 2 * P)
    a = big[P:P + 2 * h, P:P + 2 * w]
    b = big[P - dy:P - dy + 2 * h, P - dx:P - dx + 2 * w]
    return np.stack([a, b])


def flow_cases(big=True):
    out = []
    for h, w in ((16, 2048), (2048, 16)) + (((2048, 2048),) if big else ()):
        out.append(FlowCase("fb/size%dx%d" % (h, w), _shifted(31 + h, h, w, 6, -4), [("size", h, w)]))
    for h, w in ((130, 134), (134, 130), (260, 268), (268, 260)):
        out.append(FlowCase("fb/tie%dx%d" % (h, w), _shifted(7 + h + w, h, w, 4, 6), [("tie", h, w)]))
    for dy, dx in ((0, 8), (0, -8), (8, 0), (-8, 0), (-16, 24), (40, -24), (24, 40), (-40, -32)):   # full resolution
        out.append(FlowCase("fb/shift%+d%+d" % (dy, dx), _shifted(500 + dy * 3 + dx, 256, 320, dy, dx), [("shift", dy, dx)]))
    yy, xx = np.mgrid[0:128, 0:192]
    cb = np.where(((yy // 16) + (xx // 16)) % 2 == 0, 0, 255).astype(np.uint8)
    out.append(FlowCase("fb/checkerboard", np.stack([cb, 255 - cb]), [("checker",)]))
    out.append(FlowCase("fb/refused2049x16", np.zeros((2, 4098, 32), np.uint8), [("refused",)], refused=True))
    return out

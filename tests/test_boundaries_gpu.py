"""GPU parity with the CPU oracle on both sides of every host-side capacity and dispatch boundary: the fused LAST matcher's
shared-memory layout, the quad-tree's shared-memory limit, the FAST thresholds, the FAST tile pitch, the pyramid's resize
kernel and the occupancy map's hash table under load.

Each boundary is recomputed here from the formula the host code uses (the helpers below quote the line), and every test
checks which side of it the library actually took, so a moved constant fails the test instead of silently moving it
to the other branch."""
import ctypes as C
import math

import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu


def _align(v, a):
    return (v + a - 1) // a * a


# ---------------------------------------------------------------------------------------------------------------------
# matcher: fused vs unfused SearchByProjection(cur, last)
# ---------------------------------------------------------------------------------------------------------------------
GRID_CELLS = 64 * 48     # ORBM_GRID_COLS x ORBM_GRID_ROWS, include/b200orb.h
LCAP = 64                # orbm_kernels.cuh: candidate-list capacity per query
MF_RING = 64             # orbm_match.cuh: candidate lists in flight in the fused kernel


def mf_smem_bytes(cmax, lmax):
    """orbm_match.cuh mf_smem_bytes: (GRID_CELLS + 1) * 4 + mf_ring_bytes() + cmax * (4+4+4+4+4+32+4+1) + lmax * 20 + 64,
    mf_ring_bytes() = MF_RING * MF_LSTR * 4 + 3 * MF_RING * 4 with MF_LSTR = LCAP + 1."""
    ring = MF_RING * (LCAP + 1) * 4 + 3 * MF_RING * 4
    return (GRID_CELLS + 1) * 4 + ring + cmax * 57 + lmax * 20 + 64


def match_last_fused(cur_stride, last_stride):
    """orbm.cu launch_match_last + match_last_fused: cmax = align_up(cur stride, 16), lmax = last stride;
    fused <=> mf_smem_bytes(cmax, align_up(lmax, 16)) <= 200 * 1024 && cmax <= 4096."""
    cmax = _align(cur_stride, 16)
    return mf_smem_bytes(cmax, _align(last_stride, 16)) <= 200 * 1024 and cmax <= 4096


def _last_true(pred, lo, hi):
    """Largest n in [lo, hi) with pred(n), for pred true at lo, false at hi and monotone in between."""
    assert pred(lo) and not pred(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo


def _last_fused_limit(fixed_cur=None, fixed_last=None):
    """Largest n that still runs fused: n = n_cur = n_last, or the free side of a pair whose other side is fixed."""
    return _last_true(lambda n: match_last_fused(fixed_cur or n, fixed_last or n), 1, 1 << 16)


def _synthetic_pair(n_cur, n_last, seed, crowd=0):
    """Synthetic (FrameView, LastView) in the style of test_projection_last_huge_frame_uses_unfused_path: identity pose,
    every map point is a current keypoint moved by ~2 px at z = 2 m with 3 of its 32 descriptor bytes changed.
    crowd > 0 puts the first `crowd` current keypoints (octave 0, descriptors within 2 bytes of each other) into one
    40 x 40 px square and makes the first map points project into it: windows of many more than LCAP candidates."""
    from orb_slam2_ssd_semantic_b200._abi import FrameView, LastView
    rng = np.random.default_rng(seed)
    x = rng.uniform(5, 635, n_cur).astype(np.float32)
    y = rng.uniform(5, 475, n_cur).astype(np.float32)
    octave = rng.integers(0, 8, n_cur).astype(np.int32)
    desc = rng.integers(0, 256, size=(n_cur, 32), dtype=np.uint8)
    if crowd:
        x[:crowd] = rng.uniform(300, 340, crowd)
        y[:crowd] = rng.uniform(220, 260, crowd)
        octave[:crowd] = 0
        desc[:crowd] = rng.integers(0, 256, size=(1, 32), dtype=np.uint8)
        desc[:crowd, :2] ^= rng.integers(0, 256, size=(crowd, 2), dtype=np.uint8)
    sf = (1.2 ** np.arange(8)).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    cur = FrameView(x, y, octave, rng.uniform(0, 360, n_cur).astype(np.float32), np.full(n_cur, -1, np.float32), desc, T,
                    synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, 0, 640, 0, 480, sf)
    z = 2.0
    sel = rng.integers(0, n_cur, n_last)
    if crowd:
        sel[:min(crowd, n_last) // 2] = np.arange(min(crowd, n_last) // 2)
    u = x[sel] + rng.normal(0, 2, n_last)
    v = y[sel] + rng.normal(0, 2, n_last)
    xw = np.stack([(u - synth.CX) * z / synth.FX, (v - synth.CY) * z / synth.FY, np.full(n_last, z)], 1).astype(np.float32)
    d2 = desc[sel].copy()
    d2[:, :3] ^= rng.integers(0, 256, size=(n_last, 3), dtype=np.uint8)
    last = LastView(xw, np.ones(n_last, np.uint8), octave[sel], rng.uniform(0, 360, n_last).astype(np.float32), d2, T,
                    mp_obs=rng.integers(0, 2, n_last).astype(np.int32))
    return cur, last, (u.astype(np.float32), v.astype(np.float32))


def _check_last_pair(oracle, n_cur, n_last, seed, min_matches, crowd=0):
    """Run one pair through ORBmatcher and the oracle; assert equality and the launch count of the predicted path."""
    from orb_slam2_ssd_semantic_b200 import ORBmatcher
    cur, last, uv = _synthetic_pair(n_cur, n_last, seed, crowd)
    fused = match_last_fused(n_cur, n_last)
    m = ORBmatcher(0.9, True)
    before = m.launch_count()
    n_gpu, gpu = m.SearchByProjection(cur, last, 15.0, False)
    delta = m.launch_count() - before
    assert delta == (1 if fused else 4), "(%d, %d): %d launches, the %s path takes %d" % (
        n_cur, n_last, delta, "fused" if fused else "unfused", 1 if fused else 4)
    n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
    assert n_ref >= min_matches, "test is vacuous: %d matches" % n_ref
    assert n_gpu == n_ref
    bad = np.nonzero(gpu != ref)[0]
    assert bad.size == 0, "(%d, %d): %d entries differ, first %s" % (n_cur, n_last, bad.size, bad[:10])
    return cur, uv


SYM_FUSED = _last_fused_limit()                      # 2272: 77 * 2272 = 174944 <= 175036 B of staging
LOP_CUR_FUSED = _last_fused_limit(fixed_last=16)     # 3056 current keypoints against 16 map points
LOP_LAST_FUSED = _last_fused_limit(fixed_cur=100)    # 8432 map points against 100 current keypoints


@pytest.mark.parametrize("n_cur,n_last", [(SYM_FUSED, SYM_FUSED), (SYM_FUSED + 1, SYM_FUSED + 1),
                                          (LOP_CUR_FUSED, 16), (LOP_CUR_FUSED + 1, 16),
                                          (100, LOP_LAST_FUSED), (100, LOP_LAST_FUSED + 1)])
def test_last_pair_on_both_sides_of_fused_limit(oracle, n_cur, n_last):
    """SearchByProjection(cur, last) at the last size the fused kernel's shared memory takes and the first it does not,
    for a symmetric pair and for lopsided pairs with either side large."""
    _check_last_pair(oracle, n_cur, n_last, seed=n_cur * 7 + n_last, min_matches=min(n_cur, n_last) // 5)


def test_last_crowded_window_in_largest_fused_layout(oracle):
    """A 40 x 40 px square holding 600 near-identical keypoints at the symmetric fused limit: windows far over LCAP
    candidates, so the fused kernel's overflow re-walk runs with the largest shared-memory layout it accepts."""
    n = SYM_FUSED
    assert match_last_fused(n, n)
    cur, (u, v) = _check_last_pair(oracle, n, n, seed=5, min_matches=n // 5, crowd=600)
    # window of a map point of octave 0 at th = 15: |dx| < 15 and |dy| < 15 around its projection (src/Frame.cc
    # GetFeaturesInArea); the crowd's keypoints are octave 0
    r = 15.0
    crowded = [int(((np.abs(cur.x[:600] - u[i]) < r) & (np.abs(cur.y[:600] - v[i]) < r)).sum()) for i in range(300)]
    assert max(crowded) > LCAP and sum(c > LCAP for c in crowded) > 50, max(crowded)


# ---------------------------------------------------------------------------------------------------------------------
# extractor geometry: the host arithmetic of orbx::init / orbx::ensure_geometry, in float32 like the C++
# ---------------------------------------------------------------------------------------------------------------------
EDGE_THRESHOLD, FAST_BORDER, FAST_TP_SMALL = 19, 16, 48
QT_BYTES_PER_ENTRY = 2 * 8 + 2 * 4 + 16 + 16 + 16 + 4 * 4   # orbx_kernels.cuh qt_smem_bytes: 88 B per entry
QT_SMEM_LIMIT = 100 * 1024                                    # orbx.cu:261


def _f32(v):
    return np.float32(v)


def level_features(nfeatures, scale, nlevels):
    """orbx.cu:74-82 (src/ORBextractor.cc:420-434): N_l per level."""
    factor = _f32(1.0 / float(_f32(scale)))
    n_desired = _f32(_f32(nfeatures) * (_f32(1) - factor) / (_f32(1) - _f32(float(factor) ** nlevels)))
    out, total = [], 0
    for _ in range(nlevels - 1):
        out.append(int(np.rint(n_desired)))
        total += out[-1]
        n_desired = _f32(n_desired * factor)
    out.append(max(nfeatures - total, 0))
    return out


def level_sizes(rows, cols, scale, nlevels):
    """orbx.cu:68-73 and :134-136: sf[i] = (float)(sf[i-1] * (double)scale), level size = lrintf(size * (1.0f / sf))."""
    sf = [_f32(1.0)]
    for _ in range(1, nlevels):
        sf.append(_f32(float(sf[-1]) * float(_f32(scale))))
    inv = [_f32(_f32(1.0) / s) for s in sf]
    return [(int(np.rint(_f32(_f32(rows) * i))), int(np.rint(_f32(_f32(cols) * i)))) for i in inv]


def fast_cells(lh, lw):
    """orbx.cu:192-223 (src/ORBextractor.cc:775-815): the (rw, rh) of every FAST cell of one level, None when the level
    has no 30-px cell."""
    maxbx, maxby = lw - EDGE_THRESHOLD + 3, lh - EDGE_THRESHOLD + 3
    width, height = _f32(maxbx - FAST_BORDER), _f32(maxby - FAST_BORDER)
    ncols, nrows = int(width / _f32(30)), int(height / _f32(30))
    if ncols <= 0 or nrows <= 0:
        return None
    wcell, hcell = int(math.ceil(_f32(width / _f32(ncols)))), int(math.ceil(_f32(height / _f32(nrows))))
    cells = []
    for i in range(nrows):
        iniy = float(FAST_BORDER + i * hcell)
        maxy = min(iniy + hcell + 6, float(maxby))
        if iniy >= maxby - 3:
            continue
        for j in range(ncols):
            inix = float(FAST_BORDER + j * wcell)
            maxx = min(inix + wcell + 6, float(maxbx))
            if inix >= maxbx - 6:
                continue
            cells.append((int(maxx) - int(inix), int(maxy) - int(iniy)))
    return cells


def n_ini(lh, lw):
    """orbx.cu:224: nIni = std::round((float)(maxBX - minBX) / (maxBY - minBY))."""
    r = _f32(_f32(lw - EDGE_THRESHOLD + 3 - FAST_BORDER) / _f32(lh - EDGE_THRESHOLD + 3 - FAST_BORDER))
    return int(math.floor(float(r) + 0.5))


def geometry(rows, cols, nfeatures, scale, nlevels):
    """What ensure_geometry decides for one extractor: the widest FAST ROI, the keypoint capacity per frame (cap, :232-258)
    and the quad-tree's entry capacity qt_cap = align_up(max(8, max_l(max(N_l + 3, 4 * nIni) + 1)), 8) (:235, :259);
    None when a level has no FAST cell (:197-200)."""
    sizes = level_sizes(rows, cols, scale, nlevels)
    nf = level_features(nfeatures, scale, nlevels)
    rw_max, cap, qcap = 0, 0, 8
    for (lh, lw), n in zip(sizes, nf):
        cells = fast_cells(lh, lw)
        if cells is None:
            return None
        rw_max = max([rw_max] + [c[0] for c in cells])
        capl = max(n + 3, 4 * n_ini(lh, lw))
        cap += capl
        qcap = max(qcap, capl + 1)
    return dict(rw_max=rw_max, cap=cap, qt_cap=_align(qcap, 8), sizes=sizes)


def qt_fits(rows, cols, nfeatures, scale, nlevels):
    """orbx.cu:259-261: qt_smem_bytes(qt_cap) <= 100 KiB, else the first extract fails."""
    return geometry(rows, cols, nfeatures, scale, nlevels)["qt_cap"] * QT_BYTES_PER_ENTRY <= QT_SMEM_LIMIT


def _resize_table(dn, sn):
    """orbx.cu:153-163: source column of every destination column (cv::resize INTER_LINEAR)."""
    scale = 1.0 / (dn / sn)
    out = []
    for d in range(dn):
        f = float(_f32((d + 0.5) * scale - 0.5))
        i = math.floor(f)
        if i < 0:
            i = 0
        if i >= sn - 1:
            i = sn - 1
        out.append(i)
    return out


def resize_grouped(sizes):
    """orbx.cu:167-181: k_resize_g needs the 4 outputs of every thread within an 8-byte source window."""
    for l in range(1, len(sizes)):
        dn, sn = sizes[l][1], sizes[l - 1][1]
        t = _resize_table(dn, sn)
        for dx0 in range(0, dn, 4):
            sx = [t[min(dx0 + i, dn - 1)] for i in range(4)]
            if any(max(s, sx[0]) - sx[0] + 1 > 7 for s in sx[1:]):
                return False
    return True


def _qt_limit(rows, cols, scale, nlevels):
    return _last_true(lambda n: qt_fits(rows, cols, n, scale, nlevels), 1, 1 << 16)


def _cmp(K, D, K2, D2, tag=""):
    assert len(K) == len(K2), "%s: keypoint count %d vs oracle %d" % (tag, len(K), len(K2))
    for name in K.dtype.names:
        bad = np.nonzero(K[name].view(np.int32) != K2[name].view(np.int32))[0]
        assert bad.size == 0, "%s: field %s differs at %s (gpu %s, oracle %s)" % (
            tag, name, bad[:5], K[name][bad[:5]], K2[name][bad[:5]])
    assert D.shape == D2.shape
    bad = np.nonzero((D != D2).any(axis=1))[0]
    assert bad.size == 0, "%s: %d descriptors differ, first %s" % (tag, bad.size, bad[:5])


def _extract_and_compare(oracle, ex, params, img, tag, levels=False):
    K, D = ex(img)
    R = oracle.RefExtractor(*params)
    K2, D2 = R(img)
    assert (ex.candidates_per_level() == R.candidates_per_level).all(), (tag, ex.candidates_per_level(),
                                                                         R.candidates_per_level)
    _cmp(K, D, K2, D2, tag)
    assert len(K) <= ex.max_keypoints(), (tag, len(K), ex.max_keypoints())
    if levels:
        for l in range(params[2]):
            assert (ex.image_pyramid_level(l) == R.level(l)).all(), "%s: level %d" % (tag, l)
    return K


# ---------------------------------------------------------------------------------------------------------------------
# extractor: the quad-tree's shared-memory limit
# ---------------------------------------------------------------------------------------------------------------------
QT_LIMIT_1 = _qt_limit(480, 640, 1.2, 1)     # 1156: qt_cap = align8(1156 + 4) = 1160, 88 * 1160 = 102080 B
QT_LIMIT_8 = _qt_limit(480, 640, 1.2, 8)     # the largest nfeatures whose level-0 quota is still 1156


@pytest.mark.parametrize("nlevels,nfeatures", [(1, QT_LIMIT_1), (8, QT_LIMIT_8)])
def test_quadtree_at_its_shared_memory_limit(oracle, nlevels, nfeatures):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    assert qt_fits(480, 640, nfeatures, 1.2, nlevels) and not qt_fits(480, 640, nfeatures + 1, 1.2, nlevels)
    assert max(level_features(nfeatures, 1.2, nlevels)) == QT_LIMIT_1
    params = (nfeatures, 1.2, nlevels, 20, 7)
    ex = ORBextractor(*params)
    adv = synth.adversarial_frames()
    images = {"synth_frame": synth.synth_frame(1234, 0), "noise": adv["noise"], "checker1": adv["checker1"]}
    for name, img in images.items():
        K = _extract_and_compare(oracle, ex, params, img, "%s nlevels=%d nfeatures=%d" % (name, nlevels, nfeatures))
        if name == "synth_frame":
            assert (K["octave"] == 0).sum() >= 0.95 * QT_LIMIT_1   # level 0 really filled its quota


@pytest.mark.parametrize("nlevels,nfeatures", [(1, QT_LIMIT_1 + 1), (8, QT_LIMIT_8 + 1)])
def test_quadtree_refuses_one_past_its_limit(nlevels, nfeatures):
    from orb_slam2_ssd_semantic_b200 import B200OrbError, ORBextractor
    assert not qt_fits(480, 640, nfeatures, 1.2, nlevels)
    ex = ORBextractor(nfeatures, 1.2, nlevels, 20, 7)
    with pytest.raises(B200OrbError, match="quad-tree"):
        ex(synth.synth_frame(1234, 0))


# ---------------------------------------------------------------------------------------------------------------------
# extractor: FAST thresholds at their extremes (orbx.cu:456-457: 0 <= minTh <= iniTh <= 254)
# ---------------------------------------------------------------------------------------------------------------------
_TH_PAIRS = [(0, 0), (1, 0), (20, 20), (254, 0), (254, 254)]
_TH_IMAGES = ["zeros", "full", "checker2", "checker1", "noise", "lownoise", "lines", "sparse_blobs", "synth_frame", "dots"]


def _dots():
    """Single pixels of full contrast (white on black left, black on white right) 11 px apart: m(p) = 255, the one
    input that is a corner at threshold 254, with the largest response the 8-bit score packing holds (254)."""
    img = np.zeros((480, 640), np.uint8)
    img[:, 320:] = 255
    img[20:460:11, 20:300:11] = 255
    img[20:460:11, 340:620:11] = 0
    return img


def _th_image(name):
    if name == "synth_frame":
        return synth.synth_frame(1234, 2)
    return _dots() if name == "dots" else synth.adversarial_frames()[name]


@pytest.fixture(scope="module")
def th_extractors():
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    return {th: ORBextractor(1000, 1.2, 8, th[0], th[1]) for th in _TH_PAIRS}


@pytest.mark.parametrize("image", _TH_IMAGES)
@pytest.mark.parametrize("th", _TH_PAIRS, ids=["%d-%d" % t for t in _TH_PAIRS])
def test_fast_threshold_extremes(oracle, th_extractors, th, image):
    K = _extract_and_compare(oracle, th_extractors[th], (1000, 1.2, 8, th[0], th[1]), _th_image(image),
                             "%s th=%s" % (image, th))
    if image == "dots" and th[0] == 254:   # level 0 keeps its threshold-254 corners
        lvl0 = K[K["octave"] == 0]
        assert len(lvl0) > 200 and (lvl0["response"] == 254).all()


def test_fast_threshold_zero_noise_heavy_quadtree(oracle):
    """The densest FAST output (threshold 0 on uniform noise: a corner on most pixels) into a heavily loaded quad-tree."""
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    params = (5000, 1.2, 8, 0, 0)
    img = synth.adversarial_frames()["noise"]
    K = _extract_and_compare(oracle, ORBextractor(*params), params, img, "noise th=0 nfeatures=5000")
    assert len(K) >= 4500


# ---------------------------------------------------------------------------------------------------------------------
# extractor: FAST tile pitch (orbx.cu:248: SMALL when the widest ROI + 3 <= FAST_TP_SMALL) and the resize kernel
# ---------------------------------------------------------------------------------------------------------------------
def _width_with_widest_roi(rw, rows=480, scale=1.2, nlevels=8):
    """Narrowest image width from 320 px on whose widest FAST ROI over all levels is rw (a level of 2 or 3 cells per
    row: rw = ceil(width / nCols) + 6, orbx.cu:201-215)."""
    for cols in range(320, 1400):
        g = geometry(rows, cols, 1000, scale, nlevels)
        if g is not None and g["rw_max"] == rw:
            return cols
    raise AssertionError("no width with a widest FAST ROI of %d px" % rw)


_ROI_SMALL_MAX = FAST_TP_SMALL - 3


@pytest.mark.parametrize("rw", [_ROI_SMALL_MAX, _ROI_SMALL_MAX + 1], ids=["small_pitch", "big_pitch"])
def test_fast_tile_pitch_boundary(oracle, rw):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    cols = _width_with_widest_roi(rw)
    params = (1000, 1.2, 8, 20, 7)
    ex = ORBextractor(*params)
    for t in range(2):
        img = synth.synth_frame(55, t, h=480, w=cols)
        _extract_and_compare(oracle, ex, params, img, "480x%d (widest ROI %d px)" % (cols, rw), levels=t == 0)


_SCALES = [1.99, 2.0, 2.01, 2.2, 2.34]


def _levels_with_cells(scale, rows=480, cols=640):
    n = 1
    while n < 8 and geometry(rows, cols, 1000, scale, n + 1) is not None:
        n += 1
    return n


def test_resize_scales_cover_both_kernels():
    """The scale factors below reach both k_resize_g and k_resize."""
    sides = {resize_grouped(level_sizes(480, 640, s, _levels_with_cells(s))) for s in _SCALES}
    assert sides == {True, False}


@pytest.mark.parametrize("scale", _SCALES)
def test_resize_scale_factors_near_two(oracle, scale):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    nlevels = _levels_with_cells(scale)
    assert nlevels >= 3
    params = (1000, scale, nlevels, 20, 7)
    ex = ORBextractor(*params)
    for t in range(2):
        _extract_and_compare(oracle, ex, params, synth.synth_frame(1234, t), "scale %s" % scale, levels=True)


# ---------------------------------------------------------------------------------------------------------------------
# stream tracker at the fused limit: the stride of a pair is the extractor's capacity, several pairs per launch
# ---------------------------------------------------------------------------------------------------------------------
def _tracker_fused_limit(rows=480, cols=640):
    """orbs.cu:224-230: every pair of a batch has stride cap (orbx.cu:258) on both sides."""
    cap = lambda nf: geometry(rows, cols, nf, 1.2, 8)["cap"]
    return _last_true(lambda nf: match_last_fused(cap(nf), cap(nf)), 1, 1 << 16)


def _track_batch(oracle, nfeatures, F=5):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    ws = synth.WallStream(seed=1234, n=F)
    frames = [ws.frame(t) for t in range(F)]
    gray, depth, T = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), np.stack([f[3] for f in frames])
    st = StreamTracker(nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9)
    before = st.launch_count()
    kps, desc, nkp, c2l, nm = st.track_batch(gray, depth, T)
    launches = st.launch_count() - before
    R = oracle.RefExtractor(nfeatures, 1.2, 8, 20, 7)
    prev = None
    for t in range(F):
        K, D = R(gray[t])
        assert nkp[t] == len(K) and kps[t, :nkp[t]].tobytes() == K.tobytes() and (desc[t, :nkp[t]] == D).all(), t
        if prev is not None:
            cur, last = frame_views(oracle, K, D, depth[t], T[t], prev[0], prev[1], depth[t - 1], T[t - 1],
                                    R.mvScaleFactor, obs=1)
            n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
            assert n_ref > 100
            assert nm[t] == n_ref and (c2l[t, :nkp[t]] == ref).all(), "frame %d" % t
        prev = (K, D)
    return launches


def test_stream_tracker_on_both_sides_of_fused_limit(oracle):
    """nfeatures at the tracker's fused limit and one more: both batches (4 frame pairs per launch) equal the oracle
    frame by frame, and the second takes the 4-launch path where the first takes 1."""
    nf = _tracker_fused_limit()
    fused = _track_batch(oracle, nf)
    unfused = _track_batch(oracle, nf + 1)
    assert unfused - fused == 3, (fused, unfused)


# ---------------------------------------------------------------------------------------------------------------------
# occupancy map: the open-addressing table under load
# ---------------------------------------------------------------------------------------------------------------------
def _hash_slot(keys, mask):
    """ocm.cu hash_slot, the 32-bit path of tables below 2^32 slots (murmur3 block + finaliser), on packed keys."""
    k = np.asarray(keys, np.uint64)
    lo, hi = (k & np.uint64(0xffffffff)).astype(np.uint32), (k >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = lo * np.uint32(0xcc9e2d51)
        h = ((h << np.uint32(15)) | (h >> np.uint32(17))) * np.uint32(0x1b873593)
        h ^= hi * np.uint32(0x85ebca6b)
        h ^= h >> np.uint32(16)
        h *= np.uint32(0x85ebca6b)
        h ^= h >> np.uint32(13)
        h *= np.uint32(0xc2b2ae35)
        h ^= h >> np.uint32(16)
    return (h & np.uint32(mask)).astype(np.int64)


def _occupied_slots(keys, capacity):
    """Slots a linear-probing table holds for this key set.  The set does not depend on the insertion order, so it is
    what the GPU's table holds after any interleaving of its inserts."""
    occ = np.zeros(capacity, bool)
    for s in _hash_slot(keys, capacity - 1):
        while occ[s]:
            s = (s + 1) % capacity
        occ[s] = True
    return occ


def _pack(k):
    k = k.astype(np.uint64)
    return k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))


def _leaves(keys, lo):
    p = _pack(keys)
    o = np.argsort(p)
    return p[o], lo[o]


def _loaded_scene(n):
    """_scene of test_mapping_gpu (relief, invalid pixels, pixels beyond depth_max) with the lower image as ground."""
    ws = synth.WallStream(seed=99, n=n, depth0=2.0)
    yy, xx = np.mgrid[0:480, 0:640]
    out = []
    for t in range(n):
        gray, depth, rgb, T = ws.frame(t * 7)
        depth = (depth + 0.3 * np.sin(xx / 90.0) * np.cos(yy / 70.0)).astype(np.float32)
        depth[100:200, 150:300] = 1.1
        depth[::50, ::60] = 0.0
        depth[300:320, 400:460] = 3.7
        label = np.zeros(depth.shape, np.uint8)
        label[300:, :] = 1
        out.append((depth, rgb, T, label))
    return out


OCC_KEYFRAMES = 4      # 15942 leaves: 97 % of a 16384-slot table
TARGET_LOAD = 0.85


@pytest.fixture(scope="module")
def loaded_scene(oracle):
    scene = _loaded_scene(OCC_KEYFRAMES)
    ref = oracle.RefOccupancy()
    for depth, rgb, T, label in scene:
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
    kr, lr = ref.export_leaves()
    return scene, _leaves(kr, lr)


def _insert_device(pcm, scene):
    import torch
    depth = torch.from_numpy(np.stack([s[0] for s in scene])).cuda()
    rgb = torch.from_numpy(np.stack([s[1] for s in scene])).cuda()
    label = torch.from_numpy(np.stack([s[3] for s in scene])).cuda()
    T = np.stack([s[2] for s in scene]).astype(np.float32)
    pcm.insert_keyframes_device(depth.data_ptr(), rgb.data_ptr(), 480, 640, list(range(len(scene))), T, synth.FX, synth.FY,
                                synth.CX, synth.CY, d_label=label.data_ptr())
    pcm.sync()


def test_map_at_high_load_matches_oracle(loaded_scene):
    """map_capacity = the power of two just above the oracle's leaf count: leaf set, log-odds, query() of every leaf and
    of absent keys whose probe wraps past the last slot, a world-1 merge, and an export one entry short."""
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, _lib
    scene, (pk_r, lo_r) = loaded_scene
    n = len(pk_r)
    cap = 1 << int(n).bit_length()
    assert cap // 2 <= n < cap and n / cap >= TARGET_LOAD, (n, cap)
    pcm = PointCloudMapping(0.05, map_capacity=cap)
    _insert_device(pcm, scene)
    assert pcm.num_leaves() == n and pcm.num_leaves() / cap >= TARGET_LOAD
    kg, lg, _ = pcm.export_leaves()
    pk_g, lo_g = _leaves(kg, lg)
    assert len(pk_g) == n and (pk_g == pk_r).all()
    assert (lo_g.view(np.uint32) == lo_r.view(np.uint32)).all()
    assert (lo_r < 0).sum() > 1000 and (lo_r > 0).sum() > 1000
    # every leaf through the find-only probe
    res = 0.05
    centre = lambda k: ((k.astype(np.float64) - 32768 + 0.5) * res).astype(np.float32)
    for k, v in zip(kg, lg):
        got = pcm.query(centre(k))
        assert got is not None and got == v, (k, v, got)
    # absent keys whose home slot lies in the occupied run that ends at the last slot: the probe wraps to slot 0 and
    # goes on to the first empty slot
    occ = _occupied_slots(pk_r, cap)
    assert occ[-1] and occ[0], "the table's last and first slots must both be taken for a wrapping probe"
    run = cap - 1
    while occ[run - 1]:
        run -= 1
    rng = np.random.default_rng(0)
    cand = rng.integers(0, 1 << 16, size=(1 << 21, 3)).astype(np.uint64)
    cand_p = _pack(cand)
    home = _hash_slot(cand_p, cap - 1)
    absent = cand[(home >= run) & ~np.isin(cand_p, pk_r)][:50]
    assert len(absent) >= 10
    for k in absent:
        assert pcm.query(centre(k)) is None, k
    # closing the epoch of a single rank replays its own summaries on the base values: nothing changes
    pcm.merge()
    pcm.sync()
    kg2, lg2, _ = pcm.export_leaves()
    pk2, lo2 = _leaves(kg2, lg2)
    assert (pk2 == pk_g).all() and (lo2 == lo_g).all()
    # an export buffer one entry short is refused
    L = _lib.lib()
    keys = np.zeros((n, 3), np.uint16)
    lo = np.zeros(n, np.float32)
    got = C.c_int64(0)
    rc = L.ocm_export_leaves(pcm.handle, keys.ctypes.data_as(C.c_void_p), lo.ctypes.data_as(C.c_void_p), None, n - 1,
                             C.byref(got))
    assert rc == -2 and got.value == n   # B200ORB_ECAP


@pytest.mark.parametrize("capacity,slots", [(4096, 4096), (1, 2)])
def test_map_full_is_reported(loaded_scene, capacity, slots):
    """A table smaller than the scene's leaf set fills up: the insert reports "map full", no probe runs forever, the
    table holds exactly its slot count (map_capacity 1 is rounded up to 2 slots), and the handle can be destroyed."""
    from orb_slam2_ssd_semantic_b200 import B200OrbError, PointCloudMapping
    scene, (pk_r, _) = loaded_scene
    assert len(pk_r) > slots
    depth, rgb, T, label = scene[0]
    pcm = PointCloudMapping(0.05, map_capacity=capacity)
    with pytest.raises(B200OrbError, match="map full"):
        pcm.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
    assert pcm.num_leaves() == slots
    del pcm
    pcm = PointCloudMapping(0.05, map_capacity=capacity)
    with pytest.raises(B200OrbError, match="map full"):
        _insert_device(pcm, scene[:2])
    assert pcm.num_leaves() == slots
    pcm.sync()   # the error was reported once and cleared
    del pcm

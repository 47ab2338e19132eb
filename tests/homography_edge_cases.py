"""Crafted point-pair sets for findHomography(RANSAC, 3), each named after the edge of OpenCV 4.13's classic RANSAC path
and LM refinement it reaches.  Where an edge depends on which 4-subset RANSAC draws, the pairs are placed at the indices
of `subset_stream(n)`: cv::RNG((uint64)-1) draws the same index stream for every set of n pairs (a rejected subset
consumes its draws like an accepted one), so the k-th drawn subset is known before the pairs are.

`cases()` -> list of (name, src, dst) float32 [n][2].  tests/test_homography_edges_cpu.py checks that every case reaches
its edge and that the restatement equals cv2 on it; tools/make_homography_edges_golden.py stores cv2's results."""
from __future__ import annotations

import numpy as np

from oracle import homography_py as HP

F32 = np.float32
MILD = np.array([[1.1, 0.05, 3.0], [-0.04, 0.95, 1.0], [0.001, 0.002, 1.0]])


def subset_stream(n: int, k: int):
    """The first k 4-index subsets RANSAC draws for n pairs, in draw order (duplicates redrawn, as getSubset does)."""
    rng = HP.CvRNG()
    out = []
    for _ in range(k):
        idx = []
        for _ in range(4):
            while True:
                v = rng.uniform(0, n)
                if v not in idx:
                    break
            idx.append(v)
        out.append(idx)
    return out


def project(H, P) -> np.ndarray:
    """H applied to the points P in double, rounded to float32."""
    P = np.asarray(P, np.float64)
    p = np.c_[P, np.ones(len(P))] @ np.asarray(H, np.float64).T
    return (p[:, :2] / p[:, 2:]).astype(F32)


def _placed(n: int, quad_src, quad_dst, seed: int, H=MILD, noise: float = 0.3):
    """n pairs related by H with noise, the first drawn subset replaced by the given quad (in draw order)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    src = rng.uniform(0, 8, (n, 2)).astype(F32)
    dst = (project(H, src) + rng.normal(0, noise, (n, 2))).astype(F32)
    sub = subset_stream(n, 1)[0]
    src[sub] = np.asarray(quad_src, F32)
    dst[sub] = np.asarray(quad_dst, F32)
    return src, dst


# ---- haveCollinearPoints ------------------------------------------------------------------------------------------------

# Four points whose last one is collinear with two earlier ones to within FLT_EPSILON of their extent: the float
# differences (OpenCV's Point2f subtraction) and exact double differences disagree on the verdict.
COLL_FLOAT_ONLY = [[3.000901460647583, 1.5512218475341797], [-0.6213148236274719, -2.09590744972229],
                   [4.691318511962891, 6.025803565979004], [3.683513641357422, 4.4851179122924805]]
COLL_DOUBLE_ONLY = [[1.0703248977661133, 1.6041196584701538], [4.5484466552734375, 2.7166965007781982],
                    [0.7134405374526978, 0.6160812973976135], [2.7784013748168945, 1.747158408164978]]

# Two 6-pair sets (numpy default_rng(2), trials 13541 and 16126 of 3 near-collinear sources in [0, 4]^2, 3 generic
# ones, destinations through MILD with 0.5 px noise) where the float and double readings give cv2 different results.
CV_13541 = ([[2.580799102783203, 1.6282769441604614], [3.4939262866973877, 2.218404769897461],
             [4.613880634307861, 3.4919447898864746], [2.564159631729126, 1.2823803424835205],
             [5.908854007720947, 4.679009437561035], [1.6662055253982544, 0.7358803749084473]],
            [[6.355063438415527, 2.369269609451294], [7.464898586273193, 2.5651450157165527],
             [8.6766996383667, 4.794214725494385], [5.930201053619385, 1.524535894393921],
             [10.274507522583008, 5.830172061920166], [5.490209579467773, 1.225832462310791]])
# The second one also depends on Mat::dot's order of summation in the LM's gain ratio (its nu update).
CV_16126 = ([[4.125370502471924, 3.386681318283081], [-1.109547734260559, -1.1397649049758911],
             [6.150687217712402, 5.137899875640869], [0.4645399749279022, 3.130589008331299],
             [3.515886068344116, 2.840095281600952], [2.6655445098876953, 1.251197338104248]],
            [[7.578693389892578, 4.6164703369140625], [1.221490502357483, -0.5304989218711853],
             [10.387617111206055, 5.167238712310791], [3.7234809398651123, 4.329052925109863],
             [6.099270820617676, 3.1471710205078125], [6.795217514038086, 2.718754291534424]])


def _collinearity_cases():
    out = []
    for name, q in (("collinear_float_only", COLL_FLOAT_ONLY), ("collinear_double_only", COLL_DOUBLE_ONLY)):
        out.append((name, *_placed(6, q, project(MILD, q), 11)))
    for name, (s, d) in (("collinear_cv2_13541", CV_13541), ("collinear_cv2_16126_lm_dot", CV_16126)):
        out.append((name, np.array(s, F32), np.array(d, F32)))
    exact = [[2, 9], [1, 1], [3, 3], [5, 5]]                      # last point on the line through points 1 and 2
    out.append(("collinear_exact", *_placed(6, exact, project(MILD, exact), 12)))
    coinc = [[1, 2], [4, 7], [6, 1], [4, 7]]                       # last point equal to point 1
    out.append(("collinear_coincident", *_placed(6, coinc, project(MILD, coinc), 13)))
    e = float(np.spacing(F32(0.0625)))
    near = [[0.0625, 0.125], [0.25, 0.0625], [0.1875, 0.25], [0.0625 + e, 0.125]]   # last point 1 ulp from point 0
    out.append(("collinear_near_coincident", *_placed(6, near, project(MILD, near), 14)))
    horiz = [[1, 6], [2, 3], [5, 3], [7, 3]]
    out.append(("collinear_horizontal", *_placed(6, horiz, project(MILD, horiz), 15)))
    vert = [[1, 6], [4, 1], [4, 5], [4, 7]]
    out.append(("collinear_vertical", *_placed(6, vert, project(MILD, vert), 16)))
    rng = np.random.Generator(np.random.PCG64(17))                  # integer pixels: both readings agree on every draw
    src = rng.integers(0, 640, (12, 2)).astype(F32)
    dst = np.rint(project(np.diag([1.0, 1.0, 1.0]) + np.array([[0, 0, 7], [0, 0, -4], [0, 0, 0]]), src)
                  + rng.integers(-1, 2, (12, 2))).astype(F32)
    out.append(("collinear_integer_agree", src, dst))
    return out


# ---- checkSubset's orientation test -------------------------------------------------------------------------------------

QUAD = [[0, 0], [6, 0], [0, 6], [2, 2]]        # point 3 inside triangle 0 1 2: every triangle positive
ORIENT = {   # destination quads of QUAD by the number of triangles (0 1 2, 1 2 3, 0 2 3, 0 1 3) whose orientation flips
    0: [[1, 1], [8, 1], [1, 8], [3, 3]],
    1: [[1, 1], [8, 1], [1, 8], [3, -1]],      # point 3 across line 0 1
    2: [[1, 1], [8, 1], [1, 8], [-1, -1]],     # point 3 beyond vertex 0: across lines 0 1 and 0 2
    3: [[1, 1], [-6, 1], [1, 8], [-1, -1]],    # mirrored (all four flip), then point 3 back across line 0 1
    4: [[1, 1], [-6, 1], [1, 8], [-1, 3]],     # mirrored in x
}
# Triangle 0 1 2 degenerate in the source (determinant exactly 0) and mirrored elsewhere: the product 0 is not < 0, so 3
# triangles flip and the subset is rejected; unmirrored it is accepted with the same zero.
ZERO_SRC = [[0, 0], [2, 0], [4, 0], [1, 3]]
ZERO_MIRRORED = [[10, 1], [8, 1], [5, 2], [9, 4]]
ZERO_KEPT = [[1, 1], [3, 1], [6, 2], [2, 4]]


def _orientation_cases():
    out = [("orient_%d_flipped" % k, *_placed(6, QUAD, q, 20 + k, H=np.eye(3) + [[0, 0, 1], [0, 0, 1], [0, 0, 0]]))
           for k, q in ORIENT.items()]
    out.append(("orient_zero_det_mirrored", *_placed(6, ZERO_SRC, ZERO_MIRRORED, 26)))
    out.append(("orient_zero_det_kept", *_placed(6, ZERO_SRC, ZERO_KEPT, 27)))
    return out


# ---- getSubset running out of draws ------------------------------------------------------------------------------------


def _exhaustion_cases(n_after: int = 300):
    out = []
    x = np.arange(8, dtype=F32)
    line = np.stack([x * 3 + 1, np.full(8, 5, F32)], 1)           # every subset's last point lies on the line
    out.append(("draws_exhausted_no_model", line, project(MILD, line)))
    # n_after pairs: one first-drawn subset of 4 generic pairs, every other pair at one source point (mapped off the
    # model); later subsets need 3 of the 4 generic pairs, so after the first hypothesis 10000 draws in a row fail
    src = np.full((n_after, 2), 5.0, F32)
    dst = np.full((n_after, 2), 40.0, F32)
    sub = subset_stream(n_after, 1)[0]
    src[sub] = np.array(QUAD, F32) + 1
    dst[sub] = project(MILD, src[sub])
    out.append(("draws_exhausted_after_first_hypothesis", src, dst))
    return out


# ---- the inlier threshold -----------------------------------------------------------------------------------------------

THRESH_PAIR = 9          # index of the pair whose error is exactly 9.0f (and of its mirror, THRESH_PAIR + 1)
ABOVE_PAIR = 11          # index of the pair whose error is the next float above 9.0f


def _threshold_case():
    """An integer translation by (7, -4) of 9 integer points, then: two pairs at one source point displaced by +3 and -3
    in x (error exactly 9.0f: inliers, and their residuals cancel in every Jacobian column, so the refined model stays
    the translation), and one pair displaced by (3, 2^-10) (error 9 + 2^-20, the next float above 9: an outlier)."""
    src = np.array([[2, 3], [10, 1], [4, 9], [12, 12], [7, 5], [1, 11], [9, 7], [14, 2], [5, 14],
                    [8, 10], [8, 10], [3, 6]], F32)
    dst = src + F32([7, -4])
    dst[THRESH_PAIR, 0] += 3
    dst[THRESH_PAIR + 1, 0] -= 3
    dst[ABOVE_PAIR] += F32([3, 2.0 ** -10])
    return [("threshold_exactly_9", src, dst)]


# ---- the hypothesis scan ------------------------------------------------------------------------------------------------


def _scan_cases():
    out = []
    # the first subset (3 collinear sources, destinations off any line) fits a model that keeps exactly 3 pairs: it is
    # not taken (good > max(max_good, 3)); a later hypothesis with 4 is
    out.append(("scan_first_hypothesis_3_inliers",
                *_placed(6, ZERO_SRC, [[10, 10], [6, 3], [1, 5], [5, 1]], 0, noise=4.0)))
    # two groups of 6 pairs under two different homographies: the first hypothesis of each counts 6, and the later
    # one of equal count is not taken
    rng = np.random.Generator(np.random.PCG64(41))
    src = rng.uniform(0, 200, (12, 2)).astype(F32)
    H2 = np.array([[0.9, -0.1, 40.0], [0.12, 1.05, -25.0], [0.0004, -0.0003, 1.0]])
    g2 = np.zeros(12, bool)
    g2[[0, 2, 5, 7, 8, 11]] = True
    dst = np.where(g2[:, None], project(H2, src), project(MILD, src)).astype(F32)
    out.append(("scan_equal_counts_keep_first", src, dst))
    # all pairs are inliers: RANSACUpdateNumIters' denominator is 0 (below DBL_MIN), one iteration runs
    src = np.array([[3, 4], [17, 2], [9, 11], [1, 15], [12, 8], [6, 6], [15, 14], [4, 10]], F32)
    out.append(("scan_all_inliers_one_iteration", src, src + F32([5, 2])))
    # 6 related pairs among 40: the iteration count is clamped to maxIters, all 2000 iterations run
    rng = np.random.Generator(np.random.PCG64(43))
    src = rng.uniform(0, 640, (40, 2)).astype(F32)
    dst = rng.uniform(0, 640, (40, 2)).astype(F32)
    dst[:6] = project(MILD, src[:6])
    out.append(("scan_max_iters_clamp", src, dst))
    return out


# ---- runKernel's degenerate test ---------------------------------------------------------------------------------------


def _degenerate_cases():
    base = np.array([[1, 2], [5, 1], [4, 6], [0, 5]], F32)
    out = []
    s = base.copy()
    s[:, 0] = 3
    out.append(("degenerate_n4_src_x_constant", s, project(MILD, base)))
    s = base.copy()
    s[:, 1] = F32([0, 1e-30, 0, 0])                                 # deviation 1.5e-30: below DBL_EPSILON, not 0
    out.append(("degenerate_n4_src_y_below_dbl_eps", s, project(MILD, base)))
    d = project(MILD, base)
    d[:, 0] = F32([0, 3e-16, 0, 0])                                 # deviation 4.5e-16: above DBL_EPSILON
    out.append(("degenerate_n4_dst_x_above_dbl_eps", base, d))
    return out


# ---- the refinement -----------------------------------------------------------------------------------------------------


def related(seed: int, n: int, n_out: int, noise: float = 0.7, scale: float = 640.0, offset: float = 0.0):
    """n pairs through a random mild homography with noise, the first n_out of a random order replaced by uniform
    outliers; source and destination coordinates in [offset, offset + scale)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    src = rng.uniform(0, scale, (n, 2))
    H = np.eye(3) + rng.normal(0, 0.05, (3, 3))
    H[2, :2] *= 1.0 / scale
    H[:2, 2] *= scale / 10
    p = np.c_[src, np.ones(n)] @ H.T
    dst = p[:, :2] / p[:, 2:] + rng.normal(0, noise, (n, 2))
    out = rng.permutation(n)[:n_out]
    dst[out] = rng.uniform(0, scale, (n_out, 2))
    return (src + offset).astype(F32), (dst + offset).astype(F32)


def _refinement_cases():
    out = []
    src = np.array([[3, 4], [17, 2], [9, 11], [1, 15], [12, 8], [6, 6]], F32)
    out.append(("refine_zero_residuals", src, src.copy()))     # the identity: residuals 0 or below FLT_EPSILON
    out.append(("refine_coords_1e4_1e5", *related(51, 30, 6, noise=2.0, scale=9e4, offset=1e4)))
    out.append(("refine_negative_coords", *related(52, 30, 6, scale=640.0, offset=-900.0)))
    # pairs near the threshold: 19 RANSAC inliers, 17 under the refined model
    out.append(("refine_mask_differs_from_ransac", *related(0, 40, 10, noise=2.2)))
    return out


# ---- pair counts --------------------------------------------------------------------------------------------------------

LEVEL_SCALES = [F32(1.0)]
for _ in range(7):
    LEVEL_SCALES.append(F32(LEVEL_SCALES[-1] * F32(1.2)))


def _count_cases():
    out = [("count_n4", *related(61, 4, 0)), ("count_n5", *related(62, 5, 0))]
    for n, n_out in ((50, 1), (50, 0), (51, 2), (51, 1), (99, 50), (99, 20), (100, 51), (100, 30)):
        out.append(("count_n%d_out%d" % (n, n_out), *related(1000 + 10 * n + n_out, n, n_out, noise=0.3)))
    # TrackHomo's pairs are keypoint positions: level-0 integers, and level-l integers times 1.2^l rounded to float
    rng = np.random.Generator(np.random.PCG64(71))
    src = rng.integers(0, 640, (60, 2)).astype(np.float64)
    H = np.array([[1.01, 0.004, 6.0], [-0.003, 0.99, -3.0], [2e-5, -1e-5, 1.0]])
    p = np.c_[src, np.ones(60)] @ H.T
    dst = np.rint(p[:, :2] / p[:, 2:])
    dst[:14] = rng.integers(0, 640, (14, 2))
    out.append(("trackhomo_level0_integers", src.astype(F32), dst.astype(F32)))
    lev = rng.integers(0, 8, 60)
    sc = np.array([LEVEL_SCALES[k] for k in lev], F32)
    si = rng.integers(0, 400, (60, 2)).astype(F32)
    s = (si * sc[:, None]).astype(F32)
    p = np.c_[s.astype(np.float64), np.ones(60)] @ H.T
    di = np.rint(p[:, :2] / p[:, 2:] / sc[:, None].astype(np.float64)).astype(F32)
    d = (di * sc[:, None]).astype(F32)
    d[:14] = (rng.integers(0, 400, (14, 2)).astype(F32) * sc[:14, None]).astype(F32)
    out.append(("trackhomo_scaled_levels", s, d))
    return out


def cases():
    """-> list of (name, src, dst)."""
    return (_collinearity_cases() + _orientation_cases() + _exhaustion_cases() + _threshold_case() + _scan_cases()
            + _degenerate_cases() + _refinement_cases() + _count_cases())

"""Point-pair sets for findHomography(RANSAC, 3): perspective-related pairs with noise and a given outlier fraction,
sets of pure noise (every hypothesis weak: all 2000 iterations run), degenerate sets (no model) and a set on one line
(checkSubset rejects every draw: getSubset gives up before the first hypothesis)."""
import numpy as np


def related(seed: int, n: int, outliers: float, noise: float = 0.7):
    rng = np.random.Generator(np.random.PCG64(seed))
    src = rng.uniform(0, 640, (n, 2))
    H = np.eye(3) + rng.normal(0, 0.05, (3, 3))
    H[2, :2] *= 0.001
    p = np.c_[src, np.ones(n)] @ H.T
    dst = p[:, :2] / p[:, 2:] + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < outliers
    dst[out] = rng.uniform(0, 640, (int(out.sum()), 2))
    return src.astype(np.float32), dst.astype(np.float32)


def noise(seed: int, n: int):
    rng = np.random.Generator(np.random.PCG64(seed))
    return rng.uniform(0, 640, (n, 2)).astype(np.float32), rng.uniform(0, 640, (n, 2)).astype(np.float32)


def cases():
    """-> list of (name, src, dst)."""
    out = []
    for n in (4, 5, 8, 20, 51, 200, 2000):
        for k, frac in enumerate((0.0, 0.3, 0.6)):
            s, d = related(1000 * n + k, n, frac)
            out.append(("n%d_out%.1f" % (n, frac), s, d))
    out.append(("noise_40_full_run", *noise(7, 40)))
    same = np.full((6, 2), 7.0, np.float32)
    out.append(("coincident_6", same, same))
    t = np.arange(12, dtype=np.float32)
    line = np.stack([t * 3 + 1, t * 2 + 5], 1).astype(np.float32)
    out.append(("collinear_12", line, line[::-1].copy()))
    return out


def track_homo_pairs():
    """TrackHomo's pair lists (points_current, points_last) from the point-pair SearchByProjection restatement on
    tests/homo_cases.py's random frame pairs of 1000 and 2000 keypoints, and the first 51 and 200 pairs of the first:
    -> list of (name, src, dst)."""
    from oracle import homo_ref
    from tests import homo_cases

    out = []
    for n, seed in ((1000, 1), (2000, 2)):
        case = homo_cases.random_case(n, seed)
        _, _, pl, pc = homo_cases.run_restatement(
            case, lambda cur, last, th, mono: homo_ref.search_by_projection_last_pairs(cur, last, th, mono, 0.9, True))[-1]
        out.append(("track_homo_%d" % n, pc, pl))
        if n == 1000:
            out += [("track_homo_%d_first_%d" % (n, k), pc[:k].copy(), pl[:k].copy()) for k in (51, 200)]
    return out

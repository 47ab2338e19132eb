"""The crafted VoxelGrid cases of tests/voxelgrid_cases.py on the CPU: each case really contains the edge it is named
after (recomputed here in float32 numpy, as the C++ computes it), no case relies on undefined behaviour (every x * inv,
div_b product and cell index stays within int, every dx*dy*dz within long long), and the oracle's refilter
(occ_ref_global_refilter) equals an independent numpy restatement of PCL's VoxelGrid on every round.

The restatement also takes the kernel mutations that the GPU cases must catch -- truncation for floorf, int for float
subtraction, a reciprocal multiply for the centroid division, an unstable order of equal indices, rounding for the
uint8 truncation -- and each is shown here to change the result of a named case.  `>=` for `>` in the overflow test is
not among them: it changes nothing that a float32 map can reach (test_int_max_product_is_unreachable)."""
import numpy as np
import pytest

from oracle import sem_py
from tests import voxelgrid_cases as V

f32 = np.float32
CASES = V.refilter_cases()
BY_NAME = {c.name: c for c in CASES}
SEM = {c[0]: c for c in V.sem_cases()}
# the case that each kernel mutation changes (a floor-for-truncation mutant of k_gcm_index, float subtraction done in
# int, sx * (1.f / fn), an unstable sort, rounded colours)
KILLED_BY = {
    "trunc": "negative_map_floor_not_truncation",
    "int_sub": "float_sub_ties_min_b_small",
    "recip": "one_cell_of_131769_points",
    "unstable": "one_cell_of_131769_points",
    "round_rgb": "single_cell_truncated_colour",
}


def _grid(P, leaf, mut=()):
    """PCL VoxelGrid's bounding box, overflow test, min_b / div_b and linear index of the finite points P, in float32 like
    the C++ -> (d, min_b, div_b, idx); idx is None where the test overflows."""
    inv = V.inv_of(leaf)
    mn, mx = P.min(0), P.max(0)
    d = ((mx - mn) * inv).astype(np.int64) + 1
    prod = int(d[0]) * int(d[1]) * int(d[2])
    if prod > V.INT_MAX or ("ge" in mut and prod >= V.INT_MAX):
        return d, None, None, None
    fl = np.trunc if "trunc" in mut else np.floor
    min_b = fl(mn * inv).astype(np.int64)
    div = fl(mx * inv).astype(np.int64) - min_b + 1
    q = fl(P * inv)
    ijk = q.astype(np.int64) - min_b if "int_sub" in mut else (q - min_b.astype(f32)).astype(np.int64)
    return d, min_b, div, ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * (div[0] * div[1])


def restate(xyz, rgb, leaf, mut=()):
    """-> (xyz, rgb) of the filtered cloud, or None where the index space overflows."""
    fin = np.isfinite(xyz).all(1)
    P, C = xyz[fin], rgb[fin].astype(f32)
    if len(P) == 0:
        return np.zeros((0, 3), f32), np.zeros((0, 3), np.uint8)
    _, _, _, idx = _grid(P, leaf, mut)
    if idx is None:
        return None
    order = np.lexsort((-np.arange(len(idx)), idx)) if "unstable" in mut else np.argsort(idx, kind="stable")
    s = idx[order]
    starts = np.flatnonzero(np.r_[True, s[1:] != s[:-1]])
    ends = np.r_[starts[1:], len(s)]
    ox, oc = np.zeros((len(starts), 3), f32), np.zeros((len(starts), 3), np.uint8)
    for u, (b, e) in enumerate(zip(starts, ends)):
        cell = order[b:e]
        sx = np.cumsum(P[cell], 0, dtype=f32)[-1]            # sequential float sums in sorted order
        sc = np.cumsum(C[cell], 0, dtype=f32)[-1]
        fn = f32(e - b)
        ox[u] = sx * (f32(1) / fn) if "recip" in mut else sx / fn
        oc[u] = (np.rint(sc / fn) if "round_rgb" in mut else sc / fn).astype(np.uint8)
    return ox, oc


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def rounds(oracle):
    """case name -> V.expected_rounds (the oracle's input and output of every refilter round)."""
    return {c.name: V.expected_rounds(oracle, c) for c in CASES}


def test_case_names_are_unique():
    assert len(BY_NAME) == len(CASES) and len(SEM) == len(V.sem_cases())


@pytest.mark.parametrize("name", list(BY_NAME))
def test_oracle_equals_numpy_restatement(rounds, name):
    for r in rounds[name]:
        want = restate(r.xyz, r.rgb, BY_NAME[name].leaf)
        if want is None:
            assert r.overflow
            fin = np.isfinite(r.xyz).all(1)
            assert (_bits(r.out_xyz) == _bits(r.xyz[fin])).all() and (r.out_rgb == r.rgb[fin]).all()
        else:
            assert not r.overflow and len(want[0]) == len(r.out_xyz)
            assert (_bits(want[0]) == _bits(r.out_xyz)).all() and (want[1] == r.out_rgb).all()


@pytest.mark.parametrize("name", list(BY_NAME))
def test_no_undefined_behaviour(rounds, name):
    """x * inv within int for every finite point; dx*dy*dz within long long; where the grid is built, div_b[0]*div_b[1],
    the third multiplier and every index within int."""
    leaf = BY_NAME[name].leaf
    for r in rounds[name]:
        P = r.xyz[np.isfinite(r.xyz).all(1)]
        if len(P) == 0:
            continue
        assert (np.abs(np.floor(P * V.inv_of(leaf)).astype(np.float64)) < 2.0 ** 31).all()
        d, min_b, div, idx = _grid(P, leaf)
        assert (d > 0).all() and float(d[0]) * float(d[1]) * float(d[2]) < 2.0 ** 63
        if idx is not None:
            assert int(div[0]) * int(div[1]) * int(div[2]) - 1 <= V.INT_MAX
            assert idx.min() >= 0 and idx.max() <= V.INT_MAX


def _finite(r):
    return r.xyz[np.isfinite(r.xyz).all(1)]


def test_cell_boundaries(rounds):
    """On every axis, points with x * inv exactly integral and a float neighbour of one of them in the cell below."""
    for leaf in ("0p04", "0p05", "0p03", "1"):
        for sign in ("pos", "neg"):
            c = BY_NAME["cell_boundaries_leaf%s_%s" % (leaf, sign)]
            P = _finite(rounds[c.name][0])
            inv = V.inv_of(c.leaf)
            for k in range(3):
                x = np.unique(P[:, k])
                on = x[f32(x * inv) == np.floor(f32(x * inv))]
                assert len(on) >= 8 and ((on < 0).all() if sign == "neg" else (on > 0).all())
                below = np.array([V.down(v) for v in on], f32)
                assert (np.floor(below * inv) < np.floor(on * inv)).sum() >= 4
    assert float(V.inv_of(f32(0.03))) != 1.0 / float(f32(0.03))          # 0.03's inverse is inexact


def test_negative_coordinates(rounds):
    P = _finite(rounds["negative_map_floor_not_truncation"][0])
    assert (P < 0).all()
    P = _finite(rounds["mixed_sign_min_b_negative"][0])
    _, min_b, _, _ = _grid(P, BY_NAME["mixed_sign_min_b_negative"].leaf)
    q = P * V.inv_of(BY_NAME["mixed_sign_min_b_negative"].leaf)
    assert (min_b < 0).all() and (np.floor(q) != np.trunc(q)).any()
    P = _finite(rounds["signed_zeros_one_cell"][0])
    for k in range(3):
        b = set(_bits(P[:, k]).tolist())
        assert 0 in b and 0x80000000 in b


def test_float_subtraction_merges_cells(rounds):
    """floor(x * inv) - (float)min_b rounds to even and merges two cells that int subtraction keeps apart."""
    for name in ("float_sub_ties_min_b_small", "float_sub_ties_min_b_beyond_2p24", "float_sub_ties_y_leaf0p5"):
        P = _finite(rounds[name][0])
        leaf = BY_NAME[name].leaf
        _, min_b, _, idx = _grid(P, leaf)
        _, _, _, idx_int = _grid(P, leaf, ("int_sub",))
        assert len(np.unique(idx)) < len(np.unique(idx_int))
        assert (np.floor(P * V.inv_of(leaf)) > 2 ** 24).any()
        if name == "float_sub_ties_min_b_beyond_2p24":
            assert (min_b[0] > 2 ** 24)


def test_overflow_boundary(rounds):
    d, _, div, idx = _grid(_finite(rounds["overflow_test_product_int_max_minus_1"][0]), f32(1))
    assert int(np.prod(d)) == V.INT_MAX - 1 and idx is not None and (div == d).all()
    r = rounds["overflow_test_product_2p31"]
    d, _, _, idx = _grid(_finite(r[0]), f32(1))
    assert int(np.prod(d)) == 2 ** 31 and idx is None
    assert [x.overflow for x in r] == [True, True, True] and np.isnan(r[0].xyz).any()
    d, _, div, idx = _grid(_finite(rounds["div_b_exceeds_d_first_and_last_cells"][0]), f32(0.04))
    assert (div > d).all() and idx is not None
    assert [x.overflow for x in rounds["overflow_after_a_clean_round"]] == [False, True, True]


def test_overflow_key_would_wrap_to_no_cell(rounds):
    """In the overflowing grid of overflow_key_wraps_to_no_cell, the index that PCL never forms would, in 32-bit
    arithmetic, equal the all-ones no-cell key for a finite point: the device must not form it either."""
    r = rounds["overflow_key_wraps_to_no_cell"]
    P = _finite(r[0])
    inv = V.inv_of(f32(1))
    d, _, _, idx = _grid(P, f32(1))
    assert idx is None and int(np.prod(d)) == 2 ** 33 and [x.overflow for x in r] == [True, True]
    min_b = np.floor(P.min(0) * inv).astype(np.int64)
    div = np.floor(P.max(0) * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(P * inv) - min_b.astype(f32)).astype(np.int64)
    m2 = (div[0] * div[1]) % 2 ** 32
    key = (ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * m2) % 2 ** 32
    assert (key == 2 ** 32 - 1).any() and len(r[0].out_xyz) == len(P) == 3 and len(r[1].out_xyz) == 4


def test_int_max_product_is_unreachable():
    """INT_MAX is prime, so dx*dy*dz == INT_MAX needs one axis of INT_MAX: (long long)(f) == 2^31 - 2 for a float f,
    and no float lies in [2^31 - 2, 2^31 - 1).  `>` and `>=` in the overflow test agree on every float32 input."""
    n = V.INT_MAX
    assert all(n % p for p in range(2, 46341))
    assert V.down(f32(2.0 ** 31)) == f32(2.0 ** 31 - 128)


def test_cell_index_int_max(rounds):
    """A finite point whose cell index is INT_MAX, the value of the old non-finite marker; in the last case NaN points
    sort right after it."""
    for name in ("cell_index_int_max_leaf1", "cell_index_int_max_leaf0p04", "cell_index_int_max_next_to_nan"):
        r = rounds[name][0]
        _, _, _, idx = _grid(_finite(r), BY_NAME[name].leaf)
        assert idx.max() == V.INT_MAX and not r.overflow and len(r.out_xyz) == len(np.unique(idx)) >= 2
    assert np.isnan(rounds["cell_index_int_max_next_to_nan"][0].xyz).any()


def test_nonfinite_maps(rounds):
    r = rounds["only_nan_gives_no_points"][0]
    assert np.isnan(r.xyz).all(1).all() and len(r.out_xyz) == 0
    r = rounds["only_inf_gives_no_points"][0]
    assert np.isinf(r.xyz).all() and not np.isnan(r.xyz).any() and len(r.out_xyz) == 0
    assert (r.xyz > 0).any() and (r.xyz < 0).any()
    r = rounds["mixed_nonfinite_dropped"][0]
    fin = np.isfinite(r.xyz).all(1)
    assert np.isnan(r.xyz).any() and np.isinf(r.xyz).any() and 0 < fin.sum() < len(fin) and len(r.out_xyz) > 0
    r = rounds["only_nan_then_finite"]
    assert len(r[0].out_xyz) == 0 and len(r[1].out_xyz) > 0


def test_single_point_and_single_cell(rounds):
    r = rounds["single_point"][0]
    assert len(r.xyz) == 1 and (_bits(r.out_xyz) == _bits(r.xyz)).all()
    r = rounds["single_cell_truncated_colour"][0]
    assert len(r.xyz) == 5 and len(r.out_xyz) == 1
    avg = r.rgb.astype(f32).sum(0) / f32(5)
    assert (np.floor(avg) != np.rint(avg)).any()


def test_one_large_cell(rounds):
    """One cell of >= 2^17 points whose x, y sums depend on the order of addition, colour averages just below an integer."""
    r = rounds["one_cell_of_131769_points"][0]
    assert len(r.xyz) >= 2 ** 17 and len(r.out_xyz) == 1 and np.isfinite(r.xyz).all()
    for k in range(2):
        assert np.cumsum(r.xyz[:, k], dtype=f32)[-1] != np.cumsum(r.xyz[::-1, k], dtype=f32)[-1]
    avg = r.rgb.astype(f32).sum(0) / f32(len(r.rgb))
    assert (np.rint(avg) != avg.astype(np.uint8)).sum() >= 2


def test_chained_rounds(rounds):
    r = rounds["chained_three_rounds"]
    assert len(r) == 3 and all(len(x.out_xyz) > 100 for x in r)
    # each later round filters the previous centroids together with new points, some of them in the same cells
    assert all(len(r[i].xyz) == len(r[i - 1].out_xyz) + 24 * 32 for i in (1, 2))


@pytest.mark.parametrize("mut", list(KILLED_BY))
def test_mutation_changes_a_named_case(rounds, mut):
    c = BY_NAME[KILLED_BY[mut]]
    changed = False
    for r in rounds[c.name]:
        got = restate(r.xyz, r.rgb, c.leaf, (mut,))
        changed |= got is None or len(got[0]) != len(r.out_xyz) or (_bits(got[0]) != _bits(r.out_xyz)).any() or \
            (got[1] != r.out_rgb).any()
    assert changed


def test_ge_overflow_mutation_changes_nothing(rounds):
    for c in CASES:
        for r in rounds[c.name]:
            a, b = restate(r.xyz, r.rgb, c.leaf), restate(r.xyz, r.rgb, c.leaf, ("ge",))
            assert (a is None) == (b is None)


# ---- semantic per-box cases: the oracle's band points, SOR inliers and their grid ----

def _inliers(case):
    name, leaf, depth, bgr, T, fx, fy, cx, cy, objs = case
    recs, _, (xyz, _) = sem_py.keyframe(depth, bgr, T, fx, fy, cx, cy, 1, objs, leaf)
    out = []
    for o, rec in zip(objs, recs):
        idx, _ = sem_py.band(depth, o)
        P = xyz[idx]
        if len(P) < 51:
            out.append((rec, None))
            continue
        _, keep = sem_py.sor(P)
        out.append((rec, P[keep]))
    return out


def test_sem_box0_cell_index_int_max():
    (rec, P), = _inliers(SEM["sem_box0_cell_index_int_max"])
    _, _, _, idx = _grid(P, f32(1))
    assert rec.n_band == rec.n_inliers == 56 and rec.n_voxels == 2 and idx.max() == V.INT_MAX


def test_sem_overflow_keeps_negative_zero():
    (rec, P), = _inliers(SEM["sem_overflow_keeps_negative_zero"])
    _, _, _, idx = _grid(P, f32(1e-4))
    assert idx is None and rec.n_voxels == rec.n_inliers > 51
    assert _bits([rec.max_pt[0]])[0] == 0x80000000


def test_sem_tiny_leaf_every_box_overflows():
    boxes = _inliers(SEM["sem_tiny_leaf_every_box_overflows"])
    assert len(boxes) == 3
    for rec, P in boxes:
        assert P is not None and _grid(P, f32(1e-6))[3] is None and rec.n_voxels == rec.n_inliers


def test_sem_plane_on_cell_boundaries():
    case = SEM["sem_plane_on_cell_boundaries"]
    inv = V.inv_of(case[1])
    for rec, P in _inliers(case):
        q = P * inv
        assert (q[:, 2] == np.floor(q[:, 2])).all()                       # the plane's depth on a z boundary
        for k in range(2):
            assert (q[:, k] == np.floor(q[:, k])).mean() > 0.3            # x, y on boundaries
        assert _grid(P, case[1])[3] is not None and rec.n_voxels > 100


@pytest.mark.parametrize("name", list(SEM))
def test_sem_no_undefined_behaviour(name):
    """Every box's grid (where it is built) and the refilter of the whole keyframe stay within int."""
    leaf = SEM[name][1]
    P = sem_py.keyframe(*SEM[name][2:9], 1, SEM[name][9], leaf)[2][0]
    for Q in [P[np.isfinite(P).all(1)]] + [Q for _, Q in _inliers(SEM[name]) if Q is not None]:
        assert (np.abs(np.floor(Q * V.inv_of(leaf)).astype(np.float64)) < 2.0 ** 31).all()
        d, _, div, idx = _grid(Q, leaf)
        assert float(d[0]) * float(d[1]) * float(d[2]) < 2.0 ** 63
        if idx is not None:
            assert int(div[0]) * int(div[1]) * int(div[2]) - 1 <= V.INT_MAX and 0 <= idx.min() and idx.max() <= V.INT_MAX

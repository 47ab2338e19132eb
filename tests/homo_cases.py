"""Cases for the perfect tree's point-pair overload SearchByProjection(cur, last, th, bMono, points_last, points_current)
(perfect/src/ORBmatcher.cc:1727-1880) that TrackHomo calls (perfect/src/Tracking.cc:1331-1399).

Each crafted case makes one property of that overload observable, and `edge(case, result)` asserts it on a result:
  prune_kept        a match the rotation prune removes stays in both point vectors (and leaves nmatches)
  double_claim      two temporal points (Observations() == 0) take the same current keypoint: it is listed twice
  distortion        mvKeys != mvKeysUn: the pairs hold the distorted points
  append            the vectors are not empty on entry: the call appends
  retry_2th         fewer than 20 matches at th, at least 20 at 2*th after TrackHomo's clear (two calls)
  window_*          forward / backward / none / mono level windows pick three different keypoints
  outliers          mvbOutlier entries keep their MapPoint but take no part
  empty_last        a last frame without keypoints
Random frame pairs cover 1,000 and 2,000 features and both sides of the fused / generic dispatch boundary of the
device's (cur, last) search.

A case is (cur FrameView, last LastView, cur_kxy, last_kxy, last_outlier, th list, mono, pre-existing pairs).
`run_restatement` and `run_harness` return the same form: per call (nmatches, cur2last, points_last, points_current)."""
import ctypes as C
import os

import numpy as np

from orb_slam2_ssd_semantic_b200 import synth
from orb_slam2_ssd_semantic_b200._abi import LastView
from tests import match_cases as mc

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libhomoref.so")
SHIM_SO = os.path.join(ROOT, "oracle", "_ref", "libshimperfect.so")

# orbm_match.cuh mf_smem_bytes / orbm.cu match_last_fused (as tests/test_boundaries_gpu.py states them): the largest
# n = n_cur = n_last that the fused kernel takes
_RING = 64 * 65 * 4 + 3 * 64 * 4


def _fused(n):
    c = (n + 15) // 16 * 16
    return (64 * 48 + 1) * 4 + _RING + c * 57 + c * 20 + 64 <= 200 * 1024 and c <= 4096


SYM_FUSED = max(n for n in range(1, 4097) if _fused(n))


class Case:
    def __init__(self, name, cur, last, cur_kxy=None, last_kxy=None, outlier=None, ths=(15.0,), mono=False, pre=None):
        self.name, self.cur, self.last = name, cur, last
        self.cur_kxy = _xy(cur_kxy if cur_kxy is not None else np.stack([cur.x, cur.y], 1))
        self.last_kxy = _xy(last_kxy if last_kxy is not None else _seen_from_last(last))
        self.outlier = np.zeros(last.n, np.uint8) if outlier is None else np.ascontiguousarray(outlier, np.uint8)
        self.ths, self.mono = tuple(float(t) for t in ths), bool(mono)
        self.pre = np.zeros((0, 4), f32) if pre is None else np.ascontiguousarray(pre, f32).reshape(-1, 4)

    def __repr__(self):
        return self.name


def _xy(a):
    return np.ascontiguousarray(a, f32).reshape(-1, 2)


def _seen_from_last(last):
    """Where the last frame (pose = identity in every crafted case) sees its map points: its keypoints."""
    z = np.where(last.xw[:, 2] > 0, last.xw[:, 2], 1).astype(f32)
    return np.stack([last.xw[:, 0] * f32(mc.FX) / z + f32(mc.CX), last.xw[:, 1] * f32(mc.FY) / z + f32(mc.CY)], 1)


def _distort(xy):
    """A radial-plus-tangential pattern with non-zero coefficients: mvKeys (distorted) differs from mvKeysUn everywhere."""
    d = xy - np.array([mc.CX, mc.CY], f32)
    r2 = (d * d).sum(1, keepdims=True)
    return (xy + d * f32(2e-7) * r2 + np.array([0.75, -0.5], f32)).astype(f32)


def _with_outliers(last, outlier):
    """The flat view of a last frame whose outlier entries still hold their MapPoint: valid = has MapPoint && !outlier."""
    valid = last.valid & (1 - outlier)
    return LastView(last.xw, valid, last.octave, last.angle, last.mp_desc, last.Tcw, mp_obs=last.mp_obs)


# ---------------------------------------------------------------------------------------------------------------------
# crafted
# ---------------------------------------------------------------------------------------------------------------------
def _matched_scene(seed, n, angle_of, obs=1, offset=1.0, oct=0):
    """n queries, query q projects to (60 + 45 q mod 540, 60 + 40 (q // 12)) and its own keypoint sits `offset` px to the
    right at distance 10."""
    S = mc.Scene(seed)
    for q in range(n):
        u, v = 60.0 + 45.0 * (q % 12), 60.0 + 40.0 * (q // 12)
        qd = S.base()
        S.kp(u + offset, v, S.cand(qd, 10), oct=oct, angle=100.0 + angle_of(q))
        S.query(u, v, qd, oct=oct, angle=100.0, obs=obs)
    return S


def crafted():
    out = {}
    # 11 matches at rotation 0 and one at 180 degrees: 1 < 0.1 * 11, so ComputeThreeMaxima drops that bin
    S = _matched_scene(101, 12, lambda q: 180.0 if q == 11 else 0.0)
    out["prune_kept"] = Case("prune_kept", S.frame(), S.last())
    # two temporal points (no observations) whose only candidate is the same keypoint: both accept it
    S = mc.Scene(102)
    qd = S.base()
    S.kp(200.0, 200.0, S.cand(qd, 5))
    S.query(201.0, 200.0, S.cand(qd, 7), obs=0)
    S.query(199.0, 200.0, S.cand(qd, 9), obs=0)
    S.query(400.0, 300.0, S.base(), obs=0)   # no candidate in its window
    out["double_claim"] = Case("double_claim", S.frame(), S.last())
    S = _matched_scene(103, 24, lambda q: 0.0)
    cur, last = S.frame(), S.last()
    out["distortion"] = Case("distortion", cur, last, cur_kxy=_distort(np.stack([cur.x, cur.y], 1)),
                             last_kxy=_distort(_seen_from_last(last)))
    pre = np.array([[1.5, 2.5, 3.5, 4.5], [-1.0, 0.0, 639.0, 479.0], [10.25, 20.5, 30.75, 40.0]], f32)
    S = _matched_scene(104, 6, lambda q: 0.0)
    out["append"] = Case("append", S.frame(), S.last(), pre=pre)
    # every keypoint 20 px from its projection at octave 0: outside r = 15, inside r = 30
    S = _matched_scene(105, 25, lambda q: 0.0, offset=20.0)
    out["retry_2th"] = Case("retry_2th", S.frame(), S.last(), ths=(15.0, 30.0))
    # one query at octave 3 (r = 15 * 1.728): octave 0 at distance 5, octave 2 at 10, octave 4 at 20
    for name, tz, mono in (("window_none", 0.0, False), ("window_forward", -0.5, False), ("window_backward", 0.5, False),
                           ("window_mono", -0.5, True)):
        S = mc.Scene(106)
        qd = S.base()
        S.kp(300.0, 200.0, S.cand(qd, 5), oct=0)
        S.kp(302.0, 200.0, S.cand(qd, 10), oct=2)
        S.kp(298.0, 201.0, S.cand(qd, 20), oct=4)
        S.query(300.0, 200.0, qd, oct=3)
        out[name] = Case(name, S.frame(tz=tz), S.last(tz=tz), mono=mono)
    S = _matched_scene(107, 24, lambda q: 0.0)
    outlier = (np.arange(24) % 3 == 1).astype(np.uint8)
    out["outliers"] = Case("outliers", S.frame(), _with_outliers(S.last(), outlier), outlier=outlier)
    S = _matched_scene(108, 4, lambda q: 0.0)
    cur = S.frame()
    empty = LastView(np.zeros((0, 3), f32), np.zeros(0, np.uint8), np.zeros(0, np.int32), np.zeros(0, f32),
                     np.zeros((0, 32), np.uint8), np.eye(4, dtype=f32), mp_obs=np.zeros(0, np.int32))
    out["empty_last"] = Case("empty_last", cur, empty)
    return out


def edge(case, res):
    """Assert that `case` shows the property it is named after, on res = [(nmatches, cur2last, pl, pc) per call]."""
    n, c2l, pl, pc = res[-1]
    npre = len(case.pre)
    acc = len(pl) - npre
    if case.name == "prune_kept":
        assert acc == 12 and n == 11 and (c2l >= 0).sum() == 11
        assert pc[npre + 11].tolist() == case.cur_kxy[11].tolist() and c2l[11] == -1
    elif case.name == "double_claim":
        assert acc == 2 and n == 2 and pc[0].tolist() == pc[1].tolist() and (c2l >= 0).sum() == 1
    elif case.name == "distortion":
        assert acc == 24 and not np.isin(pc[:, 0], case.cur.x).any() and not np.isin(pl[:, 0], _seen_from_last(case.last)[:, 0]).any()
        assert pc.tolist() == case.cur_kxy.tolist() and pl.tolist() == case.last_kxy.tolist()
    elif case.name == "append":
        assert acc == 6 and pl[:3].tolist() == case.pre[:, :2].tolist() and pc[:3].tolist() == case.pre[:, 2:].tolist()
    elif case.name == "retry_2th":
        assert res[0][0] < 20 <= n and len(res[0][2]) == 0 and acc == 25
    elif case.name.startswith("window_"):
        want = {"window_none": 1, "window_forward": 2, "window_backward": 0, "window_mono": 1}[case.name]
        assert acc == 1 and c2l.tolist().index(0) == want
    elif case.name == "outliers":
        assert acc == 16 and n == 16 and (c2l[case.outlier == 1] == -1).all()
    elif case.name == "empty_last":
        assert acc == 0 and n == 0 and (c2l == -1).all()


# ---------------------------------------------------------------------------------------------------------------------
# random frame pairs
# ---------------------------------------------------------------------------------------------------------------------
def random_case(n, seed):
    """n current keypoints and n last keypoints in the style of tests/test_boundaries_gpu.py's synthetic pairs (identity
    pose, map points near their keypoint at z = 2 m, 3 descriptor bytes changed), with a third of the map points temporal
    (no observations), every 17th entry an outlier, distorted keypoints and unrestricted angles (the prune runs)."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(5, 635, n).astype(f32)
    y = rng.uniform(5, 475, n).astype(f32)
    octave = rng.integers(0, 8, n).astype(np.int32)
    desc = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    ang = rng.uniform(0, 360, n).astype(f32)
    T = np.eye(4, dtype=f32)
    cur = mc.FrameView(x, y, octave, ang, np.full(n, -1, f32), desc, T, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF,
                       0, 640, 0, 480, mc.SF)
    sel = rng.integers(0, n, n)
    u = x[sel] + rng.normal(0, 2, n)
    v = y[sel] + rng.normal(0, 2, n)
    z = 2.0
    xw = np.stack([(u - synth.CX) * z / synth.FX, (v - synth.CY) * z / synth.FY, np.full(n, z)], 1).astype(f32)
    d2 = desc[sel].copy()
    d2[:, :3] ^= rng.integers(0, 256, size=(n, 3), dtype=np.uint8)
    lang = (ang[sel] + rng.choice([0.0] * 17 + [60.0, 120.0, 180.0], n)).astype(f32) % f32(360)   # 5 % each: pruned
    obs = rng.integers(0, 3, n).astype(np.int32)
    has_mp = (rng.uniform(size=n) < 0.9).astype(np.uint8)
    outlier = ((np.arange(n) % 17 == 5) & (has_mp == 1)).astype(np.uint8)
    last = LastView(xw, has_mp & (1 - outlier), octave[sel], lang, d2, T, mp_obs=obs)
    last_kxy = _distort(np.stack([u, v], 1).astype(f32))
    return Case("random_%d_%d" % (n, seed), cur, last, cur_kxy=_distort(np.stack([x, y], 1)), last_kxy=last_kxy,
                outlier=outlier)


RANDOM = [(1000, 1), (2000, 2), (SYM_FUSED, 3), (SYM_FUSED + 1, 4)]


def random_cases():
    return {"random_%d_%d" % (n, s): (n, s) for n, s in RANDOM}


# ---------------------------------------------------------------------------------------------------------------------
# runners
# ---------------------------------------------------------------------------------------------------------------------
def pairs_from_accepted(case, acc, pl0, pc0):
    i = np.flatnonzero(acc >= 0)
    return (np.concatenate([pl0, case.last_kxy[i]]).astype(f32), np.concatenate([pc0, case.cur_kxy[acc[i]]]).astype(f32))


def run_restatement(case, search):
    """search(cur, last, th, mono) -> (nmatches, cur2last, last2cur_accepted): the restatement or the device.  The calls
    follow TrackHomo: the vectors start as case.pre and are cleared before every further call."""
    res = []
    pl, pc = case.pre[:, :2], case.pre[:, 2:]
    for k, th in enumerate(case.ths):
        if k:
            pl, pc = np.zeros((0, 2), f32), np.zeros((0, 2), f32)
        n, c2l, acc = search(case.cur, case.last, th, case.mono)
        pl, pc = pairs_from_accepted(case, np.asarray(acc), pl, pc)
        res.append((int(n), np.asarray(c2l, np.int32).copy(), pl, pc))
    return res


def harness(path, prefix):
    L = C.CDLL(path)
    from orb_slam2_ssd_semantic_b200 import _abi
    vp, i, fl = C.c_void_p, C.c_int, C.c_float
    f = getattr(L, prefix + "homo_pairs")
    f.argtypes = [C.POINTER(_abi.OrbmFrame), vp, C.POINTER(_abi.OrbmLast), vp, vp, fl, i, fl, i, vp, vp, C.POINTER(i), vp,
                  C.POINTER(i), i, C.POINTER(i)]
    g = getattr(L, prefix + "homo_sequence")
    g.argtypes = [vp, vp, vp, i, i, i, fl, i, i, i, fl, fl, fl, fl, fl, vp, C.POINTER(_abi.OrbmLast), vp, vp, i, i, vp, vp,
                  C.POINTER(i), vp, C.POINTER(i), C.POINTER(i), vp, C.POINTER(i), C.POINTER(i), i]
    return L


def run_harness(case, L, prefix):
    """The same calls on real perfect-tree Frames and MapPoints (oracle/homo_harness.cpp): the reference's own
    overload in libhomoref.so, the shim's in libshimperfect.so."""
    f = getattr(L, prefix + "homo_pairs")
    res = []
    pre = case.pre
    for k, th in enumerate(case.ths):
        cap = len(pre) + case.last.n + 1
        pl = np.zeros((cap, 2), f32)
        pc = np.zeros((cap, 2), f32)
        npre = 0 if k else len(pre)
        pl[:npre], pc[:npre] = pre[:npre, :2], pre[:npre, 2:]
        nl, nc, nm = C.c_int(npre), C.c_int(npre), C.c_int(0)
        c2l = np.full(max(case.cur.n, 1), -7, np.int32)
        cs, ls = case.cur.struct(), case.last.struct()
        rc = f(C.byref(cs), case.cur_kxy.ctypes.data, C.byref(ls), case.last_kxy.ctypes.data, case.outlier.ctypes.data, th,
               int(case.mono), f32(0.9), 1, c2l.ctypes.data, pl.ctypes.data, C.byref(nl), pc.ctypes.data, C.byref(nc), cap,
               C.byref(nm))
        assert rc == 0 and nl.value == nc.value
        res.append((nm.value, c2l[:case.cur.n].copy(), pl[:nl.value].copy(), pc[:nc.value].copy()))
    return res


def sequence_inputs(seed=1234, shift=0.0):
    """Two frames of synth.WallStream: frame 0 is the last frame (the oracle's keypoints, map points unprojected from
    its depth, one in five temporal, every 11th an outlier), frame 1 the images of the current one, with a dynamic-object
    mask that zeroes a 160 x 120 block, and its true pose moved `shift` metres along x."""
    from oracle import ref
    ws = synth.WallStream(seed=seed, n=2)
    f0, f1 = ws.frame(0), ws.frame(1)
    R = ref.RefExtractor(1000, 1.2, 8, 20, 7)
    k0, d0 = R(f0[0])
    _, _, xw, valid = ref.stereo_unproject(k0, f0[1], f0[3], synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    n = len(k0)
    outlier = ((np.arange(n) % 11 == 3) & (valid == 1)).astype(np.uint8)
    obs = np.where(np.arange(n) % 5 == 0, 0, 2).astype(np.int32)
    last = LastView(xw, valid & (1 - outlier), k0["octave"], k0["angle"], d0, f0[3], mp_obs=obs)
    mask = np.ones(f1[0].shape, np.uint8)
    mask[200:320, 240:400] = 0
    T = np.array(f1[3], f32).copy()
    T[0, 3] += f32(shift)
    return dict(gray=np.ascontiguousarray(f1[0]), depth=np.ascontiguousarray(f1[1], f32), mask=mask, T=T, last=last,
                last_kxy=_xy(np.stack([k0["x"], k0["y"]], 1)), outlier=outlier)


def run_sequence(inp, L, prefix, th=15):
    """TrackHomo, the masked constructor and TrackWithMotionModel's search on real perfect-tree Frames."""
    g = getattr(L, prefix + "homo_sequence")
    cap = 4096
    pl, pc = np.zeros((cap, 2), f32), np.zeros((cap, 2), f32)
    hc, tc = np.full(cap, -7, np.int32), np.full(cap, -7, np.int32)
    npts, hn, hnm, tn, tnm = (C.c_int(0) for _ in range(5))
    rows, cols = inp["gray"].shape
    ls = inp["last"].struct()
    rc = g(inp["gray"].ctypes.data, inp["depth"].ctypes.data, inp["mask"].ctypes.data, rows, cols, 1000, f32(1.2), 8, 20, 7,
           synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, inp["T"].ctypes.data, C.byref(ls), inp["last_kxy"].ctypes.data,
           inp["outlier"].ctypes.data, th, 0, pl.ctypes.data, pc.ctypes.data, C.byref(npts), hc.ctypes.data, C.byref(hn),
           C.byref(hnm), tc.ctypes.data, C.byref(tn), C.byref(tnm), cap)
    assert rc == 0
    k = npts.value
    return (hnm.value, hc[:hn.value].copy(), pl[:k].copy(), pc[:k].copy(), tnm.value, tc[:tn.value].copy())

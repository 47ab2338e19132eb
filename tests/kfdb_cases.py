"""Key-frame database scripts (KeyFrameDatabase, src/KeyFrameDatabase.cc) and the three ways to run them: the
restatement (oracle/kfdb_py.py), the reference's own source or the shim on real KeyFrames (kfdb_run of
oracle/kfdb_harness.cpp in libkfdbsrc.so / libkfdbshim.so, oracle/kfdb.mk), and the device through the Python mirror
(orb_slam2_ssd_semantic_b200.keyframedb).  Every runner returns (candidates per query, members per query).

A scene: keyframes with a BowVector, an mnId and the six database members; covisibility edges (a, b, weight); and a
script of ("add", k), ("erase", k), ("clear",), ("reloc", frame_id, words, weights), ("loop", k, min_score).
GetBestCovisibilityKeyFrames(10) is `neigh[k]`: weight descending, equal weights by higher index first -- the harness
lays the KeyFrames out in index order, so that is the reference's (weight, KeyFrame*) order."""
import ctypes as C
import os
import subprocess

import numpy as np

MEMBERS_DTYPE = np.dtype([("loop_query", "<u8"), ("loop_words", "<i4"), ("loop_score", "<f4"),
                          ("reloc_query", "<u8"), ("reloc_words", "<i4"), ("reloc_score", "<f4")])
CODES = {"add": 0, "erase": 1, "clear": 2, "reloc": 3, "loop": 4}


class Scene:
    def __init__(self, n_words, words, weights, kf_id=None, init=None, edges=(), ops=()):
        self.n_words = n_words
        self.words = [np.asarray(w, np.uint32) for w in words]
        self.weights = [np.asarray(v, np.float64) for v in weights]
        self.n_kf = len(self.words)
        self.kf_id = np.asarray(kf_id if kf_id is not None else np.arange(1, self.n_kf + 1), np.uint64)
        self.init = np.zeros(self.n_kf, MEMBERS_DTYPE) if init is None else np.asarray(init, MEMBERS_DTYPE)
        self.edges = np.asarray(list(edges), np.int32).reshape(-1, 3)
        self.ops = list(ops)
        nb = [dict() for _ in range(self.n_kf)]
        for a, b, w in self.edges:
            nb[a][b] = w
            nb[b][a] = w
        self.neigh = [[j for j, _ in sorted(d.items(), key=lambda t: (-t[1], -t[0]))][:10] for d in nb]
        self.connected = [sorted(d) for d in nb]

    def n_queries(self):
        return sum(op[0] in ("reloc", "loop") for op in self.ops)


def bow(words, rng):
    """An L1-normalised BowVector on the given (distinct) words."""
    w = np.unique(np.asarray(words, np.uint32))
    v = rng.random(len(w)) + 0.05
    return w, v / v.sum()


def dyadic(words):
    """Equal power-of-two weights (1 / 2^k on 2^k words): every L1 score between such vectors is exact."""
    w = np.asarray(words, np.uint32)
    assert len(w) & (len(w) - 1) == 0
    return w, np.full(len(w), 1.0 / len(w))


# ---------------------------------------------------------------------------------------------------------------------
def _crafted(rng):
    S = {}
    R = lambda a, b: list(range(a, b))   # noqa: E731
    # 1. threshold: max 10 (a multiple of 5) -> minCommonWords 8: 8 common words are not scored, 9 are; max 7 -> 5 / 6
    for name, nq, counts in (("threshold_mult5", 10, (10, 8, 9, 4)), ("threshold_not5", 7, (7, 5, 6, 1))):
        kb = [bow(R(0, c) + R(40, 44), rng) for c in counts]
        q = bow(R(0, nq), rng)
        ops = [("add", k) for k in range(len(kb))] + [("reloc", 100, *q), ("loop", 0, 0.0)]
        S[name] = Scene(64, [b[0] for b in kb], [b[1] for b in kb], edges=[(0, 1, 5), (1, 2, 5), (2, 3, 7)], ops=ops)
    # 2. + 3. + 4. identical dyadic BowVectors: every score is exactly 1.0.  Y has neighbours Y1..Y3 (acc 4), Z has Z1, Z2
    # (acc 3 == 0.75f * 4: not retained, strict >); the tie in bestScore keeps the first neighbour; two candidates sharing
    # their best neighbour list it once.
    P = dyadic(R(0, 8))
    words = [P[0]] * 8 + [P[0][:4]]
    weights = [P[1]] * 8 + [np.full(4, 0.25)]
    Y, Y1, Y2, Y3, Z, Z1, Z2, X, W = range(9)
    edges = [(Y, Y1, 9), (Y, Y2, 9), (Y, Y3, 8), (Z, Z1, 9), (Z, Z2, 9), (X, W, 3)]
    S["equal_scores_acc_threshold"] = Scene(64, words, weights, edges=edges,
                                            ops=[("add", k) for k in range(9)] + [("reloc", 7, *P), ("loop", W, 0.5),
                                                                                ("loop", X, 1.0), ("reloc", 8, *P)])
    # 4'. distinct scores: A and B both have K (the best-scoring keyframe) as their best neighbour
    q = bow(R(0, 16), rng)
    kb = [(q[0], q[1])] + [bow(R(0, 14) + [30 + k], rng) for k in range(4)]
    S["shared_best_neighbour"] = Scene(64, [b[0] for b in kb], [b[1] for b in kb],
                                       edges=[(1, 0, 4), (2, 0, 4), (3, 4, 2), (1, 2, 1)],
                                       ops=[("add", k) for k in range(5)] + [("reloc", 9, *q), ("loop", 3, 0.0)])
    # 5. stale mRelocScore: query 1 scores N; query 2 meets N below the threshold, and C's accumulation reads N's old score
    N, Cc = bow(R(0, 5) + R(20, 25), rng), bow(R(0, 10), rng)
    S["reloc_stale_score"] = Scene(64, [N[0], Cc[0]], [N[1], Cc[1]], edges=[(0, 1, 3)],
                                   ops=[("add", 0), ("add", 1), ("reloc", 11, *bow(R(0, 5) + R(20, 25), rng)),
                                        ("reloc", 12, *bow(R(0, 10), rng)), ("reloc", 12, *bow(R(0, 12), rng))])
    # 6. loop: Q is connected to Cn (shares words: excluded, mnLoopWords ends at 1) and Cn is A's neighbour (skipped);
    # B's score is exactly minScore (kept); then a minScore above every score
    P4 = dyadic(R(0, 4))
    Q, Cn, A, B, E = range(5)
    words = [P4[0], P4[0], np.array([0, 1, 2, 3, 50, 51, 52, 53], np.uint32), P4[0], np.array([60], np.uint32)]
    weights = [P4[1], P4[1], np.full(8, 0.125), P4[1], np.ones(1)]
    S["loop_connected_min_score"] = Scene(64, words, weights, edges=[(Q, Cn, 20), (A, Cn, 5), (A, B, 4), (E, Q, 1)],
                                          ops=[("add", k) for k in (Cn, A, B, E)] + [("loop", Q, 1.0), ("loop", Q, 0.25),
                                                                                    ("loop", Q, 1.5), ("add", Q),
                                                                                    ("loop", Cn, 0.0)])
    # 7. erase then add moves a keyframe to the end; add twice counts twice; erase after a double add; clear
    kb = [bow(R(0, 6) + [10 + k], rng) for k in range(4)]
    q = bow(R(0, 6) + [10, 11, 12, 13], rng)
    ops = [("add", 0), ("add", 1), ("add", 2), ("reloc", 20, *q), ("erase", 0), ("add", 0), ("reloc", 21, *q),
           ("add", 1), ("reloc", 22, *q), ("loop", 3, 0.0), ("erase", 1), ("reloc", 23, *q), ("erase", 1), ("erase", 1),
           ("erase", 3), ("reloc", 24, *q), ("clear",), ("reloc", 25, *q), ("add", 3), ("add", 2), ("reloc", 26, *q),
           ("loop", 0, 0.0)]
    S["erase_readd_double_clear"] = Scene(64, [b[0] for b in kb], [b[1] for b in kb], edges=[(0, 1, 2), (2, 3, 2)], ops=ops)
    # 8. empty results: no shared word, every score below minScore, an empty query BowVector, an empty database
    kb = [bow(R(0, 8), rng), bow(R(4, 12), rng)]
    S["empty_results"] = Scene(64, [b[0] for b in kb], [b[1] for b in kb], edges=[(0, 1, 1)],
                               ops=[("reloc", 30, *bow(R(0, 8), rng)), ("add", 0), ("add", 1),
                                    ("reloc", 31, *bow(R(20, 30), rng)), ("loop", 0, 2.0),
                                    ("reloc", 32, np.zeros(0, np.uint32), np.zeros(0)), ("loop", 1, 0.0)])
    # a query id equal to the members' previous one: nobody is reset or appended, the counts keep growing
    kb = [bow(R(0, 8), rng), bow(R(2, 10), rng)]
    init = np.zeros(2, MEMBERS_DTYPE)
    init["reloc_query"] = 40
    init["reloc_words"] = 3
    init["reloc_score"] = 0.5
    init["loop_query"] = 2
    init["loop_words"] = 7
    init["loop_score"] = 0.25
    S["repeated_query_id"] = Scene(64, [b[0] for b in kb], [b[1] for b in kb], init=init, edges=[(0, 1, 1)],
                                   ops=[("add", 0), ("add", 1), ("reloc", 40, *bow(R(0, 10), rng)),
                                        ("reloc", 41, *bow(R(0, 10), rng)), ("loop", 1, 0.0)])
    return S


def crafted():
    return _crafted(np.random.default_rng(7))


def random_scene(n_kf=2000, n_words=100_000, n_ops_q=40, seed=5, min_words=300, max_words=1000, script=None):
    """Case 9: Zipf-like word popularity, neighbouring keyframes along a trajectory share about half their words, the
    covisibility graph is a window along the trajectory with tied weights; queries, adds and erases interleaved."""
    rng = np.random.default_rng(seed)
    cdf = np.cumsum(1.0 / np.arange(1, n_words + 1) ** 0.9)
    cdf /= cdf[-1]
    perm = rng.permutation(n_words).astype(np.uint32)

    def draw(k):
        return np.unique(perm[np.minimum(np.searchsorted(cdf, rng.random(k)), n_words - 1)])

    words, weights = [], []
    prev = draw(600)
    for i in range(n_kf):
        k = int(rng.integers(min_words, max_words + 1))
        keep = prev[rng.random(len(prev)) < 0.5]
        w = np.unique(np.concatenate([keep, draw(k)]))
        if len(w) > max_words:
            w = np.sort(rng.choice(w, max_words, replace=False))
        b = bow(w, rng)
        words.append(b[0])
        weights.append(b[1])
        prev = w
    edges = []
    for i in range(n_kf):
        for d in range(1, 8):
            if i + d < n_kf:
                edges.append((i, i + d, int(rng.integers(15, 19)) - d))   # small range: many equal weights
    init = np.zeros(n_kf, MEMBERS_DTYPE)
    if script == "probe":   # every keyframe added, then reloc and loop queries in turn
        ops = [("add", k) for k in range(n_kf)]
        for q in range(n_ops_q):
            if q % 2 == 0:
                src = int(rng.integers(0, n_kf))
                w = np.unique(np.concatenate([words[src][rng.random(len(words[src])) < 0.6], draw(300)]))
                ops.append(("reloc", 1_000_000 + q, *bow(w, rng)))
            else:
                ops.append(("loop", int(rng.integers(0, n_kf)), 0.01))
        return Scene(n_words, words, weights, init=init, edges=edges, ops=ops)
    ops = [("add", k) for k in range(n_kf // 2)]
    nxt = n_kf // 2
    fid = 1_000_000
    for q in range(n_ops_q):
        for _ in range(int(rng.integers(5, 40))):
            if nxt < n_kf:
                ops.append(("add", nxt))
                nxt += 1
        for _ in range(int(rng.integers(0, 4))):
            ops.append(("erase", int(rng.integers(0, nxt))))
        if q % 7 == 3:
            ops.append(("add", int(rng.integers(0, nxt))))                # re-add or add twice
        if q % 2 == 0:
            src = int(rng.integers(0, nxt))                                # a frame near a mapped place
            w = np.unique(np.concatenate([words[src][rng.random(len(words[src])) < 0.6], draw(300)]))
            ops.append(("reloc", fid, *bow(w, rng)))
            fid += 1
        else:
            k = int(rng.integers(0, nxt))
            ops.append(("loop", k, float(rng.choice([0.0, 0.01, 0.02, 0.05]))))
    return Scene(n_words, words, weights, init=init, edges=edges, ops=ops)


def growth_scene():
    """Case 10: one handle whose slot table and word pool grow past several 1 MiB block boundaries between queries."""
    rng = np.random.default_rng(11)
    n_kf = 60
    words, weights = [], []
    for i in range(n_kf):
        b = bow(rng.choice(200_000, int(rng.integers(5000, 20000)), replace=False), rng)
        words.append(b[0])
        weights.append(b[1])
    ops = []
    for i in range(n_kf):
        ops.append(("add", i))
        if i % 6 == 5:
            ops.append(("reloc", 500 + i, *bow(np.concatenate([words[i - 1], words[i - 3][:100]]), rng)))
            ops.append(("loop", i - 2, 0.0))
    edges = [(i, i + 1, 3) for i in range(n_kf - 1)]
    return Scene(200_000, words, weights, edges=edges, ops=ops)


# ---------------------------------------------------------------------------------------------------------------------
def _flat(scene):
    off = np.zeros(scene.n_kf + 1, np.int64)
    off[1:] = np.cumsum([len(w) for w in scene.words])
    W = np.concatenate(scene.words + [np.zeros(0, np.uint32)]).astype(np.uint32)
    V = np.concatenate(scene.weights + [np.zeros(0)]).astype(np.float64)
    code = np.array([CODES[o[0]] for o in scene.ops], np.int32)
    arg = np.zeros(len(scene.ops), np.int32)
    oid = np.zeros(len(scene.ops), np.uint64)
    omin = np.zeros(len(scene.ops), np.float32)
    qw, qv = [], []
    for i, o in enumerate(scene.ops):
        if o[0] in ("add", "erase"):
            arg[i] = o[1]
        elif o[0] == "reloc":
            arg[i] = len(qw)
            oid[i] = o[1]
            qw.append(np.asarray(o[2], np.uint32))
            qv.append(np.asarray(o[3], np.float64))
        elif o[0] == "loop":
            arg[i] = o[1]
            omin[i] = o[2]
    qoff = np.zeros(len(qw) + 1, np.int64)
    qoff[1:] = np.cumsum([len(w) for w in qw])
    QW = np.concatenate(qw + [np.zeros(0, np.uint32)]).astype(np.uint32)
    QV = np.concatenate(qv + [np.zeros(0)]).astype(np.float64)
    return off, W, V, code, arg, oid, omin, QW, QV, qoff


def _members(arr):
    return tuple(np.ascontiguousarray(arr[f]) for f in MEMBERS_DTYPE.names)


_ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
_SRCLIB = {"refsrc": "libkfdbsrc.so", "shimsrc": "libkfdbshim.so"}
_loaded = {}


def src_available():
    """oracle/_ref/libkfdbsrc.so and libkfdbshim.so exist, or the reference is here to build them (oracle/kfdb.mk)."""
    return all(os.path.exists(os.path.join(_ORACLE, "_ref", f)) for f in _SRCLIB.values()) or \
        os.path.exists("/root/reference/src/KeyFrameDatabase.cc")


def srclib(prefix):
    """'refsrc': the reference's own KeyFrameDatabase.cc; 'shimsrc': the reference's KeyFrame.cc over the shim."""
    if prefix not in _loaded:
        path = os.path.join(_ORACLE, "_ref", _SRCLIB[prefix])
        if not os.path.exists(path):
            subprocess.check_call(["make", "-C", _ORACLE, "-f", "kfdb.mk", "-s"])
        _loaded[prefix] = C.CDLL(path)
    return _loaded[prefix]


def run_src(prefix, scene, members_every_query=True, with_times=False):
    """kfdb_run of oracle/kfdb_harness.cpp in libkfdbsrc.so (prefix 'refsrc') or libkfdbshim.so ('shimsrc')
    -> (cands, members, neigh[, op seconds])."""
    vp = C.c_void_p
    f = getattr(srclib(prefix), prefix + "_kfdb_run")
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, C.c_int] + [vp] * 7 + [vp, C.c_int64, vp, C.c_int] + [vp] * 3
    off, W, V, code, arg, oid, omin, QW, QV, qoff = _flat(scene)
    p = lambda a: a.ctypes.data_as(vp)   # noqa: E731
    nq = scene.n_queries()
    cap = max(1, nq * scene.n_kf)
    cand = np.zeros(cap, np.int32)
    coff = np.zeros(len(scene.ops) + 1, np.int64)
    mem = np.zeros((nq if members_every_query else 1) * scene.n_kf + 1, MEMBERS_DTYPE)
    neigh = np.zeros(11 * scene.n_kf + 1, np.int32)
    sec = np.zeros(len(scene.ops) + 1, np.float64)
    init = np.ascontiguousarray(scene.init)
    edges = np.ascontiguousarray(scene.edges.reshape(-1)) if len(scene.edges) else np.zeros(1, np.int32)
    rc = f(scene.n_words, scene.n_kf, p(W), p(V), p(off), p(scene.kf_id), p(init), len(scene.edges), p(edges),
           len(scene.ops), p(code), p(arg), p(oid), p(omin), p(QW), p(QV), p(qoff), p(cand), cap, p(coff),
           int(members_every_query), p(mem), p(neigh), p(sec))
    assert rc == 0, rc
    cands, qsec = [], []
    for i, o in enumerate(scene.ops):
        if o[0] in ("reloc", "loop"):
            cands.append(cand[coff[i]:coff[i + 1]].copy())
            qsec.append(sec[i])
    n_snap = nq if members_every_query else 1
    members = [_members(mem[i * scene.n_kf:(i + 1) * scene.n_kf]) for i in range(n_snap)]
    nb = [list(neigh[11 * i + 1:11 * i + 1 + neigh[11 * i]]) for i in range(scene.n_kf)]
    out = (cands, members, nb)
    return out + (np.array(qsec),) if with_times else out


def run_device(scene, members_every_query=True, db=None, timer=None):
    """The Python mirror on the GPU -> (cands, members).  timer(fn) -> fn() may wrap each query."""
    from orb_slam2_ssd_semantic_b200.keyframedb import KeyFrameDatabase
    db = db if db is not None else KeyFrameDatabase(scene.n_words)
    for k in range(scene.n_kf):
        db.init_members(k, scene.init[k].tolist())
    cands, members = [], []
    call = timer or (lambda fn: fn())

    def snap():
        a = np.zeros(scene.n_kf, MEMBERS_DTYPE)
        for k in range(scene.n_kf):
            a[k] = db.members[k]
        return _members(a)
    for o in scene.ops:
        if o[0] == "add":
            db.add(o[1], (scene.words[o[1]], scene.weights[o[1]]))
        elif o[0] == "erase":
            db.erase(o[1])
        elif o[0] == "clear":
            db.clear()
        else:
            if o[0] == "reloc":
                c = call(lambda: db.DetectRelocalizationCandidates(o[1], (o[2], o[3]), scene.neigh))
            else:
                c = call(lambda: db.DetectLoopCandidates(int(scene.kf_id[o[1]]), (scene.words[o[1]], scene.weights[o[1]]),
                                                         scene.connected[o[1]], scene.neigh, o[2]))
            cands.append(np.array(c, np.int32))
            if members_every_query:
                members.append(snap())
    if not members_every_query:
        members.append(snap())
    return cands, members

"""KeyFrameDatabase (src/KeyFrameDatabase.cc) restated in plain Python (TEST INFRASTRUCTURE): the inverted file as the
reference holds it -- one list of keyframes per word, in add order -- and both Detect* members line by line, floats in
float32, the L1 score in double (DBoW2 TemplatedVocabulary::score as oracle/standin restates it, TemplatedVocabulary.h:
79-89).  GetBestCovisibilityKeyFrames(10) is an input: `neigh[kf]` (the reference orders equal weights by address).

`run(scene)` replays a tests/kfdb_cases.py script and returns what oracle/refsrc_harness.cpp's kfdb_run flattens."""
import numpy as np

F32 = np.float32
MEMBERS = ("mnLoopQuery", "mnLoopWords", "mLoopScore", "mnRelocQuery", "mnRelocWords", "mRelocScore")


class KF:
    def __init__(self, idx, mnId, words, weights, members):
        self.idx, self.mnId = idx, int(mnId)
        self.bow = list(zip((int(w) for w in words), (float(v) for v in weights)))   # BowVector: ascending word ids
        lq, lw, ls, rq, rw, rs = members
        self.mnLoopQuery, self.mnLoopWords, self.mLoopScore = int(lq), int(lw), F32(ls)
        self.mnRelocQuery, self.mnRelocWords, self.mRelocScore = int(rq), int(rw), F32(rs)


def score(v1, v2):
    """TemplatedVocabulary::score, L1: the common words in ascending order, summed in double."""
    s, i, j = 0.0, 0, 0
    while i < len(v1) and j < len(v2):
        if v1[i][0] == v2[j][0]:
            a, b = v1[i][1], v2[j][1]
            s += abs(a - b) - abs(a) - abs(b)
            i += 1
            j += 1
        elif v1[i][0] < v2[j][0]:
            i += 1
        else:
            j += 1
    return -s / 2.0


class KeyFrameDatabase:
    def __init__(self, n_words):                                            # :32-36
        self.n_words = n_words
        self.inv = [[] for _ in range(n_words)]

    def add(self, kf):                                                      # :39-45
        for w, _ in kf.bow:
            self.inv[w].append(kf)

    def erase(self, kf):                                                    # :47-67: the first occurrence per list
        for w, _ in kf.bow:
            lst = self.inv[w]
            for k, x in enumerate(lst):
                if x is kf:
                    del lst[k]
                    break

    def clear(self):                                                        # :69-73
        self.inv = [[] for _ in range(self.n_words)]

    def detect_loop(self, q, connected, neigh, min_score):                  # :76-197
        min_score = F32(min_score)
        shared = []
        for w, _ in q.bow:                                                  # :86-104
            for k in self.inv[w]:
                if k.mnLoopQuery != q.mnId:
                    k.mnLoopWords = 0
                    if k not in connected:
                        k.mnLoopQuery = q.mnId
                        shared.append(k)
                k.mnLoopWords += 1
        if not shared:
            return []
        max_common = max(k.mnLoopWords for k in shared)                     # :113-118
        min_common = int(F32(max_common) * F32(0.8))                        # :120
        score_and_match = []
        for k in shared:                                                    # :125-139
            if k.mnLoopWords > min_common:
                si = F32(score(q.bow, k.bow))
                k.mLoopScore = si
                if si >= min_score:
                    score_and_match.append((si, k))
        if not score_and_match:
            return []
        acc_and_match, best_acc = [], min_score                             # :144-173
        for si, k in score_and_match:
            best, acc, best_kf = si, si, k
            for k2 in neigh(k):
                if k2.mnLoopQuery == q.mnId and k2.mnLoopWords > min_common:
                    acc = F32(acc + k2.mLoopScore)
                    if k2.mLoopScore > best:
                        best_kf, best = k2, k2.mLoopScore
            acc_and_match.append((acc, best_kf))
            if acc > best_acc:
                best_acc = acc
        return retain(acc_and_match, best_acc)

    def detect_reloc(self, mnId, bow, neigh):                               # :199-309
        shared = []
        for w, _ in bow:                                                    # :207-222
            for k in self.inv[w]:
                if k.mnRelocQuery != mnId:
                    k.mnRelocWords = 0
                    k.mnRelocQuery = mnId
                    shared.append(k)
                k.mnRelocWords += 1
        if not shared:
            return []
        max_common = max(k.mnRelocWords for k in shared)                    # :228-235
        min_common = int(F32(max_common) * F32(0.8))
        score_and_match = []
        for k in shared:                                                    # :242-253
            if k.mnRelocWords > min_common:
                si = F32(score(bow, k.bow))
                k.mRelocScore = si
                score_and_match.append((si, k))
        if not score_and_match:
            return []
        acc_and_match, best_acc = [], F32(0)                                # :258-287
        for si, k in score_and_match:
            best, acc, best_kf = si, si, k
            for k2 in neigh(k):
                if k2.mnRelocQuery != mnId:
                    continue
                acc = F32(acc + k2.mRelocScore)
                if k2.mRelocScore > best:
                    best_kf, best = k2, k2.mRelocScore
            acc_and_match.append((acc, best_kf))
            if acc > best_acc:
                best_acc = acc
        return retain(acc_and_match, best_acc)


def retain(acc_and_match, best_acc):                                        # :176-196, :290-306
    thr = F32(F32(0.75) * best_acc)
    out, seen = [], set()
    for acc, k in acc_and_match:
        if acc > thr and k.idx not in seen:
            out.append(k.idx)
            seen.add(k.idx)
    return out


def snapshot(kfs):
    return tuple(np.array([getattr(k, a) for k in kfs], dt) for a, dt in zip(MEMBERS, ("<u8", "<i4", "<f4") * 2))


def run(scene, members_every_query=True):
    """-> (candidates per query, members per query (or once at the end), the neighbour lists used)."""
    kfs = [KF(i, scene.kf_id[i], scene.words[i], scene.weights[i], scene.init[i]) for i in range(scene.n_kf)]
    conn = [set() for _ in kfs]
    for a, b, _ in scene.edges:
        conn[a].add(kfs[b])
        conn[b].add(kfs[a])
    db = KeyFrameDatabase(scene.n_words)
    cands, members = [], []
    neigh = lambda k: [kfs[j] for j in scene.neigh[k.idx]]   # noqa: E731
    for op in scene.ops:
        if op[0] == "add":
            db.add(kfs[op[1]])
        elif op[0] == "erase":
            db.erase(kfs[op[1]])
        elif op[0] == "clear":
            db.clear()
        else:
            if op[0] == "reloc":
                c = db.detect_reloc(int(op[1]), list(zip((int(w) for w in op[2]), (float(v) for v in op[3]))), neigh)
            else:
                c = db.detect_loop(kfs[op[1]], conn[op[1]], neigh, op[2])
            cands.append(np.array(c, np.int32))
            if members_every_query:
                members.append(snapshot(kfs))
    if not members_every_query:
        members.append(snapshot(kfs))
    return cands, members

"""Host-side mirror of ORB_SLAM2::KeyFrameDatabase (include/KeyFrameDatabase.h, src/KeyFrameDatabase.cc) over the
orbv_db_* entries of libb200orb.so.  Keyframes are integer slots; a BowVector is (word ids ascending, weights).  The
inverted-file walk, the common-word counts and the L1 scores run on the GPU; the covisibility accumulation and the
0.75f * bestAccScore filter run here in float32, as the reference writes them, on the caller's
GetBestCovisibilityKeyFrames(10) lists (`best_covisibles[slot]`).

The six members the database writes on a KeyFrame (mnLoopQuery, mnLoopWords, mLoopScore, mnRelocQuery, mnRelocWords,
mRelocScore) are kept per slot in `members`: set them with `init_members` for keyframes that a query may read before
they are added (the reference reads them on every neighbour), else a slot starts at zero on its first `add`."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._abi import ptr

MEMBERS_DTYPE = np.dtype([("loop_query", "<u8"), ("loop_words", "<i4"), ("loop_score", "<f4"),
                          ("reloc_query", "<u8"), ("reloc_words", "<i4"), ("reloc_score", "<f4")])   # OrbvDbMembers
HIT_DTYPE = np.dtype([("slot", "<i4"), ("words", "<i4"), ("query", "<u8"), ("score", "<f4"), ("flags", "<i4")])  # OrbvDbHit
RELOC, LOOP = 0, 1
APPENDED, SCORED = 1, 2
F32 = np.float32


def _bow(bow):
    w, v = bow
    return np.ascontiguousarray(w, np.uint32), np.ascontiguousarray(v, np.float64)


class KeyFrameDatabase:
    def __init__(self, n_words: int, device: int = 0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._L.orbv_db_create(int(device), int(n_words), C.byref(self._h)))
        self.n_words = n_words
        self.members = {}   # slot -> np.void of MEMBERS_DTYPE: the keyframe's six members
        self._added = set()  # slots the device knows

    def __del__(self):
        try:
            if self._h:
                self._L.orbv_db_destroy(self._h)
        except Exception:
            pass

    def init_members(self, slot: int, members) -> None:
        self.members[slot] = np.array([tuple(members)], MEMBERS_DTYPE)[0]

    def add(self, slot: int, bow) -> None:
        """KeyFrameDatabase::add (:39-45)."""
        w, v = _bow(bow)
        m = self.members.get(slot)
        if m is None:
            m = np.zeros(1, MEMBERS_DTYPE)[0]
        buf = np.array([m], MEMBERS_DTYPE)
        _lib.check(self._L.orbv_db_add(self._h, int(slot), ptr(w), ptr(v), len(w), ptr(buf)))
        self.members[slot] = buf[0]
        self._added.add(slot)

    def erase(self, slot: int) -> None:
        """KeyFrameDatabase::erase (:47-67); a slot never added is left alone, like the reference."""
        if slot in self._added:
            _lib.check(self._L.orbv_db_erase(self._h, int(slot)))

    def clear(self) -> None:
        """KeyFrameDatabase::clear (:69-73)."""
        _lib.check(self._L.orbv_db_clear(self._h))

    def state(self, slot: int):
        """(the device's copy of the slot's members, how many times the slot is in the database)."""
        m = np.zeros(1, MEMBERS_DTYPE)
        cnt, live = C.c_int(), C.c_int()
        _lib.check(self._L.orbv_db_state(self._h, int(slot), ptr(m), C.byref(cnt), C.byref(live)))
        return m[0], cnt.value

    def launch_count(self) -> int:
        return int(self._L.orbv_db_launch_count(self._h))

    def _walk(self, kind, qid, bow, connected=()):
        """The device part of a query: returns lKFsSharingWords (slots, in list order) after writing back the members."""
        w, v = _bow(bow)
        live = C.c_int()
        _lib.check(self._L.orbv_db_state(self._h, -1, None, None, C.byref(live)))
        hits = np.zeros(max(live.value, 1), HIT_DTYPE)
        conn = np.ascontiguousarray(list(connected), np.int32)
        napp, nmet = C.c_int(), C.c_int()
        _lib.check(self._L.orbv_db_query(self._h, kind, int(qid), ptr(w), ptr(v), len(w), ptr(conn), len(conn), ptr(hits),
                                         live.value, C.byref(napp), C.byref(nmet)))
        pre = "loop_" if kind == LOOP else "reloc_"
        for r in hits[:nmet.value]:
            m = self.members[int(r["slot"])]
            m[pre + "query"], m[pre + "words"], m[pre + "score"] = r["query"], r["words"], r["score"]
        return [int(s) for s in hits["slot"][:napp.value]]

    def DetectLoopCandidates(self, kf_id: int, bow, connected, best_covisibles, min_score) -> list:
        """KeyFrameDatabase::DetectLoopCandidates (:76-197) for keyframe `kf_id` with GetConnectedKeyFrames() = connected."""
        M = self.members
        shared = self._walk(LOOP, kf_id, bow, [c for c in connected if c in M])
        if not shared:
            return []
        min_score = F32(min_score)
        max_common = max(int(M[s]["loop_words"]) for s in shared)
        min_common = int(F32(max_common) * F32(0.8))
        score_and_match = [(M[s]["loop_score"], s) for s in shared
                           if M[s]["loop_words"] > min_common and M[s]["loop_score"] >= min_score]
        if not score_and_match:
            return []
        acc_and_match = []
        best_acc = min_score
        for si, s in score_and_match:                                    # :148-173
            best, acc, best_kf = si, si, s
            for n in best_covisibles[s]:
                m = M.get(n)
                if m is not None and m["loop_query"] == kf_id and m["loop_words"] > min_common:
                    acc = F32(acc + m["loop_score"])
                    if m["loop_score"] > best:
                        best_kf, best = n, m["loop_score"]
            acc_and_match.append((acc, best_kf))
            if acc > best_acc:
                best_acc = acc
        return _retain(acc_and_match, best_acc)

    def DetectRelocalizationCandidates(self, frame_id: int, bow, best_covisibles) -> list:
        """KeyFrameDatabase::DetectRelocalizationCandidates (:199-309) for a Frame with mnId = frame_id."""
        M = self.members
        shared = self._walk(RELOC, frame_id, bow)
        if not shared:
            return []
        max_common = max(int(M[s]["reloc_words"]) for s in shared)
        min_common = int(F32(max_common) * F32(0.8))
        score_and_match = [(M[s]["reloc_score"], s) for s in shared if M[s]["reloc_words"] > min_common]
        if not score_and_match:
            return []
        acc_and_match = []
        best_acc = F32(0)
        for si, s in score_and_match:                                    # :262-287, a stale mRelocScore included
            best, acc, best_kf = si, si, s
            for n in best_covisibles[s]:
                m = M.get(n)
                if m is None or m["reloc_query"] != frame_id:
                    continue
                acc = F32(acc + m["reloc_score"])
                if m["reloc_score"] > best:
                    best_kf, best = n, m["reloc_score"]
            acc_and_match.append((acc, best_kf))
            if acc > best_acc:
                best_acc = acc
        return _retain(acc_and_match, best_acc)


def _retain(acc_and_match, best_acc):
    """:176-196 / :290-306: every keyframe whose accumulated score is > 0.75f * bestAccScore, once, in list order."""
    thr = F32(F32(0.75) * best_acc)
    out, seen = [], set()
    for acc, s in acc_and_match:
        if acc > thr and s not in seen:
            out.append(s)
            seen.add(s)
    return out

"""Restatement of the perfect tree's point-pair overload SearchByProjection(cur, last, th, bMono, points_last,
points_current) (perfect/src/ORBmatcher.cc:1727-1880).  TEST INFRASTRUCTURE ONLY.

The overload is SearchByProjection(cur, last, th, bMono) (src/ORBmatcher.cc:1578-1724) token for token plus one pair per
accepted query, pushed inside `if(bestDist<=TH_HIGH)` before the rotation prune (:1835-1836).  So nmatches and the
pointer state are those of the 4-argument restatement (oracle/match_ref.cpp through oracle/ref.py), and the list of
accepted queries comes from the same restatement run on prefixes of the last frame: the search visits the queries in
order and the prune runs after the loop, so query i accepted keypoint j exactly when, after the queries 0..i alone and
without the prune, j holds i (`CurrentFrame.mvpMapPoints[bestIdx2]=pMP` at :1832; no later query of the prefix overwrote
it)."""
from __future__ import annotations

import numpy as np

from oracle import ref


def search_by_projection_last_pairs(cur, last, th, mono=False, nnratio=0.9, check_ori=True):
    """cur: _abi.FrameView, last: _abi.LastView -> (nmatches, cur2last, last2cur): last2cur[i] = the current keypoint
    query i accepted before the rotation prune, or -1."""
    from orb_slam2_ssd_semantic_b200._abi import LastView
    nm, c2l = ref.search_by_projection_last(cur, last, th, mono, nnratio, check_ori)
    acc = np.full(last.n, -1, np.int32)
    prefix = LastView(last.xw, np.zeros(last.n, np.uint8), last.octave, last.angle, last.mp_desc, last.Tcw,
                      mp_obs=last.mp_obs)
    for i in np.flatnonzero(last.valid):
        prefix.valid[i] = 1   # the queries after i stay invalid: the loop skips them
        _, state = ref.search_by_projection_last(cur, prefix, th, mono, nnratio, False)
        j = np.flatnonzero(state == i)
        if j.size:
            acc[i] = j[0]
    return nm, c2l, acc

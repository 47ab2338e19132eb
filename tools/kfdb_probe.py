"""Key-frame database timing: the reference's own DetectRelocalizationCandidates / DetectLoopCandidates
(src/KeyFrameDatabase.cc in oracle/_ref/libkfdbsrc.so) against the same members through shim/KeyFrameDatabase.h on the GPU
(oracle/_ref/libkfdbshim.so, the reference's KeyFrame objects), on the same host and inputs: synthetic maps of 100, 1,000,
10,000 and 50,000 keyframes (tests/kfdb_cases.random_scene: 300-1,000 words each over 10^5 words, Zipf-like), every
keyframe added, then reloc and loop queries in turn.  Each Detect* call is timed with steady_clock; both end on the host
(the shim's device call ends in its one sync).  Candidates and the final six members of every keyframe must be equal.
Prints one JSON line per map size; `python tools/kfdb_probe.py [out.json]` also writes them all to a file."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import kfdb_cases  # noqa: E402
from tests.refpins import digest  # noqa: E402

WARMUP, TIMED = 10, 200


def stats(t):
    t = np.asarray(t) * 1e6
    return {"median_us": float(np.median(t)), "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90))}


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"gpu": gpu, "warmup": WARMUP, "timed": TIMED, "sizes": []}
    for n in (100, 1000, 10000, 50000):
        scene = kfdb_cases.random_scene(n_kf=n, n_ops_q=WARMUP + TIMED, seed=100 + n, script="probe")
        r = kfdb_cases.run_src("refsrc", scene, members_every_query=False, with_times=True)
        s = kfdb_cases.run_src("shimsrc", scene, members_every_query=False, with_times=True)
        equal = digest(r[:2]) == digest(s[:2])
        row = {"keyframes": n, "words_total": int(sum(len(w) for w in scene.words)), "equal": equal}
        for kind, sel in (("reloc", 0), ("loop", 1)):
            idx = [i for i in range(WARMUP, WARMUP + TIMED) if i % 2 == sel]
            row[kind] = {"reference": stats(r[3][idx]), "device": stats(s[3][idx]),
                         "mean_candidates": float(np.mean([len(r[0][i]) for i in idx]))}
        print(json.dumps(row), flush=True)
        res["sizes"].append(row)
        assert equal, n
    res["all_equal"] = all(r["equal"] for r in res["sizes"])
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)
    print(gpu)


if __name__ == "__main__":
    main()

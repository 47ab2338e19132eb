"""Keyframes with detector boxes for the semantic-cluster parity tests (src/pointcloudmapping.cc:399-488): frames of the
synthetic room stream, each with a list of (x, y, width, height, class_id, prob) boxes in detector order and, where a
case needs it, crafted depth inside a box."""
import numpy as np

from orb_slam2_ssd_semantic_b200 import synth

LEAF = 0.04
_ROOM = {}


def room_frame(t, seed=11):
    if seed not in _ROOM:
        _ROOM[seed] = synth.RoomStream(seed=seed, n=64)
    _, depth, rgb, T = _ROOM[seed].frame(t)
    return depth.copy(), np.ascontiguousarray(rgb), T


def _many(seed=3, n=32):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n):
        w, h = rng.uniform(8, 160), rng.uniform(8, 120)
        out.append((float(np.float32(rng.uniform(-10, 640 - w / 2))), float(np.float32(rng.uniform(-10, 480 - h / 2))),
                    float(np.float32(w)), float(np.float32(h)), int(rng.integers(0, 21)), float(np.float32(rng.uniform(0.4, 1.0)))))
    return out


def scene(name):
    """-> (depth, bgr, Tcw, objects)."""
    if name == "overlap":        # three overlapping boxes: later boxes paint over earlier ones
        depth, bgr, T = room_frame(5)
        objs = [(100.7, 80.2, 200.5, 150.9, 9, 0.9), (180.0, 120.5, 160.3, 140.0, 15, 0.8), (150.2, 100.0, 60.0, 60.0, 5, 0.7)]
    elif name == "edges":        # x < 1, y < 1, past the bottom and right edges, wider than the image (w - 2 > cols)
        depth, bgr, T = room_frame(17)
        objs = [(0.5, 0.3, 80.0, 60.0, 20, 0.9), (600.0, 430.0, 100.0, 90.0, 9, 0.95), (-3.0, 200.0, 50.0, 40.0, 15, 0.6),
                (-20.0, 300.0, 700.0, 12.0, 3, 0.99), (630.0, 100.0, 40.0, 50.0, 1, 0.8)]
    elif name == "small_missing":   # < 51 band points, all-zero depth (mean count 0), all-NaN depth, below the gate
        depth, bgr, T = room_frame(29)
        depth[348:412, 48:112] = 0.0
        depth[48:92, 398:442] = np.nan
        objs = [(300.0, 200.0, 6.0, 6.0, 9, 0.9), (50.0, 350.0, 60.0, 50.0, 15, 0.9), (400.0, 50.0, 40.0, 40.0, 20, 0.9),
                (200.0, 200.0, 50.0, 40.0, 5, 0.3), (220.0, 260.0, 90.0, 70.0, 5, float(np.float32(0.54)))]
    elif name == "many":         # 32 boxes in one keyframe
        depth, bgr, T = room_frame(41)
        objs = _many()
    elif name == "big":          # one box of more than 60k band points: a gently tilted plane inside it
        depth, bgr, T = room_frame(53)
        cols = np.arange(640, dtype=np.float32)
        depth[79:300, 99:410] = np.float32(2.0) + np.float32(0.0005) * (cols[99:410] - np.float32(99))
        objs = [(100.0, 80.0, 300.0, 210.0, 20, 0.97)]
    else:
        raise KeyError(name)
    return depth, bgr, T, objs


NAMES = ["overlap", "edges", "small_missing", "many", "big"]

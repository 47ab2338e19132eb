"""oracle/occ_py.py -- TEST INFRASTRUCTURE, NOT PRODUCT.

Second, independent restatement (numpy scalars + plain Python) of the keyframe -> point cloud -> OctoMap path, used only to
cross-check oracle/occ_ref.cpp on small images:
  MapDrawer::GeneratePointCloud  perfect/src/MapDrawer.cc:641-675  (gates, float back-projection, VoxelGrid 1 cm, transform)
  MapDrawer::InsertScan          perfect/src/MapDrawer.cc:946-1025 (free = ray cells of ground points, occupied = endpoints)
  octomap semantics              SURVEY App. A.6 (coordToKeyChecked, computeRayKeys, updateNodeLogOdds with clamping)
Written from the reference text and the appendix, not from occ_ref.cpp: float32 arithmetic is spelled out with np.float32
so that the two restatements can only agree if both follow the same rounding sequence.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32


def _logodds(p: float) -> np.float32:
    return F32(math.log(p / (1.0 - p)))


class PyOccupancy:
    def __init__(self, resolution=0.05, prob_hit=0.7, prob_miss=0.4, clamp_min=0.12, clamp_max=0.97, depth_min=0.5,
                 depth_max=3.0, y_max=3.0, leaf=0.01):
        self.res = float(resolution)
        self.res_factor = 1.0 / self.res
        self.hit, self.miss = _logodds(prob_hit), _logodds(prob_miss)
        self.cmin, self.cmax = _logodds(clamp_min), _logodds(clamp_max)
        self.depth_min, self.depth_max, self.y_max, self.leaf = F32(depth_min), F32(depth_max), F32(y_max), F32(leaf)
        self.leaves: dict[tuple[int, int, int], np.float32] = {}
        self.points = np.zeros((0, 3), np.float32)
        self.labels = np.zeros(0, np.uint8)

    # ---- MapDrawer::GeneratePointCloud ---------------------------------------------------------------------------
    def generate(self, depth, Tcw, fx, fy, cx, cy, label=None):
        fx, fy, cx, cy = F32(fx), F32(fy), F32(cx), F32(cy)
        inv_leaf = F32(1.0) / self.leaf
        cells: dict[tuple[int, int, int], list] = {}
        rows, cols = depth.shape
        for m in range(rows):
            for n in range(cols):
                d = F32(depth[m, n])
                if d < self.depth_min or d > self.depth_max:
                    continue
                z = d
                x = F32(F32(F32(n) - cx) * z) / fx       # (n - cx) * z / fx, every step rounded to float
                y = F32(F32(F32(m) - cy) * z) / fy
                if y < -self.y_max or y > self.y_max:
                    continue
                if math.isfinite(x) and math.isfinite(y) and math.isfinite(z):
                    key = (int(math.floor(F32(z * inv_leaf))), int(math.floor(F32(y * inv_leaf))), int(math.floor(F32(x * inv_leaf))))
                else:                                    # NaN depth passes both gates: one cell of its own, emitted last
                    key = (math.inf, math.inf, math.inf)
                acc = cells.setdefault(key, [F32(0), F32(0), F32(0), 0, 0 if label is None else int(label[m, n])])
                acc[0] = F32(acc[0] + x); acc[1] = F32(acc[1] + y); acc[2] = F32(acc[2] + z)   # row-major pixel order
                acc[3] += 1
        T = [[float(v) for v in row] for row in np.asarray(Tcw, np.float32).reshape(4, 4)]   # float pose widened to double
        # inverse of the isometry, every product and sum in double, left to right
        Rt = [[T[j][i] for j in range(3)] for i in range(3)]
        ti = [-(T[0][i] * T[0][3] + T[1][i] * T[1][3] + T[2][i] * T[2][3]) for i in range(3)]
        pts, labs = [], []
        for key in sorted(cells):                        # PCL emits the cells in ascending linear index (iz, iy, ix)
            sx, sy, sz, cnt, lab = cells[key]
            c = [float(F32(sx / F32(cnt))), float(F32(sy / F32(cnt))), float(F32(sz / F32(cnt)))]
            pts.append([F32(Rt[i][0] * c[0] + Rt[i][1] * c[1] + Rt[i][2] * c[2] + ti[i]) for i in range(3)])
            labs.append(lab)
        self.points = np.array(pts, np.float32).reshape(-1, 3)
        self.labels = np.array(labs, np.uint8)
        if len(self.labels) < 50:      # perfect/src/MapDrawer.cc:676-680: a cloud of < 50 points is all ground
            self.labels[:] = 1
        return self.points

    # ---- octomap -------------------------------------------------------------------------------------------------
    def coord_to_key(self, c) -> int | None:
        if not math.isfinite(c):      # a non-finite coordinate never makes a key
            return None
        k = int(math.floor(self.res_factor * float(c))) + 32768
        return k if 0 <= k < 65536 else None

    def point_key(self, p):
        k = [self.coord_to_key(p[i]) for i in range(3)]
        return None if None in k else tuple(k)

    def ray_keys(self, origin, end):
        """OcTreeBaseImpl::computeRayKeys: the cells from the origin's to the one before the end point's."""
        ko, ke = self.point_key(origin), self.point_key(end)
        if ko is None or ke is None:
            return None
        if ko == ke:
            return []
        out = [ko]
        o = [F32(v) for v in origin]
        direction = [F32(F32(end[i]) - o[i]) for i in range(3)]
        # octomath Vector3::norm_sq() (octomap 1.9.x): x*x + y*y + z*z in float, widened for the sqrt only
        n2 = F32(F32(F32(direction[0] * direction[0]) + F32(direction[1] * direction[1])) + F32(direction[2] * direction[2]))
        length = F32(math.sqrt(float(n2)))
        direction = [F32(direction[i] / length) for i in range(3)]
        step, tmax, tdelta, cur = [0] * 3, [0.0] * 3, [0.0] * 3, list(ko)
        for i in range(3):
            step[i] = 1 if direction[i] > 0 else (-1 if direction[i] < 0 else 0)
            if step[i] != 0:
                border = (float(cur[i] - 32768) + 0.5) * self.res
                border += float(F32(step[i] * self.res * 0.5))
                tmax[i] = (border - float(o[i])) / float(direction[i])
                tdelta[i] = self.res / abs(float(direction[i]))
            else:
                tmax[i] = tdelta[i] = 1.7976931348623157e308
        while True:
            if tmax[0] < tmax[1]:
                dim = 0 if tmax[0] < tmax[2] else 2
            else:
                dim = 1 if tmax[1] < tmax[2] else 2
            cur[dim] = (cur[dim] + step[dim]) & 0xffff
            tmax[dim] += tdelta[dim]
            if tuple(cur) == ke:
                break
            if min(tmax) > float(length):
                break
            out.append(tuple(cur))
        return out

    def _update(self, key, occupied):
        v = F32(self.leaves.get(key, F32(0)) + (self.hit if occupied else self.miss))
        self.leaves[key] = min(max(v, self.cmin), self.cmax)

    # ---- MapDrawer::InsertScan (+ UpdateOctomap's sensor origin = translation of Tcw) ---------------------------------
    def insert_scan(self, Tcw):
        T = np.asarray(Tcw, np.float32).reshape(4, 4)
        origin = [T[0, 3], T[1, 3], T[2, 3]]
        free, occ = set(), set()
        for p, lab in zip(self.points, self.labels):
            if lab:
                r = self.ray_keys(origin, p)
                if r is not None:
                    free.update(r)
            else:
                k = self.point_key(p)
                if k is not None:
                    occ.add(k)
        for k in free:
            if k not in occ:
                self._update(k, False)
        for k in occ:
            self._update(k, True)

    def insert_keyframe(self, Tcw, depth, fx, fy, cx, cy, label=None):
        self.generate(np.asarray(depth, np.float32), Tcw, fx, fy, cx, cy, label)
        self.insert_scan(Tcw)
        return len(self.points)

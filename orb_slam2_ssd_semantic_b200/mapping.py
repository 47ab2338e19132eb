"""Host-side mirror of PointCloudMapping (reference include/pointcloudmapping.h:50-56) in its occupancy mode:
insertKeyFrame() pushes one RGB-D keyframe through MapDrawer::GeneratePointCloud + InsertScan semantics
(perfect/src/MapDrawer.cc:641-675, 946-1025) on the GPU."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _lib
from ._abi import GCM_CLUSTER, GcmCluster, OcmMergeStats, OcmParams, gcm_objects, ptr


class PointCloudMapping:
    def __init__(self, resolution: float = 0.05, prob_hit=0.7, prob_miss=0.4, clamp_min=0.12, clamp_max=0.97,
                 depth_min=0.5, depth_max=3.0, y_max=3.0, leaf=0.01, map_capacity=0, device: int = 0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        self.params = OcmParams(resolution, prob_hit, prob_miss, clamp_min, clamp_max, depth_min, depth_max, y_max, leaf,
                                map_capacity)
        _lib.check(self._L.ocm_create(C.byref(self.params), int(device), C.byref(self._h)))
        self.resolution = float(resolution)

    def __del__(self):
        try:
            if self._h:
                self._L.ocm_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def shutdown(self):   # PointCloudMapping::shutdown (src/pointcloudmapping.cc:104-113): nothing to join here
        _lib.check(self._L.ocm_sync(self._h))

    def insertKeyFrame(self, Tcw, depth, rgb, fx, fy, cx, cy, ground_label=None):
        """insertKeyFrame(kf, color, depth[, imgRGB]) (src/pointcloudmapping.cc:116-128): kf supplies GetPose() and the
        intrinsics; depth f32 metres; rgb u8 BGR like cv::Mat."""
        depth = np.ascontiguousarray(depth, np.float32)
        rgb = np.ascontiguousarray(rgb, np.uint8)
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        lab = None if ground_label is None else np.ascontiguousarray(ground_label, np.uint8)
        rows, cols = depth.shape
        assert rgb.shape == (rows, cols, 3)
        _lib.check(self._L.ocm_insert_keyframe(self._h, ptr(depth), ptr(rgb), rows, cols, ptr(T), float(fx), float(fy),
                                               float(cx), float(cy), ptr(lab)))

    def insert_keyframe_device(self, d_depth: int, d_rgb: int, rows: int, cols: int, Tcw, fx, fy, cx, cy, d_label: int = 0):
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        _lib.check(self._L.ocm_insert_keyframe_device(self._h, C.c_void_p(d_depth), C.c_void_p(d_rgb), rows, cols, ptr(T),
                                                      float(fx), float(fy), float(cx), float(cy),
                                                      C.c_void_p(d_label) if d_label else None))

    def insert_keyframes_device(self, d_depth: int, d_rgb: int, rows: int, cols: int, frame_idx, Tcw, fx, fy, cx, cy,
                                rgb_idx=None, d_label: int = 0, label_idx=None):
        """Keyframes (order = insertion order) of an RGB-D batch resident in HBM; one enqueue.  Keyframe i reads depth
        image frame_idx[i], colour image rgb_idx[i] and (when d_label is given) ground-label image label_idx[i]
        (default: the same index)."""
        idx = np.ascontiguousarray(frame_idx, np.int32)
        ridx = None if rgb_idx is None else np.ascontiguousarray(rgb_idx, np.int32)
        lidx = None if label_idx is None else np.ascontiguousarray(label_idx, np.int32)
        T = np.ascontiguousarray(Tcw, np.float32).reshape(len(idx), 16)
        _lib.check(self._L.ocm_insert_keyframes_labeled_device(
            self._h, C.c_void_p(d_depth), C.c_void_p(d_rgb), C.c_void_p(d_label) if d_label else None, rows, cols, ptr(idx),
            ptr(ridx), ptr(lidx), len(idx), ptr(T), float(fx), float(fy), float(cx), float(cy)))

    # ---- multi-GPU merge (ocm_merge_nccl) ----
    def nccl_init(self, rank: int, world: int, device: int, group=None):
        """Create this map's NCCL communicator: rank 0 draws the unique id, torch.distributed (plumbing only; gloo or
        nccl) hands it to the other ranks."""
        import torch
        import torch.distributed as dist
        uid = np.zeros(128, np.uint8)
        if rank == 0:
            _lib.check(self._L.ocm_nccl_unique_id(ptr(uid)))
        obj = [uid.tobytes()]
        if world > 1:
            dist.broadcast_object_list(obj, src=0, group=group)
        uid = np.frombuffer(obj[0], np.uint8).copy()
        self._comm = C.c_void_p()
        _lib.check(self._L.ocm_nccl_comm_create(ptr(uid), int(rank), int(world), int(device), C.byref(self._comm)))
        return self._comm

    def merge(self, stream: int = 0):
        """ocm_merge_nccl: close the epoch -- exchange the summaries of everything inserted since the last merge with
        the other ranks and replay all shards in rank order.  Returns OcmMergeStats."""
        st = OcmMergeStats()
        comm = getattr(self, "_comm", None)
        _lib.check(self._L.ocm_merge_nccl(self._h, comm, C.c_void_p(stream) if stream else None, C.byref(st)))
        return st

    def last_batch_stats(self):
        """(points, voxels touched) of the last round (<= 32 keyframes) of a batch insert."""
        a, b = C.c_int64(0), C.c_int64(0)
        _lib.check(self._L.ocm_last_batch_stats(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def UpdateOctomap(self, keyframes):
        """MapDrawer::UpdateOctomap (perfect/src/MapDrawer.cc:610-638): inserts keyframes [lastKeyframeSize, N-1) of the
        list -- the NEWEST keyframe is never inserted (`i < N-1`, :615) -- and remembers N-1.  `keyframes` is the whole
        list so far, each (Tcw, depth, rgb, fx, fy, cx, cy[, ground_label])."""
        N = len(keyframes)
        last = getattr(self, "lastKeyframeSize", 0)
        if N > 1:
            for i in range(last, N - 1):
                self.insertKeyFrame(*keyframes[i])
            self.lastKeyframeSize = N - 1

    def insert_keyframes_u16(self, depth_u16: np.ndarray, rgb: np.ndarray, depth_factor: float, Tcw, fx, fy, cx, cy,
                             label: np.ndarray = None):
        """Keyframes from HOST buffers as the reference's callers hold them: CV_16U depth [n,rows,cols] (converted with
        depth_factor = 1/DepthMapFactor on the device) and colour [n,rows,cols,3].  Asynchronous: the arrays (page-locked
        for a truly asynchronous upload) must stay untouched until sync()."""
        if depth_u16.dtype != np.uint16 or rgb.dtype != np.uint8 or not depth_u16.flags.c_contiguous or not rgb.flags.c_contiguous:
            raise ValueError("insert_keyframes_u16 takes C-contiguous uint16 depth and uint8 colour arrays (no hidden copies)")
        n, rows, cols = depth_u16.shape
        assert rgb.shape == (n, rows, cols, 3)
        T = np.ascontiguousarray(Tcw, np.float32).reshape(n, 16)
        if label is not None and (label.dtype != np.uint8 or not label.flags.c_contiguous or label.shape != (n, rows, cols)):
            raise ValueError("label must be a C-contiguous uint8 [n, rows, cols] array")
        _lib.check(self._L.ocm_insert_keyframes_u16_labeled(self._h, ptr(depth_u16), ptr(rgb), ptr(label), rows, cols, n,
                                                            float(np.float32(depth_factor)), ptr(T), float(fx), float(fy),
                                                            float(cx), float(cy)))

    def last_points(self):
        n = C.c_int(0)
        _lib.check(self._L.ocm_last_points(self._h, None, None, 0, C.byref(n)))
        xyz = np.zeros((n.value, 3), np.float32)
        rgb = np.zeros((n.value, 3), np.uint8)
        if n.value:
            _lib.check(self._L.ocm_last_points(self._h, ptr(xyz), ptr(rgb), n.value, C.byref(n)))
        return xyz, rgb

    def num_leaves(self) -> int:
        return int(self._L.ocm_num_leaves(self._h))

    def export_leaves(self):
        n = self.num_leaves()
        keys = np.zeros((max(n, 1), 3), np.uint16)
        lo = np.zeros(max(n, 1), np.float32)
        rgb = np.zeros((max(n, 1), 3), np.uint8)
        cnt = C.c_int64(0)
        _lib.check(self._L.ocm_export_leaves(self._h, ptr(keys), ptr(lo), ptr(rgb), n, C.byref(cnt)))
        return keys[:cnt.value], lo[:cnt.value], rgb[:cnt.value]

    def query(self, xyz):
        p = np.ascontiguousarray(xyz, np.float32)
        v, f = C.c_float(0), C.c_int(0)
        _lib.check(self._L.ocm_query(self._h, ptr(p), C.byref(v), C.byref(f)))
        return (v.value if f.value else None)

    def SaveOctoMap(self, name: str):
        """MapDrawer::SaveOctoMap (perfect/src/MapDrawer.cc:1103-1111): writes the map as a pruned ColorOcTree `.ot` file
        (octovis-readable), the tree built on the device (ocm_save_ot).  Returns (depth-16 cells in the map, nodes)."""
        nodes = C.c_int64(0)
        _lib.check(self._L.ocm_save_ot(self._h, os.fsencode(name), C.byref(nodes)))
        return self.num_leaves(), nodes.value

    def LoadOctoMap(self, name: str = "octomap.ot"):
        """MapDrawer::LoadOctoMap (:1113-1117): replaces the map by the leaves of an `.ot` file; inserts and merges
        continue from it."""
        _lib.check(self._L.ocm_load_ot(self._h, os.fsencode(name)))

    def read_ot(self, data: bytes):
        """LoadOctoMap from the bytes of an `.ot` file."""
        buf = np.frombuffer(data, np.uint8)
        _lib.check(self._L.ocm_read_ot(self._h, ptr(buf) if len(buf) else None, len(buf)))

    def tree_build(self):
        """ocm_tree_build: the pruned ColorOcTree of the map as it stands, kept on the device.  -> (nodes, leaves)."""
        nn, nl = C.c_int64(0), C.c_int64(0)
        _lib.check(self._L.ocm_tree_build(self._h, C.byref(nn), C.byref(nl)))
        return nn.value, nl.value

    def write_ot(self) -> bytes:
        """The `.ot` bytes of the last tree_build()."""
        n = C.c_int64(0)
        _lib.check(self._L.ocm_write_ot(self._h, None, 0, C.byref(n)))
        buf = np.zeros(n.value, np.uint8)
        _lib.check(self._L.ocm_write_ot(self._h, ptr(buf), n.value, C.byref(n)))
        return buf.tobytes()

    def tree_leaves(self):
        """The pruned leaves of the last tree_build() in file order -> (keys[n,3] u16 of the min corner, depth[n] u8,
        log-odds[n], rgb[n,3])."""
        n = C.c_int64(0)
        _lib.check(self._L.ocm_tree_leaves(self._h, None, None, None, None, 0, C.byref(n)))
        m = max(n.value, 1)
        keys, depth = np.zeros((m, 3), np.uint16), np.zeros(m, np.uint8)
        lo, rgb = np.zeros(m, np.float32), np.zeros((m, 3), np.uint8)
        _lib.check(self._L.ocm_tree_leaves(self._h, ptr(keys), ptr(depth), ptr(lo), ptr(rgb), n.value, C.byref(n)))
        return keys[:n.value], depth[:n.value], lo[:n.value], rgb[:n.value]

    def sync(self):
        _lib.check(self._L.ocm_sync(self._h))

    def stream(self) -> int:
        return int(self._L.ocm_stream(self._h) or 0)

    def launch_count(self) -> int:
        return int(self._L.ocm_launch_count(self._h))

    @property
    def handle(self):
        return self._h


class GlobalCloudMapping:
    """T-variant dense map (src/pointcloudmapping.cc): the accumulated colour cloud `globalMap`.

    `insertKeyFrame` = generatePointCloud + removeNaN + `*globalMap += cloud`; `refilter` = the VoxelGrid(resolution)
    pass over the whole map that the viewer thread runs after every batch of keyframes; `points()` = globalMap."""

    def __init__(self, resolution: float = 0.04, device: int = 0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._L.gcm_create(float(np.float32(resolution)), int(device), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._L.gcm_destroy(h)
            self._h = None

    def insertKeyFrame(self, Tcw, depth, color_bgr, fx, fy, cx, cy):
        depth = np.ascontiguousarray(depth, np.float32)
        bgr = np.ascontiguousarray(color_bgr, np.uint8)
        rows, cols = depth.shape
        assert bgr.shape == (rows, cols, 3)
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        _lib.check(self._L.gcm_add_keyframe(self._h, ptr(depth), ptr(bgr), rows, cols, ptr(T), float(fx), float(fy),
                                            float(cx), float(cy)))

    def insert_keyframe_device(self, d_depth: int, d_bgr: int, rows: int, cols: int, Tcw, fx, fy, cx, cy):
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        _lib.check(self._L.gcm_add_keyframe_device(self._h, C.c_void_p(d_depth), C.c_void_p(d_bgr), rows, cols, ptr(T),
                                                   float(fx), float(fy), float(cx), float(cy)))

    def insertKeyFrameObjects(self, Tcw, depth, color_bgr, fx, fy, cx, cy, keyframe_index, objects):
        """One keyframe of the semantic loop (src/pointcloudmapping.cc:413-485) with the detector's boxes `objects` (a
        GCM_OBJECT_DTYPE array or (x, y, width, height, class_id, prob) tuples, detector order): paints each box's depth
        band, appends the painted keyframe's cloud unless keyframe_index is even and there are no boxes, and returns one
        GcmCluster record per box (gcm_add_keyframe_objects)."""
        depth = np.ascontiguousarray(depth, np.float32)
        bgr = np.ascontiguousarray(color_bgr, np.uint8)
        rows, cols = depth.shape
        assert bgr.shape == (rows, cols, 3)
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        objs = gcm_objects(objects)
        out = (GcmCluster * max(len(objs), 1))()
        _lib.check(self._L.gcm_add_keyframe_objects(self._h, ptr(depth), ptr(bgr), rows, cols, ptr(T), float(fx), float(fy),
                                                    float(cx), float(cy), int(keyframe_index),
                                                    ptr(objs) if len(objs) else None, len(objs), out))
        return list(out)[:len(objs)]

    def insert_keyframe_objects_device(self, d_depth: int, d_bgr: int, rows: int, cols: int, Tcw, fx, fy, cx, cy,
                                       keyframe_index, objects):
        """insertKeyFrameObjects with depth and colour already in device memory."""
        T = np.ascontiguousarray(Tcw, np.float32).reshape(16)
        objs = gcm_objects(objects)
        out = (GcmCluster * max(len(objs), 1))()
        _lib.check(self._L.gcm_add_keyframe_objects_device(self._h, C.c_void_p(d_depth), C.c_void_p(d_bgr), rows, cols, ptr(T),
                                                           float(fx), float(fy), float(cx), float(cy), int(keyframe_index),
                                                           ptr(objs) if len(objs) else None, len(objs), out))
        return list(out)[:len(objs)]

    def refilter(self):
        _lib.check(self._L.gcm_refilter(self._h))

    def size(self) -> int:
        return int(self._L.gcm_size(self._h))

    def points(self):
        """-> (xyz float32 [n,3], rgb uint8 [n,3]) of globalMap, in VoxelGrid cell order after a refilter."""
        n = C.c_longlong(0)
        _lib.check(self._L.gcm_export(self._h, None, None, 0, C.byref(n)))
        xyz = np.zeros((max(n.value, 1), 3), np.float32)
        rgb = np.zeros((max(n.value, 1), 3), np.uint8)
        _lib.check(self._L.gcm_export(self._h, ptr(xyz), ptr(rgb), n.value, C.byref(n)))
        return xyz[:n.value], rgb[:n.value]


class SemanticClusters:
    """The cluster database of the T variant (PointCloudMapping::clusters, sem_merge, src/pointcloudmapping.cc:246-322)
    over named records.  Each cluster is a dict: object_name, class_id, prob (float32), centroid / minPt / maxPt
    (float32[3]).  merge() takes a gcm_add_keyframe_objects record with status GCM_CLUSTER and the detector's name."""

    OBJ_SIZE = np.full(21, 0.6, np.float32)    # obj_size_ (:62-70): metres within which two clusters are one object
    OBJ_SIZE[5], OBJ_SIZE[9], OBJ_SIZE[15], OBJ_SIZE[20] = np.float32(0.06), np.float32(0.5), np.float32(0.35), np.float32(0.25)

    def __init__(self):
        self.clusters = []

    def merge_record(self, name: str, class_id: int, prob, rec):
        assert rec.status == GCM_CLUSTER
        self.merge(name, class_id, prob, np.array(rec.centroid, np.float32), np.array(rec.min_pt, np.float32),
                   np.array(rec.max_pt, np.float32))

    def merge(self, name, class_id, prob, centroid, min_pt, max_pt):
        f = np.float32
        c = dict(object_name=name, class_id=int(class_id), prob=f(prob), centroid=np.asarray(centroid, f).copy(),
                 minPt=np.asarray(min_pt, f).copy(), maxPt=np.asarray(max_pt, f).copy())
        best, center_distance = None, f(100)
        for x in self.clusters:                          # every cluster with the same name, in database order
            if x["object_name"] != name:
                continue
            d = c["centroid"] - x["centroid"]            # Eigen norm(): float squares summed left to right, float sqrt
            dist = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2], dtype=f)
            if dist < center_distance:
                center_distance, best = dist, x
        if best is not None and center_distance < self.OBJ_SIZE[c["class_id"]]:
            best["prob"] = f(np.float64(f(best["prob"] + c["prob"])) / 2.0)
            best["centroid"] = (best["centroid"] + c["centroid"]) / f(2.0)
            best["minPt"] = np.where(best["minPt"] > c["minPt"], c["minPt"], best["minPt"])
            best["maxPt"] = np.where(best["maxPt"] > c["maxPt"], c["maxPt"], best["maxPt"])   # the min of the maxima (:308-310)
        else:
            self.clusters.append(c)

"""Batched stream pipeline (north_star's many-frame mode) over orbs_* of the C-ABI: per frame of a batch,
extract + ComputeStereoFromRGBD + UnprojectStereo of the previous frame + SearchByProjection(cur, last)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._abi import OrbsBatch, OrbsParams, OrbsResults, OrbxParams, ptr
from .extractor import KP_DTYPE


class StreamTracker:
    def __init__(self, nfeatures=1000, scaleFactor=1.2, nlevels=8, iniThFAST=20, minThFAST=7, fx=535.4, fy=539.2,
                 cx=320.1, cy=247.6, bf=40.0, th=15.0, nnratio=0.9, checkOri=True, max_frames=256, device=0):
        self._L = _lib.lib()
        self._h = C.c_void_p()
        p = OrbsParams(OrbxParams(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST), fx, fy, cx, cy, bf, th,
                       nnratio, int(checkOri), max_frames)
        _lib.check(self._L.orbs_create(C.byref(p), int(device), C.byref(self._h)))
        self.cap = int(self._L.orbx_max_keypoints(self._L.orbs_extractor(self._h)))
        self.nlevels = nlevels

    def __del__(self):
        try:
            if self._h:
                self._L.orbs_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def alloc_outputs(self, nframes: int, pinned: bool = False):
        """Output buffers for track_batch (kps, desc, nkp, cur2last, nmatch); pinned=True uses page-locked host
        memory (through torch) so the device->host copies are plain DMA."""
        cap = self.cap
        shapes = [((nframes, cap), KP_DTYPE), ((nframes, cap, 32), np.uint8), ((nframes,), np.int32),
                  ((nframes, cap), np.int32), ((nframes,), np.int32)]
        if not pinned:
            return tuple(np.zeros(s, d) for s, d in shapes)
        import torch
        outs = []
        self._pinned_keep = []
        for s, d in shapes:
            nbytes = int(np.prod(s)) * np.dtype(d).itemsize
            t = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
            self._pinned_keep.append(t)
            outs.append(t.numpy().view(d).reshape(s))
        return tuple(outs)

    _DTYPES = dict(gray=np.uint8, depth=np.float32, depth_u16=np.uint16, Tcw=np.float32, flow=np.float32, prev_gray=np.uint8)

    def _host_batch(self, form: str, wait: bool, out, depth_factor=0.0, binary_threshold=0.0, homography=False, **arrays):
        """One host batch through orbs_submit.  arrays: gray, one depth, Tcw, and flow or prev_gray (the flow computed on
        the device; None: the sequence starts at gray[0]).  The track_* forms (wait) convert the arrays and end in sync();
        the submit_* forms take them as they are (no hidden copies) and return after enqueueing."""
        for k, a in arrays.items():
            if a is None and k == "prev_gray":
                continue
            dt = self._DTYPES[k]
            if wait:
                arrays[k] = np.ascontiguousarray(a, dt)
            elif a.dtype != dt or not a.flags.c_contiguous:
                raise ValueError("%s takes C-contiguous %s arrays (no hidden copies)" % (form, np.dtype(dt).name))
        gray, Tcw, flow, prev = arrays["gray"], arrays["Tcw"], arrays.get("flow"), arrays.get("prev_gray")
        F, rows, cols = gray.shape
        assert arrays.get("depth", arrays.get("depth_u16")).shape == gray.shape and Tcw.size == F * 16
        if "flow" in arrays and flow.shape != (F, rows // 2, cols // 2, 2):
            raise ValueError("flow must be [nframes][rows/2][cols/2][2] float32, got %s" % (flow.shape,))
        if prev is not None and (prev.dtype != np.uint8 or prev.shape != (rows, cols)):
            raise ValueError("prev_gray must be a rows x cols uint8 image or None")
        outs = out if out is not None else self.alloc_outputs(F)
        b = OrbsBatch(F, rows, cols, 0, ptr(gray), ptr(arrays.get("depth")), ptr(arrays.get("depth_u16")),
                      float(np.float32(depth_factor)), ptr(Tcw), ptr(flow), int("prev_gray" in arrays or homography),
                      ptr(prev), float(binary_threshold), int(homography))
        _lib.check(self._L.orbs_submit(self._h, C.byref(b), C.byref(OrbsResults(*[ptr(a) for a in outs], self.cap))))
        if not wait:
            return out
        self.sync()
        return tuple(outs)

    def _device_batch(self, d_gray: int, d_depth: int, d_Tcw: int, d_flow, binary_threshold, nframes: int, rows: int,
                      cols: int):
        b = OrbsBatch(nframes, rows, cols, 1, d_gray, d_depth, None, 0.0, d_Tcw, d_flow, 0, None, float(binary_threshold))
        _lib.check(self._L.orbs_submit(self._h, C.byref(b), None))

    def track_batch(self, gray: np.ndarray, depth: np.ndarray, Tcw: np.ndarray, out=None):
        """Host buffers in, host buffers out (the reference-facing call; copies are inside)."""
        return self._host_batch("track_batch", True, out, gray=gray, depth=depth, Tcw=Tcw)

    def track_batch_u16(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray, out=None):
        """Like track_batch with the sensor's CV_16U depth; convertTo(CV_32F, depth_factor) runs on the device."""
        return self._host_batch("track_batch_u16", True, out, depth_factor, gray=gray, depth_u16=depth_u16, Tcw=Tcw)

    def submit_batch_u16(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray, out):
        """Asynchronous track_batch_u16: returns after enqueueing; `out` (alloc_outputs(pinned=True)) is valid after
        sync().  The input arrays must be page-locked, C-contiguous and stay untouched until then."""
        return self._host_batch("submit_batch_u16", False, out, depth_factor, gray=gray, depth_u16=depth_u16, Tcw=Tcw)

    def track_batch_u16_masked(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                               flow: np.ndarray, binary_threshold: float = 40.0, out=None):
        """The `perfect` variant's masked frames (perfect/src/Tracking.cc:703-719): like track_batch_u16, with the dynamic
        mask of each frame computed on the device from its half-resolution optical flow (flow[n][rows/2][cols/2][2],
        calcOpticalFlowFarneback's output; a zero field for a frame without a predecessor) and the keypoints outside the
        mask dropped before tracking.  The outputs describe the filtered frames; dynamic_mask(frame) returns the masks."""
        return self._host_batch("track_batch_u16_masked", True, out, depth_factor, binary_threshold, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw, flow=flow)

    def submit_batch_u16_masked(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                                flow: np.ndarray, binary_threshold: float, out):
        """Asynchronous track_batch_u16_masked (as submit_batch_u16): every input, the flow included, must be page-locked,
        C-contiguous and untouched until sync()."""
        return self._host_batch("submit_batch_u16_masked", False, out, depth_factor, binary_threshold, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw, flow=flow)

    def track_batch_u16_flow(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                             prev_gray=None, binary_threshold: float = 40.0, out=None):
        """track_batch_u16_masked with the optical flow computed on the device from the gray frames (pyrDown +
        calcOpticalFlowFarneback, perfect/src/Flow.cc:26-29): prev_gray is the frame before gray[0], None when the
        sequence starts at gray[0] (its flow is the zero field).  No flow crosses the host link."""
        return self._host_batch("track_batch_u16_flow", True, out, depth_factor, binary_threshold, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw, prev_gray=prev_gray)

    def submit_batch_u16_flow(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                              prev_gray, binary_threshold: float, out):
        """Asynchronous track_batch_u16_flow (as submit_batch_u16): every input, prev_gray included, must be page-locked,
        C-contiguous and untouched until sync()."""
        return self._host_batch("submit_batch_u16_flow", False, out, depth_factor, binary_threshold, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw, prev_gray=prev_gray)

    def track_batch_u16_homography(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                                   binary_threshold: float = 40.0, out=None):
        """track_batch_u16_flow along the reference's whole live path (perfect/src/Tracking.cc:703-719): before each
        frame's ComputeMask, TrackHomo (:1331-1399) searches frame t against the filtered frame t-1 and, with at least 20
        matches and more than 50 pairs, fits findHomography(points_current, points_last, RANSAC, 3); a found H makes the
        mask that of the frame warped by H (perfect/src/Flow.cc:73-80).  Everything stays on the device; the batch starts a
        sequence (frame 0 has no last frame, frame 1 no velocity) unless continue_after() carries one into it.  homography(frame) reports each frame's branch."""
        return self._host_batch("track_batch_u16_homography", True, out, depth_factor, binary_threshold, True, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw)

    def submit_batch_u16_homography(self, gray: np.ndarray, depth_u16: np.ndarray, depth_factor: float, Tcw: np.ndarray,
                                    binary_threshold: float, out):
        """Asynchronous track_batch_u16_homography (as submit_batch_u16): every input must be page-locked, C-contiguous
        and untouched until sync()."""
        return self._host_batch("submit_batch_u16_homography", False, out, depth_factor, binary_threshold, True, gray=gray,
                                depth_u16=depth_u16, Tcw=Tcw)

    HOMO_BRANCHES = ("no_last", "no_velocity", "few_matches", "few_pairs", "no_model", "warped")

    def homography(self, frame: int):
        """-> (branch name, nmatches, npairs, H 3x3 float64 or None) of `frame` of the last batch, which must have been a
        homography batch: what TrackHomo did for it (HOMO_BRANCHES, include/b200orb.h ORBS_HOMO_*), the count of its final
        search, points_current.size() and the model findHomography returned."""
        H = np.zeros(9, np.float64)
        br, nm, npairs = C.c_int(0), C.c_int(0), C.c_int(0)
        _lib.check(self._L.orbs_read_homography(self._h, int(frame), ptr(H), C.byref(br), C.byref(nm), C.byref(npairs)))
        name = self.HOMO_BRANCHES[br.value]
        return name, nm.value, npairs.value, (H.reshape(3, 3) if name == "warped" else None)

    def track_batch_masked_device(self, d_gray: int, d_depth: int, d_Tcw: int, d_flow: int, binary_threshold: float,
                                  nframes: int, rows: int, cols: int):
        """track_batch_device with the dynamic mask; d_flow = [nframes][rows/2][cols/2][2] f32 in HBM. Asynchronous."""
        if not d_flow:   # a NULL flow would make it an unmasked batch
            raise _lib.B200OrbError(-1, "bad argument")
        self._device_batch(d_gray, d_depth, d_Tcw, d_flow, binary_threshold, nframes, rows, cols)

    def dynamic_mask(self, frame: int):
        """-> (mask rows x cols uint8 0 / 1, filtered) of `frame` of the last batch, which must have been masked:
        FrameDrawer's mDynMask and whether the 65 % rule dropped keypoints of that frame."""
        rows, cols = self._mask_shape()
        mask = np.zeros((rows, cols), np.uint8)
        filtered = C.c_int(0)
        _lib.check(self._L.orbs_read_dynamic_mask(self._h, int(frame), ptr(mask), C.byref(filtered)))
        return mask, bool(filtered.value)

    def _mask_shape(self):
        r, c = C.c_int(0), C.c_int(0)
        _lib.check(self._L.orbx_level_dims(self._L.orbs_extractor(self._h), 0, C.byref(r), C.byref(c)))
        return r.value, c.value

    def set_chunk_frames(self, frames: int):
        """Frames per upload chunk of the host-buffer calls (default 128)."""
        _lib.check(self._L.orbs_set_chunk_frames(self._h, int(frames)))

    def chain_after(self, prev: "StreamTracker"):
        """The next submitted batch starts its kernels when `prev`'s kernels are done (uploads are not held back)."""
        _lib.check(self._L.orbs_chain_after(self._h, prev._h))

    def continue_after(self, prev: "StreamTracker"):
        """The next submitted batch continues the sequence of `prev`'s last batch (prev may be self): its frame 0 is
        tracked against that batch's last frame, a device_flow batch takes that frame's image as frame 0's predecessor,
        and a homography batch's TrackHomo chain carries on.  Consumed by the next batch; `prev` may go once this
        returns."""
        _lib.check(self._L.orbs_continue(self._h, prev._h))

    def track_batch_device(self, d_gray: int, d_depth: int, d_Tcw: int, nframes: int, rows: int, cols: int):
        """Device pointers (ints) in; results stay in HBM (device_results()). Asynchronous."""
        self._device_batch(d_gray, d_depth, d_Tcw, None, 0.0, nframes, rows, cols)

    def device_results(self):
        ps = [C.c_void_p() for _ in range(5)]
        cap = C.c_int()
        _lib.check(self._L.orbs_device_results(self._h, *[C.byref(p) for p in ps], C.byref(cap)))
        return [p.value for p in ps], cap.value

    def frame_glue(self, frame: int, n: int):
        """(uright, depth, xw, valid) of the first n keypoints of `frame` of the last batch."""
        cap = self.cap
        ur, dp, xw, va = np.zeros(cap, np.float32), np.zeros(cap, np.float32), np.zeros((cap, 3), np.float32), np.zeros(cap, np.uint8)
        _lib.check(self._L.orbs_read_frame_glue(self._h, int(frame), ptr(ur), ptr(dp), ptr(xw), ptr(va), cap))
        return ur[:n], dp[:n], xw[:n], va[:n]

    STAGES = ("resize", "fast", "quadtree", "blur", "orient_desc", "glue", "match")

    def profile_enable(self, on: bool = True):
        _lib.check(self._L.orbx_profile_enable(self._L.orbs_extractor(self._h), int(on)))

    def profile_read(self):
        """-> ({stage: total ms}, frames, runs) since the last read (synchronises)."""
        ms = np.zeros(7, np.float32)
        fr, runs = C.c_longlong(0), C.c_int(0)
        _lib.check(self._L.orbx_profile_read(self._L.orbs_extractor(self._h), ptr(ms), C.byref(fr), C.byref(runs)))
        return dict(zip(self.STAGES, ms.tolist())), fr.value, runs.value

    def sync(self):
        _lib.check(self._L.orbs_sync(self._h))

    def stream(self) -> int:
        return int(self._L.orbs_stream(self._h) or 0)

    def launch_count(self) -> int:
        return int(self._L.orbs_launch_count(self._h))

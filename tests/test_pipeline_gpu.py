"""GPU parity of the batched stream pipeline (extract -> stereo/unproject glue -> SearchByProjection) vs the
oracle run stage by stage on the CPU."""
import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth
from tests.helpers import frame_views

pytestmark = pytest.mark.gpu


def _stream_batch_matches_oracle(oracle, rows, cols, nfeatures=1000):
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    F = 5
    ws = synth.WallStream(seed=1234, n=F, h=rows, w=cols)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames])
    T = np.stack([f[3] for f in frames])
    st = StreamTracker(nfeatures, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9)
    kps, desc, nkp, c2l, nm = st.track_batch(gray, depth, T)
    R = oracle.RefExtractor(nfeatures, 1.2, 8, 20, 7)
    prev = None
    for t in range(F):
        K, D = R(gray[t])
        assert nkp[t] == len(K)
        assert kps[t, :nkp[t]].tobytes() == K.tobytes()
        assert (desc[t, :nkp[t]] == D).all()
        if prev is None:
            assert nm[t] == 0 and (c2l[t, :nkp[t]] == -1).all()
        else:
            cur, last = frame_views(oracle, K, D, depth[t], T[t], prev[0], prev[1], depth[t - 1], T[t - 1],
                                    R.mvScaleFactor, obs=1, rows=rows, cols=cols)
            n_ref, ref = oracle.search_by_projection_last(cur, last, 15.0, False, 0.9, True)
            assert n_ref > 100
            assert nm[t] == n_ref
            assert (c2l[t, :nkp[t]] == ref).all()
        prev = (K, D)


def test_stream_batch_matches_oracle(oracle):
    _stream_batch_matches_oracle(oracle, 480, 640)


def test_stream_batch_matches_oracle_kitti_width(oracle):
    """376 x 1241 (KITTI): the tracker hands the extractor rows of 1241 bytes, which are not 4-byte aligned."""
    _stream_batch_matches_oracle(oracle, 376, 1241)


def test_stream_batch_matches_oracle_non_fused(oracle):
    """3000 features: a frame pair no longer fits the fused LAST kernel's shared memory, so the 4 pairs of the batch go
    through the separate query / grid / candidate / resolve kernels."""
    _stream_batch_matches_oracle(oracle, 480, 640, nfeatures=3000)


def test_u16_depth_path_equals_float_path():
    """track_batch_u16 (device-side convertTo(CV_32F, 1/5000)) == track_batch on the float depth the
    reference would have computed (src/Tracking.cc:366-367)."""
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    F = 4
    ws = synth.WallStream(seed=77, n=F)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames])
    T = np.stack([f[3] for f in frames])
    d16 = np.rint(depth.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    assert (d16.astype(np.float32) * factor == depth).all()
    st = StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    a = st.track_batch(gray, depth, T)
    b = st.track_batch_u16(gray, d16, factor, T)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    assert b[4][1:].min() > 100


def _u16_batch(seed, F, **geom):
    ws = synth.WallStream(seed=seed, n=F, **geom)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames])
    T = np.stack([f[3] for f in frames])
    d16 = np.rint(depth.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    return gray, d16, d16.astype(np.float32) * factor, factor, T


def test_host_depth_kinds_equal_on_one_handle():
    """One handle fed page-locked CV_16U depth (read in place under the keypoints), pageable CV_16U depth (uploaded,
    then gathered), f32 depth and page-locked CV_16U again: the depth staging of the handle grows between the calls,
    and every output is byte-identical across the four."""
    import torch
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    gray, d16, depth, factor, T = _u16_batch(78, 3)
    pinned = torch.from_numpy(d16).pin_memory()
    st = StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    outs = [st.track_batch_u16(gray, pinned.numpy(), factor, T), st.track_batch_u16(gray, d16, factor, T),
            st.track_batch(gray, depth, T), st.track_batch_u16(gray, pinned.numpy(), factor, T)]
    for o in outs[1:]:
        for x, y in zip(outs[0], o):
            assert x.tobytes() == y.tobytes()
    assert outs[0][4][1:].min() > 100


def test_u16_pageable_depth_odd_pixel_count():
    """Pageable CV_16U depth whose batch holds an odd number of pixels (3 x 401 x 533) == track_batch on the
    matching f32 depth."""
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    gray, d16, depth, factor, T = _u16_batch(79, 3, h=401, w=533)
    assert d16.size % 4
    st = StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF)
    a = st.track_batch(gray, depth, T)
    b = st.track_batch_u16(gray, d16, factor, T)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    assert b[4][1:].min() > 50


@pytest.mark.gpu
def test_two_batches_in_flight_equal_synchronous_calls():
    """submit_batch_u16 on two alternating handles == track_batch_u16, batch by batch."""
    import torch
    from orb_slam2_ssd_semantic_b200 import StreamTracker
    ws = synth.WallStream(seed=9)
    batches = []
    for b in range(3):
        frames = [ws.frame(b * 5 + i) for i in range(5)]
        gray = torch.from_numpy(np.stack([f[0] for f in frames])).pin_memory()
        depth = np.stack([f[1] for f in frames])
        d16 = torch.from_numpy(np.rint(depth.astype(np.float64) * synth.DEPTH_FACTOR).astype(np.uint16)).pin_memory()
        T = torch.from_numpy(np.ascontiguousarray(np.stack([f[3] for f in frames]), np.float32)).pin_memory()
        batches.append((gray, d16, T))
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    mk = lambda: StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, max_frames=5)
    ref = mk()
    want = [[x.copy() for x in ref.track_batch_u16(g.numpy(), d.numpy(), factor, T.numpy())] for g, d, T in batches]
    trk = [mk(), mk()]
    outs = [t.alloc_outputs(5, pinned=True) for t in trk]
    got = []
    for k, (g, d, T) in enumerate(batches):
        if k >= 2:
            trk[k & 1].sync()
            got.append([x.copy() for x in outs[k & 1]])
        trk[k & 1].chain_after(trk[(k + 1) & 1])   # orbs_chain_after: kernels of consecutive batches in order
        trk[k & 1].submit_batch_u16(g.numpy(), d.numpy(), factor, T.numpy(), outs[k & 1])
    for k in range(max(0, len(batches) - 2), len(batches)):
        trk[k & 1].sync()
        got.append([x.copy() for x in outs[k & 1]])
    for w, g in zip(want, got):
        n = w[2]
        assert (g[2] == n).all() and (g[4] == w[4]).all()
        for f in range(5):
            assert g[0][f, :n[f]].tobytes() == w[0][f, :n[f]].tobytes()
            assert g[1][f, :n[f]].tobytes() == w[1][f, :n[f]].tobytes()
            assert (g[3][f, :n[f]] == w[3][f, :n[f]]).all()
    with pytest.raises(ValueError):
        trk[0].submit_batch_u16(batches[0][0].numpy()[:, ::2], batches[0][1].numpy(), factor, batches[0][2].numpy(), outs[0])


def test_full_size_batch_against_cpu_pipeline(oracle):
    """The bench workload at full size (256 frames 640x480, every 12th frame a keyframe): per-frame keypoint and match
    counts of the whole batch and the leaf count of the occupancy map against the multi-threaded CPU pipeline
    (oracle/pipeline_ref.cpp); three frames spread over the batch are additionally compared keypoint by keypoint."""
    import os
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, StreamTracker
    F, KF = 256, 12
    ws = synth.WallStream(seed=1234, n=F)
    frames = [ws.frame(t) for t in range(F)]
    gray = np.stack([f[0] for f in frames])
    depth = np.stack([f[1] for f in frames])
    rgb = np.stack([f[2] for f in frames])
    T = np.stack([f[3] for f in frames]).astype(np.float32)
    st = StreamTracker(1000, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9,
                       max_frames=F)
    kps, desc, nkp, c2l, nm = st.track_batch(gray, depth, T)
    pcm = PointCloudMapping(0.05)
    kfs = list(range(0, F, KF))
    for t in kfs:
        pcm.insertKeyFrame(T[t], depth[t], rgb[t], synth.FX, synth.FY, synth.CX, synth.CY)
    nthreads = min(os.cpu_count() or 1, 64)
    _, nkp_ref, nm_ref = oracle.pipeline_run(gray, depth, T, nthreads, rgb=rgb, kf_every=KF)
    assert (nkp == nkp_ref).all() and nkp.min() > 900
    assert (nm == nm_ref).all() and nm[1:].min() > 100
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    for t in (0, 131, 255):
        K, D = R(gray[t])
        assert kps[t, :nkp[t]].tobytes() == K.tobytes() and (desc[t, :nkp[t]] == D).all()
    ref_map = oracle.RefOccupancy()
    for t in kfs:
        ref_map.insert_keyframe(T[t], depth[t], rgb[t], synth.FX, synth.FY, synth.CX, synth.CY, None)
    kr, lr = ref_map.export_leaves()
    kg, lg, _ = pcm.export_leaves()
    assert len(kg) == len(kr) and pcm.num_leaves() == len(kr)
    pk = lambda k: np.sort(k.astype(np.uint64)[:, 0] | (k.astype(np.uint64)[:, 1] << np.uint64(16)) | (k.astype(np.uint64)[:, 2] << np.uint64(32)))
    assert (pk(kg) == pk(kr)).all()


def test_full_size_bench_workload_against_reference_sources(oracle):
    """The bench workload at full size, as bench.py runs it: one 256-frame batch of the ROOM stream (non-planar, panning
    camera), ORBextractor(2000, ...), SearchByProjection(th = 15) -- per-frame keypoint and match counts of the whole batch
    against the reference's OWN tracking sources (oracle/_ref: Frame constructor + ORBmatcher of /root/reference), three
    frames keypoint by keypoint against the oracle, and the occupancy map of the batch's 22 keyframes with the GT floor as
    ground label (free-space rays) against the sequential occupancy oracle: same leaf set, log-odds bit-equal."""
    import os
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, StreamTracker
    F, KF, NF = 256, 12, 2000
    rs = synth.RoomStream(seed=1234, n=F)
    frames = [rs.frame(t, with_label=True) for t in range(F)]
    gray, depth = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    rgb, T = np.stack([f[2] for f in frames]), np.stack([f[3] for f in frames]).astype(np.float32)
    label = np.stack([f[4] for f in frames])
    st = StreamTracker(NF, 1.2, 8, 20, 7, synth.FX, synth.FY, synth.CX, synth.CY, synth.BF, th=15.0, nnratio=0.9, max_frames=F)
    kps, desc, nkp, c2l, nm = st.track_batch(gray, depth, T)
    nthreads = min(os.cpu_count() or 1, 64)
    run = oracle.src_pipeline_run if oracle.refsrc_available() else oracle.pipeline_run
    _, nkp_ref, nm_ref = run(gray, depth, T, nthreads, NF, fx=synth.FX, fy=synth.FY, cx=synth.CX, cy=synth.CY, bf=synth.BF)
    assert (nkp == nkp_ref).all() and nkp.min() > 1900
    assert (nm == nm_ref).all() and nm[1:].min() > 300
    R = oracle.RefExtractor(NF, 1.2, 8, 20, 7)
    for t in (0, 131, 255):
        K, D = R(gray[t])
        assert kps[t, :nkp[t]].tobytes() == K.tobytes() and (desc[t, :nkp[t]] == D).all()
    import torch
    kfs = list(range(0, F, KF))
    pcm = PointCloudMapping(0.05)
    d_depth, d_rgb, d_lab = torch.from_numpy(depth).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(label).cuda()
    pcm.insert_keyframes_device(d_depth.data_ptr(), d_rgb.data_ptr(), 480, 640, kfs, T[kfs], synth.FX, synth.FY, synth.CX, synth.CY,
                                d_label=d_lab.data_ptr())
    pcm.sync()
    ref_map = oracle.RefOccupancy()
    ref_map.insert_keyframes_mt(depth, rgb, label, kfs, T[kfs], synth.FX, synth.FY, synth.CX, synth.CY, nthreads)
    kr, lr = ref_map.export_leaves()
    kg, lg, _ = pcm.export_leaves()
    pk = lambda k: k.astype(np.uint64)[:, 0] | (k.astype(np.uint64)[:, 1] << np.uint64(16)) | (k.astype(np.uint64)[:, 2] << np.uint64(32))
    og, orr = np.argsort(pk(kg)), np.argsort(pk(kr))
    assert len(kg) == len(kr) and (pk(kg)[og] == pk(kr)[orr]).all()
    assert (lg[og].view(np.uint32) == lr[orr].view(np.uint32)).all()
    assert (lr < 0).sum() > 5000 and (lr > 0).sum() > 5000

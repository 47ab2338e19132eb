"""GPU, 2 ranks over NCCL: keyframes sharded across GPUs, per-rank occupancy maps merged by ocm_merge_nccl (the
exchange of per-voxel clamp-add summaries) == the sequential single-map result of the CPU oracle (log-odds within
1e-5, same leaf set).

The tolerance is deliberate here, unlike the single-device tests: a merge replays min(max(x + a, lo), hi) where a is
the sum of a rank's updates since the last merge, added up in its own order, so x + a can differ from the sequential
clamped sum in the last bits."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _scene(n):
    from orb_slam2_ssd_semantic_b200 import synth
    ws = synth.WallStream(seed=7, n=n, depth0=2.0)
    out = []
    for t in range(n):
        gray, depth, rgb, T = ws.frame(t * 9)
        yy, xx = np.mgrid[0:480, 0:640]
        depth = (depth + 0.25 * np.sin(xx / 80.0 + t) * np.cos(yy / 60.0)).astype(np.float32)
        out.append((depth, rgb, T))
    return out


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, synth
    from orb_slam2_ssd_semantic_b200 import distributed as D
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        scene = _scene(6)
        b, e = D.shard_range(len(scene), world, rank)
        pcm = PointCloudMapping(0.05, device=rank)
        pcm.nccl_init(rank, world, rank)
        label = np.zeros((480, 640), np.uint8)
        label[320:, :] = 1
        for depth, rgb, T in scene[b:e]:
            pcm.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
        st = pcm.merge()
        keys, lo, _ = pcm.export_leaves()
        q.put((rank, keys, lo, st.bytes_sent))
    finally:
        dist.destroy_process_group()


def test_two_gpu_map_merge_equals_sequential(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from orb_slam2_ssd_semantic_b200 import synth
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
    ref = oracle.RefOccupancy()
    label = np.zeros((480, 640), np.uint8)
    label[320:, :] = 1
    for depth, rgb, T in _scene(6):
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, label)
    kr, lr = ref.export_leaves()

    def pack(k, v):
        k = k.astype(np.uint64)
        p = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
        o = np.argsort(p)
        return p[o], v[o]
    pr, vr = pack(kr, lr)
    for rank, keys, lo, nbytes in res:
        pg, vg = pack(keys, lo)
        assert len(pg) == len(pr) and (pg == pr).all(), "rank %d leaf set differs" % rank
        assert np.abs(vg - vr).max() <= 1e-5
        assert nbytes > 0


# ---- ocm_merge_nccl: the C-ABI epoch merge (packed 24-byte records, one grouped NCCL broadcast per epoch) ----
def _room(n, step=7):
    from orb_slam2_ssd_semantic_b200 import synth
    rs = synth.RoomStream(seed=11, n=n * step + 1)
    return [rs.frame(t * step, with_label=True) for t in range(n)]   # gray, depth, rgb, T, floor label


def _worker_nccl(rank, world, port, q, epochs, per_epoch):
    import torch
    import torch.distributed as dist
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, synth
    from orb_slam2_ssd_semantic_b200 import distributed as D
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        scene = _room(epochs * per_epoch)
        pcm = PointCloudMapping(0.05, device=rank)
        pcm.nccl_init(rank, world, rank)
        sent = 0
        for e in range(epochs):
            b, en = D.shard_range(per_epoch, world, rank)
            for gray, depth, rgb, T, lab in scene[e * per_epoch + b: e * per_epoch + en]:
                pcm.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, lab)
            st = pcm.merge()
            assert st.world == world and st.rank == rank
            sent += st.bytes_sent
        keys, lo, _ = pcm.export_leaves()
        q.put((rank, keys, lo, sent))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_ocm_merge_nccl_epochs_equal_sequential(oracle, world):
    """Keyframes of a non-planar scene with GT-floor ground labels (free-space rays), sharded over `world` GPUs in two
    epochs with ocm_merge_nccl after each: every rank ends with the leaf set and log-odds (1e-5) of the sequential
    single-map oracle."""
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    import torch.multiprocessing as mp
    from orb_slam2_ssd_semantic_b200 import synth
    epochs, per_epoch = 2, max(world, 4)
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_nccl, args=(r, world, port, q, epochs, per_epoch)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=900) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
    ref = oracle.RefOccupancy()
    for gray, depth, rgb, T, lab in _room(epochs * per_epoch):
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, lab)
    kr, lr = ref.export_leaves()

    def pack(k, v):
        k = k.astype(np.uint64)
        p = k[:, 0] | (k[:, 1] << np.uint64(16)) | (k[:, 2] << np.uint64(32))
        o = np.argsort(p)
        return p[o], v[o]
    pr, vr = pack(kr, lr)
    assert (vr < 0).sum() > 1000 and (vr > 0).sum() > 1000     # free cells from the ground rays AND occupied cells
    for rank, keys, lo, sent in res:
        pg, vg = pack(keys, lo)
        assert len(pg) == len(pr) and (pg == pr).all(), "rank %d leaf set differs" % rank
        assert np.abs(vg - vr).max() <= 1e-5
        assert sent > 0


def test_ocm_merge_single_rank_is_identity(oracle):
    """world = 1 (no communicator): merge() only closes the epoch; values keep following the sequential oracle."""
    from orb_slam2_ssd_semantic_b200 import PointCloudMapping, synth
    scene = _room(4)
    pcm = PointCloudMapping(0.05)
    ref = oracle.RefOccupancy()
    for i, (gray, depth, rgb, T, lab) in enumerate(scene):
        pcm.insertKeyFrame(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, lab)
        ref.insert_keyframe(T, depth, rgb, synth.FX, synth.FY, synth.CX, synth.CY, lab)
        if i % 2 == 1:
            st = pcm.merge()
            assert st.world == 1 and st.records_total == st.records_sent > 0
    kg, lg, _ = pcm.export_leaves()
    kr, lr = ref.export_leaves()
    a = {tuple(k): v for k, v in zip(kg.tolist(), lg.tolist())}
    b = {tuple(k): v for k, v in zip(kr.tolist(), lr.tolist())}
    assert a.keys() == b.keys()
    assert max(abs(a[k] - b[k]) for k in a) <= 1e-5

"""CPU suite for the N>1 logic: frame sharding, and the clamp-add composition algebra that makes the sharded occupancy
map equal the sequential one."""
import numpy as np

from orb_slam2_ssd_semantic_b200 import distributed as D


def test_shard_ranges_cover_everything():
    for n in (0, 1, 7, 256, 1000):
        for world in (1, 2, 3, 8):
            got = []
            for r in range(world):
                b, e = D.shard_range(n, world, r)
                assert 0 <= b <= e <= n
                got.extend(range(b, e))
                hb, b2, e2 = D.shard_frames_with_halo(n, world, r)
                assert (b2, e2) == (b, e) and hb == max(b - 1, 0)
            assert got == list(range(n))


def _seq_apply(v, deltas, cmin, cmax):
    for d in deltas:
        v = np.float32(min(max(np.float32(v + d), cmin), cmax))
    return v


def test_shard_summaries_in_order_equal_sequential(oracle):
    """The per-voxel clamp-add summaries of consecutive shards, applied in shard order (what ocm_merge_nccl does),
    give the log-odds of applying every update sequentially."""
    hit, miss, cmin, cmax = [np.float32(v) for v in oracle.RefOccupancy().constants()]
    rng = np.random.default_rng(0)
    for _ in range(300):
        seqs = [rng.choice([hit, miss], size=rng.integers(0, 12)) for _ in range(3)]   # three shards of updates
        # per-shard summary, built exactly like apply_slot does (ocm.cu)
        summ = []
        for s in seqs:
            a, lo, hi = np.float32(0), np.float32(-np.inf), np.float32(np.inf)
            for d in s:
                a = np.float32(a + d)
                lo = np.float32(min(max(np.float32(lo + d), cmin), cmax))
                hi = np.float32(min(max(np.float32(hi + d), cmin), cmax))
            summ.append((a, lo, hi))
        v = np.float32(0)
        for (a, lo, hi) in summ:    # apply shards in order (k_merge_pack packs them, k_merge_apply applies them)
            v = np.float32(min(max(np.float32(v + a), lo), hi))
        ref = _seq_apply(np.float32(0), np.concatenate(seqs) if sum(map(len, seqs)) else [], cmin, cmax)
        assert abs(float(v) - float(ref)) <= 1e-5


def test_bench_strong_scaling_partition():
    """bench.py's frame shards at 1 / 2 / 3 / 4 / 8 ranks: every frame of a step is owned by exactly one rank, pieces stay
    inside their batch, a tracked piece (owned frames + the halo frame) never exceeds a batch, keyframes are partitioned."""
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    total = bench.SUB * bench.BATCH
    for world in (1, 2, 3, 4, 8):
        owner = np.full(total, -1)
        nkf = 0
        for rank in range(world):
            pieces = bench.rank_pieces(world, rank)
            assert pieces, (world, rank)
            for (b, lo, hi) in pieces:
                assert 0 <= lo < hi <= bench.BATCH
                assert hi - max(lo - 1, 0) <= bench.BATCH
                assert (owner[b * bench.BATCH + lo:b * bench.BATCH + hi] == -1).all()
                owner[b * bench.BATCH + lo:b * bench.BATCH + hi] = rank
                nkf += sum(1 for t in range(lo, hi) if t % bench.KF_EVERY == 0)
            # contiguous global range
            g = [b * bench.BATCH + lo for (b, lo, hi) in pieces] + [pieces[-1][0] * bench.BATCH + pieces[-1][2]]
            assert all(x <= y for x, y in zip(g, g[1:]))
        assert (owner >= 0).all() and (np.diff(owner) >= 0).all()
        assert nkf == bench.SUB * len(range(0, bench.BATCH, bench.KF_EVERY))

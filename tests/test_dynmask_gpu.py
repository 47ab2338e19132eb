"""GPU parity of the dynamic-mask stages through the C-ABI (dynm_*): bit-exact against the cv2-pinned oracle and
against OpenCV's own outputs (tests/golden/dynmask_*.npz)."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def dm():
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    return DynamicMask()


def test_element_matches_cv2(dm):
    g = np.load(os.path.join(GOLD, "dynmask_a.npz"))
    assert (dm.element() == g["element"]).all()


@pytest.mark.parametrize("name", ["a", "b", "c", "d", "e"])
def test_mask_from_flow_equals_cv2_golden(dm, name):
    g = np.load(os.path.join(GOLD, "dynmask_%s.npz" % name))
    shape = tuple(int(v) for v in g["shape"])
    m = dm.mask_from_flow(g["flow"], float(g["thr"]), shape)
    assert m.shape == shape
    assert (np.packbits(m) == g["mask"]).all()


def test_mask_from_flow_full_size_against_oracle(dm):
    """640x480 frames: half-resolution 240x320 flow, threshold floor, NaN and huge values."""
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200.synth import flow_field
    flow = flow_field(31, 240, 320, blobs=10)
    flow[17, 23] = (np.nan, 1.0)
    flow[100, 200] = (np.inf, 0.0)
    flow[0, 0] = (1e20, 1e20)
    for thr in (1.0, 40.0, 150.0):
        m = dm.mask_from_flow(flow, thr)
        assert (m == O.mask_from_flow(flow, thr)).all(), thr
    m = dm.mask_from_flow(flow, 40.0, (481, 641))          # odd-sized gray image
    assert (m == O.mask_from_flow(flow, 40.0, (481, 641))).all()
    from orb_slam2_ssd_semantic_b200 import B200OrbError
    with pytest.raises(B200OrbError):
        dm.mask_from_flow(flow, 40.0, (479, 640))
    n0 = dm.launch_count()
    dm.mask_from_flow(flow, 40.0)
    assert dm.launch_count() - n0 == 4


def test_mask_batch_device(dm):
    import torch
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.synth import flow_field
    flows = np.stack([flow_field(40 + i, 60, 80) for i in range(3)])
    d_flow = torch.from_numpy(flows).cuda()
    d_mask = torch.zeros((3, 120, 160), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L = _lib.lib()
    _lib.check(L.dynm_mask_from_flow_batch_device(dm._h, C.c_void_p(d_flow.data_ptr()), 3, 60, 80, 40.0, C.c_void_p(d_mask.data_ptr()),
                                                  120, 160))
    _lib.check(L.dynm_sync(dm._h))
    out = d_mask.cpu().numpy()
    for i in range(3):
        assert (out[i] == O.mask_from_flow(flows[i], 40.0)).all()


def _random_kps(rng, n, rows, cols):
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = rng.uniform(19, cols - 20, n).astype(np.float32)
    kps["y"] = rng.uniform(19, rows - 20, n).astype(np.float32)
    kps["angle"] = rng.uniform(0, 360, n).astype(np.float32)
    kps["octave"] = rng.integers(0, 8, n)
    kps["response"] = rng.integers(7, 200, n).astype(np.float32)
    return kps, rng.integers(0, 256, (n, 32)).astype(np.uint8)


def test_filter_keypoints_against_oracle(dm):
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200.synth import flow_field
    rng = np.random.Generator(np.random.PCG64(9))
    mask = O.mask_from_flow(flow_field(11, 240, 320), 40.0)          # a real mask: ~2/3 static
    for n in (0, 1, 255, 256, 257, 2011):
        kps, desc = _random_kps(rng, n, 480, 640)
        k2, d2 = dm.filter_keypoints(mask, kps, desc)
        kr, dr = O.filter_keypoints(mask, kps, desc)
        assert len(k2) == len(kr) and k2.tobytes() == kr.tobytes() and (d2 == dr).all(), n
    assert 0 < len(kr) < 2011
    # a mask that is 1 on at most 65 % of the pixels filters nothing; values other than 1 do not count as inside
    kps, desc = _random_kps(rng, 500, 480, 640)
    m2 = np.zeros((480, 640), np.uint8)
    m2[:300] = 1
    k2, d2 = dm.filter_keypoints(m2, kps, desc)
    assert len(k2) == 500 and (d2 == desc).all()
    m3 = np.full((480, 640), 1, np.uint8)
    m3[:, 100:200] = 2
    k3, d3 = dm.filter_keypoints(m3, kps, desc)
    kr, dr = O.filter_keypoints(m3, kps, desc)
    assert len(k3) == len(kr) < 500 and k3.tobytes() == kr.tobytes() and (d3 == dr).all()
    # strided mask view
    big = np.ones((480, 700), np.uint8)
    big[:, :640] = mask
    k4, d4 = dm.filter_keypoints(big[:, :640], kps, desc)
    kr, dr = O.filter_keypoints(mask, kps, desc)
    assert k4.tobytes() == kr.tobytes() and (d4 == dr).all()


def test_filter_batch_device_on_extractor_layout(dm):
    """The batched entry on the layout orbx_device_results() / orbs_device_results() hand out ([F][cap] keypoints,
    [F][cap][32] descriptors, [F] counts in HBM), filled with a real extraction."""
    import torch
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200 import ORBextractor, _lib, synth
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    L = _lib.lib()
    F = 3
    imgs = np.stack([synth.synth_frame(1234, t) for t in range(F)])
    ex = ORBextractor(1000, 1.2, 8, 20, 7)
    ref = ex.extract_batch(imgs)
    cap = ex.max_keypoints() + 64
    kps = np.zeros((F, cap), KP_DTYPE)
    desc = np.zeros((F, cap, 32), np.uint8)
    cnt = np.zeros(F, np.int32)
    for f in range(F):
        cnt[f] = len(ref[f][0])
        kps[f, :cnt[f]] = ref[f][0]
        desc[f, :cnt[f]] = ref[f][1]
    masks = np.stack([O.mask_from_flow(synth.flow_field(50 + t, 240, 320), 40.0) for t in range(F)])
    masks[1] = 0          # sum <= 65 %: frame 1 keeps everything
    d_k = torch.from_numpy(kps.view(np.uint8).reshape(F, cap * 28)).cuda()
    d_d, d_n, d_m = torch.from_numpy(desc).cuda(), torch.from_numpy(cnt).cuda(), torch.from_numpy(masks).cuda()
    torch.cuda.synchronize()
    _lib.check(L.dynm_filter_keypoints_batch_device(dm._h, C.c_void_p(d_m.data_ptr()), F, 480, 640, C.c_void_p(d_k.data_ptr()),
                                                    C.c_void_p(d_d.data_ptr()), C.c_void_p(d_n.data_ptr()), cap))
    _lib.check(L.dynm_sync(dm._h))
    n = d_n.cpu().numpy()
    kp = d_k.cpu().numpy().reshape(-1).view(KP_DTYPE).reshape(F, cap)
    ds = d_d.cpu().numpy()
    for f in range(F):
        kr, dr = O.filter_keypoints(masks[f], ref[f][0], ref[f][1])
        assert n[f] == len(kr) and kp[f, :n[f]].tobytes() == kr.tobytes() and (ds[f, :n[f]] == dr).all(), f
    assert n[1] == len(ref[1][0]) and 0 < n[0] < len(ref[0][0])


@pytest.mark.parametrize("shape", [(800, 1408), (801, 1409)])
def test_mask_from_flow_beyond_the_tracker_limit(dm, shape):
    """A 400 x 704 flow: both masks have more than the 29039 words per plane the batch tracker's one-CTA-per-frame kernel
    fits in shared memory; the per-stage entry takes them."""
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200.synth import flow_field
    assert shape[0] * ((shape[1] + 31) // 32) > 29039
    flow = flow_field(61, 400, 704, blobs=12)
    flow[399, 703] = (np.nan, 0.0)
    assert (dm.mask_from_flow(flow, 40.0, shape) == O.mask_from_flow(flow, 40.0, shape)).all()


def test_mask_batch_device_equals_tracker_mask():
    """dynm_mask_from_flow_batch_device and the batch tracker's masked frames (orbs_read_dynamic_mask) give the same mask,
    bit for bit, on one 481 x 641 batch over the same flow."""
    import torch
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.dynmask import DynamicMask
    from tests.test_masked_tracking_gpu import _batch, _blob, _flows, _tracker
    F, rows, cols = 4, 481, 641
    gray, d16, _, factor, T = _batch(91, F, rows, cols)
    flow = _flows(F, rows, cols, 700)
    flow[2] = _blob(240, 320, 120, 319, 50, 70, (30.0, -12.0))
    flow[3, 5, 7] = (np.inf, np.nan)
    st = _tracker(1000, F)
    st.track_batch_u16_masked(gray, d16, factor, T, flow, 47.0)
    dm = DynamicMask()
    d_flow = torch.from_numpy(flow).cuda()
    d_mask = torch.full((F, rows, cols), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _lib.check(_lib.lib().dynm_mask_from_flow_batch_device(dm._h, C.c_void_p(d_flow.data_ptr()), F, rows // 2, cols // 2, 47.0,
                                                           C.c_void_p(d_mask.data_ptr()), rows, cols))
    _lib.check(_lib.lib().dynm_sync(dm._h))
    out = d_mask.cpu().numpy()
    for t in range(F):
        m, _ = st.dynamic_mask(t)
        assert out[t].tobytes() == m.tobytes(), t
    assert 0 < out.mean() < 1


def test_filter_keypoints_sum_beyond_32_bits(dm):
    """cv::sum of a 4106 x 4106 mask of 255s is 4 299 105 180: above 65 % of the pixels, so every keypoint is dropped
    (none sits on a 1), although the sum modulo 2^32 is not."""
    from oracle import dynmask_py as O
    rows = cols = 4106
    total = rows * cols * 255
    assert total >= 2 ** 32 and total % 2 ** 32 <= 0.65 * rows * cols
    mask = np.full((rows, cols), 255, np.uint8)
    kps, desc = _random_kps(np.random.Generator(np.random.PCG64(12)), 700, rows, cols)
    k2, d2 = dm.filter_keypoints(mask, kps, desc)
    kr, dr = O.filter_keypoints(mask, kps, desc)
    assert len(kr) == 0 and len(k2) == 0
    mask[:, :cols // 2] = 1                      # sum still above 65 %: the left half's keypoints stay
    k2, d2 = dm.filter_keypoints(mask, kps, desc)
    kr, dr = O.filter_keypoints(mask, kps, desc)
    assert 0 < len(kr) < 700 and k2.tobytes() == kr.tobytes() and (d2 == dr).all()


def test_filter_batch_device_counts_above_cap(dm):
    """dynm_filter_keypoints_batch_device when counts[f] exceeds cap: only the first cap keypoints are filtered, and the
    count becomes the number kept.  481 x 641 masks put the frames after the first at unaligned addresses; one carries
    stray values, which count by their value in the sum and never as inside."""
    import torch
    from oracle import dynmask_py as O
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    from orb_slam2_ssd_semantic_b200.synth import flow_field
    rng = np.random.Generator(np.random.PCG64(13))
    F, rows, cols, cap = 3, 481, 641, 700
    masks = np.stack([O.mask_from_flow(flow_field(80 + t, 240, 320), 40.0, (rows, cols)) for t in range(F)])
    masks[2, ::3, ::5] = 2
    masks[2, 100:110] = 255
    kps = np.zeros((F, cap), KP_DTYPE)
    desc = np.zeros((F, cap, 32), np.uint8)
    for f in range(F):
        kps[f], desc[f] = _random_kps(rng, cap, rows, cols)
    cnt = np.array([cap + 1, 333, 1 << 30], np.int32)
    d_k = torch.from_numpy(kps.view(np.uint8).reshape(F, cap * 28)).cuda()
    d_d, d_n, d_m = torch.from_numpy(desc).cuda(), torch.from_numpy(cnt).cuda(), torch.from_numpy(masks).cuda()
    torch.cuda.synchronize()
    _lib.check(_lib.lib().dynm_filter_keypoints_batch_device(dm._h, C.c_void_p(d_m.data_ptr()), F, rows, cols,
                                                             C.c_void_p(d_k.data_ptr()), C.c_void_p(d_d.data_ptr()),
                                                             C.c_void_p(d_n.data_ptr()), cap))
    _lib.check(_lib.lib().dynm_sync(dm._h))
    n = d_n.cpu().numpy()
    kp = d_k.cpu().numpy().reshape(-1).view(KP_DTYPE).reshape(F, cap)
    ds = d_d.cpu().numpy()
    dropped = []
    for f in range(F):
        m = min(int(cnt[f]), cap)
        kr, dr = O.filter_keypoints(masks[f], kps[f, :m], desc[f, :m])
        assert n[f] == len(kr) and kp[f, :n[f]].tobytes() == kr.tobytes() and (ds[f, :n[f]] == dr).all(), f
        dropped.append(0 < len(kr) < m)
    assert dropped == [False, True, True]        # frame 0's mask is 64.8 % ones: nothing is dropped

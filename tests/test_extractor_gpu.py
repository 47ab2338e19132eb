"""GPU parity of the extractor: CUDA path (through the C-ABI) vs the CPU oracle, bit-exact."""
import numpy as np
import pytest

from orb_slam2_ssd_semantic_b200 import synth

pytestmark = pytest.mark.gpu


def _cmp(K, D, K2, D2, tag=""):
    assert len(K) == len(K2), "%s: keypoint count %d vs oracle %d" % (tag, len(K), len(K2))
    for name in K.dtype.names:
        bad = np.nonzero(K[name].view(np.int32) != K2[name].view(np.int32))[0]
        assert bad.size == 0, "%s: field %s differs at %s (gpu %s, oracle %s)" % (
            tag, name, bad[:5], K[name][bad[:5]], K2[name][bad[:5]])
    assert D.shape == D2.shape
    bad = np.nonzero((D != D2).any(axis=1))[0]
    assert bad.size == 0, "%s: %d descriptors differ, first %s" % (tag, bad.size, bad[:5])


@pytest.fixture(scope="module")
def ex1000():
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    return ORBextractor(1000, 1.2, 8, 20, 7)


def test_config1_single_frame(ex1000, oracle):
    img = synth.synth_frame(1234, 0)
    K, D = ex1000(img)
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    K2, D2 = R(img)
    assert (ex1000.candidates_per_level() == R.candidates_per_level).all()
    _cmp(K, D, K2, D2, "synth0")
    assert len(K) >= 1000


def test_pyramid_levels(ex1000, oracle):
    img = synth.synth_frame(1234, 1)
    ex1000(img)
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    R(img)
    for l in range(8):
        assert (ex1000.image_pyramid_level(l) == R.level(l)).all(), "level %d" % l
        assert (ex1000.image_pyramid_level(l, bordered=True) == R.level(l, bordered=True)).all(), "bordered %d" % l


@pytest.mark.parametrize("name", ["zeros", "full", "checker2", "checker1", "noise", "lownoise", "lines", "sparse_blobs"])
def test_adversarial(ex1000, oracle, name):
    img = synth.adversarial_frames()[name]
    K, D = ex1000(img)
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    K2, D2 = R(img)
    assert (ex1000.candidates_per_level() == R.candidates_per_level).all(), (ex1000.candidates_per_level(), R.candidates_per_level)
    _cmp(K, D, K2, D2, name)


def test_batch_2000(oracle):
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    ex = ORBextractor(2000, 1.2, 8, 20, 7)
    imgs = np.stack([synth.synth_frame(1234, t) for t in range(6)])
    res = ex.extract_batch(imgs)
    R = oracle.RefExtractor(2000, 1.2, 8, 20, 7)
    for t, (K, D) in enumerate(res):
        K2, D2 = R(imgs[t])
        _cmp(K, D, K2, D2, "batch frame %d" % t)


@pytest.mark.parametrize("shape,params", [((240, 320), (500, 1.2, 8, 20, 7)), ((480, 752), (1200, 1.2, 8, 20, 7)),
                                          ((376, 1241), (2000, 1.2, 8, 20, 7)), ((300, 300), (300, 1.5, 4, 30, 10)),
                                          ((480, 640), (50, 1.2, 8, 20, 7)), ((480, 640), (1000, 1.2, 1, 20, 7)),
                                          ((401, 533), (1000, 1.2, 8, 20, 7)), ((480, 640), (500, 2.5, 3, 20, 7))])
def test_other_geometries(oracle, shape, params):
    # 401x533: odd level sizes and cell shapes; scale factor 2.5: the pyramid through k_resize instead of k_resize_g
    from orb_slam2_ssd_semantic_b200 import ORBextractor
    img = synth.synth_frame(77, 3, h=shape[0], w=shape[1])
    K, D = ORBextractor(*params)(img)
    K2, D2 = oracle.RefExtractor(*params)(img)
    _cmp(K, D, K2, D2, str((shape, params)))


def _device_to_host(ptr, nbytes):
    """Host copy of `nbytes` at device address `ptr` (a buffer the library owns)."""
    import types
    import torch
    view = types.SimpleNamespace(__cuda_array_interface__={"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False),
                                                           "version": 2})
    return torch.as_tensor(view, device="cuda").cpu().numpy()


def test_device_batch_unaligned_level0(ex1000, oracle):
    """orbx_extract_batch_device on frames whose level 0 is not 4-byte aligned (pointer 1 byte past an aligned address,
    odd pitch, odd frame stride): bit-exact with the oracle, and the level-0 read-back is the input."""
    import ctypes as C
    import torch
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.extractor import KP_DTYPE
    F, rows, cols, pitch = 3, 480, 640, 643
    fstride = rows * pitch + 5
    imgs = np.stack([synth.synth_frame(1234, t) for t in range(F)])
    host = np.zeros(1 + F * fstride, np.uint8)
    for f in range(F):
        host[1 + f * fstride:1 + f * fstride + rows * pitch].reshape(rows, pitch)[:, :cols] = imgs[f]
    d_buf = torch.from_numpy(host).cuda()
    L, h = _lib.lib(), ex1000.handle
    _lib.check(L.orbx_extract_batch_device(h, C.c_void_p(d_buf.data_ptr() + 1), F, rows, cols, pitch, fstride))
    _lib.check(L.orbx_sync(h))
    d_kps, d_desc, d_n, cap = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int()
    _lib.check(L.orbx_device_results(h, C.byref(d_kps), C.byref(d_desc), C.byref(d_n), C.byref(cap)))
    cap = cap.value
    n = _device_to_host(d_n.value, 4 * F).view(np.int32)
    kps = _device_to_host(d_kps.value, KP_DTYPE.itemsize * cap * F).view(KP_DTYPE).reshape(F, cap)
    desc = _device_to_host(d_desc.value, 32 * cap * F).reshape(F, cap, 32)
    R = oracle.RefExtractor(1000, 1.2, 8, 20, 7)
    for f in range(F):
        K2, D2 = R(imgs[f])
        _cmp(kps[f, :n[f]], desc[f, :n[f]], K2, D2, "unaligned device frame %d" % f)
        assert (ex1000.image_pyramid_level(0, frame=f) == imgs[f]).all(), "level 0 of frame %d" % f


def test_strided_and_empty(ex1000, oracle):
    big = synth.synth_frame(5, 0, h=500, w=700)
    view = big[10:490, 30:670]   # non-contiguous rows
    K, D = ex1000(view)
    K2, D2 = oracle.RefExtractor(1000, 1.2, 8, 20, 7)(np.ascontiguousarray(view))
    _cmp(K, D, K2, D2, "strided")
    K, D = ex1000(np.zeros((0, 0), np.uint8))
    assert len(K) == 0 and D.shape == (0, 32)

"""orbs_continue without a GPU: the entry is exported and bound, and NULL handles are refused before any CUDA call."""
import ctypes as C


def test_continue_is_exported_and_bound():
    from orb_slam2_ssd_semantic_b200 import _lib
    from orb_slam2_ssd_semantic_b200.pipeline import StreamTracker
    assert "orbs_continue" in _lib.EXPORTS
    L = _lib.lib()
    assert L.orbs_continue.argtypes == [C.c_void_p, C.c_void_p]
    assert callable(StreamTracker.continue_after)


def test_continue_refuses_null_handles():
    from orb_slam2_ssd_semantic_b200 import _lib
    L = _lib.lib()
    assert L.orbs_continue(None, None) == -1
    assert b"bad argument" in L.b200orb_last_error()

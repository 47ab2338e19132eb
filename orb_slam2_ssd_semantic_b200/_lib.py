"""ctypes binding of libb200orb.so (include/b200orb.h).  Fails loudly: no CPU fallback exists."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200ORB_LIB: development override, the path of another build of the library
_SO = os.environ.get("B200ORB_LIB") or os.path.join(_HERE, "libb200orb.so")


class B200OrbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("libb200orb error %d: %s" % (code, msg))
        self.code = code


from ._abi import OrbmFrustumPoints, OrbmTriKF, OcmParams, OrbmBow, OrbmFrame, OrbmLast, OrbmQueries, OrbmTrackPoints, OrbsBatch, OrbsParams, OrbsResults, OrbxParams  # noqa: E402,F401


_lib = None

# every symbol include/b200orb.h declares that is implemented so far (tests check the .so exports them)
EXPORTS = [
    "b200orb_last_error", "b200orb_device_count", "b200orb_version", "b200orb_get_tuning",
    "orbx_create", "orbx_destroy", "orbx_max_keypoints", "orbx_extract", "orbx_extract_batch",
    "orbx_extract_batch_device", "orbx_device_results", "orbx_sync", "orbx_stream", "orbx_level_dims",
    "orbx_get_level", "orbx_scale_tables", "orbx_candidates_per_level", "orbx_get_candidates", "orbx_launch_count",
    "orbx_max_keypoints_for", "orbx_distribute",
    "orbx_profile_enable", "orbx_profile_read",
    "orbm_hamming", "orbm_create", "orbm_destroy", "orbm_launch_count", "orbm_search_by_projection_last",
    "orbm_search_by_projection_last_pairs",
    "orbm_search_by_projection_points", "orbm_search_by_bow", "orbm_search_by_bow_kf", "orbm_search_projected", "orbm_search_best", "orbm_search_for_initialization", "orbm_search_for_triangulation", "orbm_is_in_frustum", "orbm_undistort_keypoints", "orbv_create", "orbv_destroy", "orbv_num_words", "orbv_launch_count", "orbv_transform",
    "orbv_db_create", "orbv_db_destroy", "orbv_db_add", "orbv_db_erase", "orbv_db_clear", "orbv_db_query", "orbv_db_state",
    "orbv_db_launch_count",
    "orbs_create", "orbs_destroy", "orbs_submit", "orbs_set_chunk_frames", "orbs_chain_after", "orbs_continue",
    "orbs_device_results",
    "orbs_read_frame_glue", "orbs_sync", "orbs_read_dynamic_mask", "orbs_read_homography",
    "orbs_stream", "orbs_launch_count", "orbs_extractor",
    "gcm_create", "gcm_destroy", "gcm_add_keyframe", "gcm_add_keyframe_device", "gcm_refilter", "gcm_size", "gcm_export", "gcm_sync", "gcm_launch_count",
    "gcm_add_keyframe_objects", "gcm_add_keyframe_objects_device",
    "ocm_default_params", "ocm_create", "ocm_destroy", "ocm_insert_keyframe", "ocm_insert_keyframe_device",
    "ocm_last_points", "ocm_num_leaves", "ocm_export_leaves", "ocm_query", "ocm_sync", "ocm_stream", "ocm_launch_count",
    "ocm_insert_keyframes_labeled_device", "ocm_insert_keyframes_u16_labeled", "ocm_merge_nccl", "ocm_nccl_unique_id",
    "ocm_nccl_comm_create", "ocm_nccl_comm_destroy", "ocm_last_batch_stats",
    "ocm_tree_build", "ocm_write_ot", "ocm_tree_leaves", "ocm_save_ot", "ocm_read_ot", "ocm_load_ot", "ocm_ot_leaves",
    "dynm_create", "dynm_destroy", "dynm_launch_count", "dynm_stream", "dynm_sync", "dynm_element", "dynm_mask_from_flow",
    "dynm_mask_from_flow_batch_device", "dynm_filter_keypoints", "dynm_filter_keypoints_batch_device",
    "dynm_farneback", "dynm_flow_batch_device", "dynm_warp_perspective", "dynm_warp_perspective_batch_device",
    "dynm_find_homography",
]


def library_path() -> str:
    return _SO


def lib() -> C.CDLL:
    """Load libb200orb.so (built in-tree by __graft_entry__.build() / csrc/Makefile)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise B200OrbError(-100, "%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                 "(there is no CPU fallback)" % _SO)
    L = C.CDLL(_SO)
    vp, i, sz = C.c_void_p, C.c_int, C.c_size_t
    L.b200orb_last_error.restype = C.c_char_p
    L.b200orb_version.restype = C.c_char_p
    L.b200orb_device_count.restype = i
    L.b200orb_get_tuning.argtypes = [C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    L.orbx_create.argtypes = [C.POINTER(OrbxParams), i, C.POINTER(vp)]
    L.orbx_destroy.argtypes = [vp]
    L.orbx_destroy.restype = None
    L.orbx_max_keypoints.argtypes = [vp]
    L.orbx_extract.argtypes = [vp, vp, i, i, sz, vp, vp, i, vp]
    L.orbx_extract_batch.argtypes = [vp, vp, i, i, i, sz, sz, vp, vp, i, vp]
    L.orbx_extract_batch_device.argtypes = [vp, vp, i, i, i, sz, sz]
    L.orbx_device_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(i)]
    L.orbx_sync.argtypes = [vp]
    L.orbx_stream.argtypes = [vp]
    L.orbx_stream.restype = vp
    L.orbx_level_dims.argtypes = [vp, i, C.POINTER(i), C.POINTER(i)]
    L.orbx_get_level.argtypes = [vp, i, i, i, vp, sz]
    L.orbx_scale_tables.argtypes = [vp, vp, vp, vp, vp, vp]
    L.orbx_candidates_per_level.argtypes = [vp, i, vp]
    L.orbx_get_candidates.argtypes = [vp, i, i, vp, i, C.POINTER(i)]
    L.orbx_max_keypoints_for.argtypes = [vp, i, i, C.POINTER(i)]
    L.orbx_distribute.argtypes = [vp, i, i, i, i, vp, i, vp, i, C.POINTER(i)]
    L.orbx_launch_count.argtypes = [vp]
    L.orbx_launch_count.restype = C.c_longlong
    L.orbx_profile_enable.argtypes = [vp, i]
    L.orbx_profile_read.argtypes = [vp, vp, C.POINTER(C.c_longlong), C.POINTER(i)]
    L.orbm_hamming.argtypes = [vp, vp]
    L.orbm_create.argtypes = [i, C.POINTER(vp)]
    L.orbm_destroy.argtypes = [vp]
    L.orbm_destroy.restype = None
    L.orbm_launch_count.argtypes = [vp]
    L.orbm_launch_count.restype = C.c_longlong
    L.orbm_search_by_projection_last.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmLast), C.c_float, i,
                                                 C.c_float, i, vp, C.POINTER(i)]
    L.orbm_search_by_projection_last_pairs.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmLast), C.c_float, i,
                                                       C.c_float, i, vp, vp, C.POINTER(i)]
    L.orbm_search_by_projection_points.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmTrackPoints), C.c_float,
                                                   C.c_float, vp, C.POINTER(i)]
    L.orbm_search_projected.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmQueries), i, i, i, vp, C.POINTER(i)]
    L.orbm_search_by_bow.argtypes = [vp, C.POINTER(OrbmBow), C.POINTER(OrbmBow), C.c_float, i, vp, C.POINTER(i)]
    L.orbm_search_by_bow_kf.argtypes = [vp, C.POINTER(OrbmBow), C.POINTER(OrbmBow), C.c_float, i, vp, C.POINTER(i)]
    L.orbm_search_best.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmQueries), i, vp, vp, vp]
    L.orbm_search_for_initialization.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmFrame), vp, i, C.c_float, i, vp, C.POINTER(i)]
    L.orbm_search_for_triangulation.argtypes = [vp, C.POINTER(OrbmTriKF), C.POINTER(OrbmTriKF), vp, C.c_float, C.c_float, vp, vp, i,
                                                i, i, vp, C.POINTER(i)]
    L.orbm_is_in_frustum.argtypes = [vp, C.POINTER(OrbmFrame), C.POINTER(OrbmFrustumPoints), C.c_float, C.c_float] + [vp] * 6
    L.orbm_undistort_keypoints.argtypes = [vp, vp, i, vp, vp, i, vp]
    L.orbv_create.argtypes = [i, i, i, i, vp, vp, vp, vp, C.POINTER(vp)]
    L.orbv_destroy.argtypes = [vp]
    L.orbv_destroy.restype = None
    L.orbv_num_words.argtypes = [vp]
    L.orbv_launch_count.argtypes = [vp]
    L.orbv_launch_count.restype = C.c_longlong
    L.orbv_transform.argtypes = [vp, vp, i, i, vp, vp, vp]
    L.orbv_db_create.argtypes = [i, i, C.POINTER(vp)]
    L.orbv_db_destroy.argtypes = [vp]
    L.orbv_db_destroy.restype = None
    L.orbv_db_add.argtypes = [vp, i, vp, vp, i, vp]
    L.orbv_db_erase.argtypes = [vp, i]
    L.orbv_db_clear.argtypes = [vp]
    L.orbv_db_query.argtypes = [vp, i, C.c_uint64, vp, vp, i, vp, i, vp, i, C.POINTER(i), C.POINTER(i)]
    L.orbv_db_state.argtypes = [vp, i, vp, C.POINTER(i), C.POINTER(i)]
    L.orbv_db_launch_count.argtypes = [vp]
    L.orbv_db_launch_count.restype = C.c_longlong
    L.dynm_create.argtypes = [i, C.POINTER(vp)]
    L.dynm_destroy.argtypes = [vp]
    L.dynm_destroy.restype = None
    L.dynm_launch_count.argtypes = [vp]
    L.dynm_launch_count.restype = C.c_longlong
    L.dynm_stream.argtypes = [vp]
    L.dynm_stream.restype = vp
    L.dynm_sync.argtypes = [vp]
    L.dynm_element.argtypes = [vp, vp]
    L.dynm_mask_from_flow.argtypes = [vp, vp, i, i, C.c_float, vp, i, i]
    L.dynm_mask_from_flow_batch_device.argtypes = [vp, vp, i, i, i, C.c_float, vp, i, i]
    L.dynm_filter_keypoints.argtypes = [vp, vp, i, i, sz, vp, vp, i, C.POINTER(i)]
    L.dynm_filter_keypoints_batch_device.argtypes = [vp, vp, i, i, i, vp, vp, vp, i]
    L.dynm_farneback.argtypes = [vp, vp, vp, i, i, vp]
    L.dynm_flow_batch_device.argtypes = [vp, vp, vp, i, i, i, vp]
    L.dynm_warp_perspective.argtypes = [vp, vp, i, i, vp, vp]
    L.dynm_warp_perspective_batch_device.argtypes = [vp, vp, i, i, i, vp, vp]
    L.dynm_find_homography.argtypes = [vp, vp, vp, i, vp, vp, vp]
    L.orbs_create.argtypes = [C.POINTER(OrbsParams), i, C.POINTER(vp)]
    L.orbs_destroy.argtypes = [vp]
    L.orbs_destroy.restype = None
    L.orbs_submit.argtypes = [vp, C.POINTER(OrbsBatch), C.POINTER(OrbsResults)]
    L.orbs_set_chunk_frames.argtypes = [vp, i]
    L.orbs_chain_after.argtypes = [vp, vp]
    L.orbs_continue.argtypes = [vp, vp]
    L.orbs_device_results.argtypes = [vp] + [C.POINTER(vp)] * 5 + [C.POINTER(i)]
    L.orbs_read_frame_glue.argtypes = [vp, i, vp, vp, vp, vp, i]
    L.orbs_read_dynamic_mask.argtypes = [vp, i, vp, C.POINTER(i)]
    L.orbs_read_homography.argtypes = [vp, i, vp, C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    L.orbs_sync.argtypes = [vp]
    L.orbs_stream.argtypes = [vp]
    L.orbs_stream.restype = vp
    L.orbs_launch_count.argtypes = [vp]
    L.orbs_launch_count.restype = C.c_longlong
    L.orbs_extractor.argtypes = [vp]
    L.orbs_extractor.restype = vp
    f = C.c_float
    L.ocm_create.argtypes = [C.POINTER(OcmParams), i, C.POINTER(vp)]
    L.ocm_destroy.argtypes = [vp]
    L.ocm_destroy.restype = None
    L.ocm_insert_keyframe.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f, vp]
    L.ocm_insert_keyframe_device.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f, vp]
    L.gcm_create.argtypes = [f, i, C.POINTER(vp)]
    L.gcm_destroy.argtypes = [vp]
    L.gcm_destroy.restype = None
    L.gcm_add_keyframe.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f]
    L.gcm_add_keyframe_device.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f]
    L.gcm_add_keyframe_objects.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f, C.c_longlong, vp, i, vp]
    L.gcm_add_keyframe_objects_device.argtypes = [vp, vp, vp, i, i, vp, f, f, f, f, C.c_longlong, vp, i, vp]
    L.gcm_refilter.argtypes = [vp]
    L.gcm_size.argtypes = [vp]
    L.gcm_size.restype = C.c_longlong
    L.gcm_export.argtypes = [vp, vp, vp, C.c_longlong, C.POINTER(C.c_longlong)]
    L.gcm_sync.argtypes = [vp]
    L.gcm_launch_count.argtypes = [vp]
    L.gcm_launch_count.restype = C.c_longlong
    L.ocm_insert_keyframes_labeled_device.argtypes = [vp, vp, vp, vp, i, i, vp, vp, vp, i, vp, f, f, f, f]
    L.ocm_insert_keyframes_u16_labeled.argtypes = [vp, vp, vp, vp, i, i, i, f, vp, f, f, f, f]
    L.ocm_merge_nccl.argtypes = [vp, vp, vp, vp]
    L.ocm_nccl_unique_id.argtypes = [vp]
    L.ocm_nccl_comm_create.argtypes = [vp, i, i, i, C.POINTER(vp)]
    L.ocm_nccl_comm_destroy.argtypes = [vp]
    L.ocm_last_batch_stats.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.ocm_last_points.argtypes = [vp, vp, vp, i, C.POINTER(i)]
    L.ocm_num_leaves.argtypes = [vp]
    L.ocm_num_leaves.restype = C.c_int64
    L.ocm_export_leaves.argtypes = [vp, vp, vp, vp, C.c_int64, C.POINTER(C.c_int64)]
    L.ocm_query.argtypes = [vp, vp, C.POINTER(f), C.POINTER(i)]
    i64p = C.POINTER(C.c_int64)
    L.ocm_tree_build.argtypes = [vp, i64p, i64p]
    L.ocm_write_ot.argtypes = [vp, vp, C.c_int64, i64p]
    L.ocm_tree_leaves.argtypes = [vp, vp, vp, vp, vp, C.c_int64, i64p]
    L.ocm_save_ot.argtypes = [vp, C.c_char_p, i64p]
    L.ocm_read_ot.argtypes = [vp, vp, C.c_int64]
    L.ocm_load_ot.argtypes = [vp, C.c_char_p]
    L.ocm_ot_leaves.argtypes = [vp, C.c_int64, C.POINTER(C.c_double), vp, vp, vp, vp, C.c_int64, i64p]
    L.ocm_sync.argtypes = [vp]
    L.ocm_stream.argtypes = [vp]
    L.ocm_stream.restype = vp
    L.ocm_launch_count.argtypes = [vp]
    L.ocm_launch_count.restype = C.c_longlong
    _lib = L
    return L


def check(rc: int) -> None:
    if rc != 0:
        raise B200OrbError(rc, lib().b200orb_last_error().decode("utf-8", "replace"))

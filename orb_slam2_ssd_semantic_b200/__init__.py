"""orb_slam2_ssd_semantic_b200 -- H100 (sm_90a) implementation of the ORB-SLAM2 hot path.

Host-side mirror of the reference's class surface for the path (ORBextractor, ORBmatcher,
PointCloudMapping) over the C-ABI of libb200orb.so (include/b200orb.h).  There is no CPU fallback:
every operator raises if the CUDA library or a GPU is missing.
"""
from ._lib import B200OrbError, lib, library_path  # noqa: F401
from .extractor import KP_DTYPE, ORBextractor  # noqa: F401
from .matcher import ORBmatcher, FrameView, LastView, TrackPointsView, BowView, QueriesView  # noqa: F401
from .pipeline import StreamTracker  # noqa: F401
from .mapping import GlobalCloudMapping, PointCloudMapping, SemanticClusters  # noqa: F401
from .vocabulary import ORBVocabulary  # noqa: F401
from .keyframedb import KeyFrameDatabase  # noqa: F401

__all__ = ["ORBextractor", "KP_DTYPE", "B200OrbError", "lib", "library_path"]

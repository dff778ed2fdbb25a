"""centerpose_b200 -- H100-native (sm_90a) CenterPose inference hot path.

Public surface (mirrors the reference's, see INTEGRATION.md):
    create_model, load_model, save_model      <- lib.models.model
    ObjectPoseDetector, detector_factory      <- lib.detectors.*
    MultiCategoryDetector                     <- one checkpoint per category, all in one plan
    MultiCategoryTracker                      <- the same for CenterPoseTrack checkpoints, one tracker for all
    TrackGraph                                <- run_batch(track=True) of video slots, replayed as a CUDA graph
    MultiCategoryTrackGraph                   <- the same for a MultiCategoryTracker's categories
    DetectGraph                               <- run_batch of a detection model's cameras, replayed as a CUDA graph
    LensDistortion                            <- a camera's lens distortion, undistorted inside the pre-process
    MultiCategoryDetectGraph                  <- the same for a MultiCategoryDetector's categories
    decode_pnp, decode_params, make_meta      <- fused decode / grouping / PnP stage
    dcn_v2_forward / dcn_v2_backward          <- `_ext.dcn_v2_forward` / `_ext.dcn_v2_backward`
The hot path lives in libcenterpose_b200.so (include/centerpose_b200.h); there is
no PyTorch or CPU fallback.
"""
from .model import create_model, load_model, save_model, DLASegB200, PoseResNetB200          # noqa: F401
from .detector import MultiCategoryDetector, MultiCategoryTracker, ObjectPoseDetector, detector_factory  # noqa: F401
from .engine import Engine, InferGraph, decode_pnp, decode_params, make_meta, dcn_v2_forward, dcn_v2_backward, preprocess, preprocess_ragged, preprocess_yuv420, preprocess_formats, preprocess_remap, conv2d_nhwc  # noqa: F401
from .graph import DetectGraph, MultiCategoryDetectGraph                     # noqa: F401
from .lens import LensDistortion                                             # noqa: F401
from .opts import default_opt                                                # noqa: F401
from .tracker import MultiCategoryTrackGraph, Tracker, TrackGraph, track_to_dict, tracks_to_results  # noqa: F401
from .pipeline import BatchPipeline, TrackPipeline                           # noqa: F401

__version__ = "0.1.0"

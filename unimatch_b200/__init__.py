"""unimatch_b200 -- H100-native (sm_90a) implementation of the UniMatch matching inference path.

    from unimatch_b200 import UniMatch      # drop-in for reference unimatch.unimatch.UniMatch (inference)

The C-ABI library (libunimatch_sm100.so) is loaded -- and built with nvcc when the in-tree copy is stale -- the first
time `ops`, `UniMatch` or one of the inference / validation / submission drivers is touched; `spec`, `synthetic` and `sharding` are plain Python and
import without it (the CPU reference arm of bench.py and the oracle tests never map the product library).
There is no CPU / eager fallback for the `torch.ops.unimatch_sm100.*` ops.
"""
import importlib

from .spec import BASELINE_CONFIGS, WORKLOADS, param_spec   # noqa: F401

_LAZY = {
    "ops": (".ops", None),
    "UniMatch": (".unimatch", "UniMatch"),
    "InputPadder": (".inference", "InputPadder"),
    "forward_backward_consistency_check": (".inference", "forward_backward_consistency_check"),
    "infer_flow": (".inference", "infer_flow"),
    "infer_stereo": (".inference", "infer_stereo"),
    "infer_depth": (".inference", "infer_depth"),
    "BatchedFlowRunner": (".inference", "BatchedFlowRunner"),
    "infer_flow_video": (".inference", "infer_flow_video"),
    "VideoFlowRunner": (".inference", "VideoFlowRunner"),
    "VideoTrackRunner": (".inference", "VideoTrackRunner"),
    "chain_tracks": (".inference", "chain_tracks"),
    "PointTrackRunner": (".inference", "PointTrackRunner"),
    "track_points": (".inference", "track_points"),
    "MultiFlowTrackRunner": (".inference", "MultiFlowTrackRunner"),
    "multi_flow_tracks": (".inference", "multi_flow_tracks"),
    "multi_flow_sources": (".inference", "multi_flow_sources"),
    "flow_to_image": (".inference", "flow_to_image"),
    "infer_depth_sequence": (".inference", "infer_depth_sequence"),
    "DepthSequenceRunner": (".inference", "DepthSequenceRunner"),
    "StereoRunner": (".inference", "StereoRunner"),
    "MixedSizeStereoRunner": (".inference", "MixedSizeStereoRunner"),
    "MixedSizeFlowRunner": (".inference", "MixedSizeFlowRunner"),
    "MixedSizeDepthRunner": (".inference", "MixedSizeDepthRunner"),
    "disparity_to_image": (".inference", "disparity_to_image"),
    "depth_to_image": (".inference", "depth_to_image"),
    "warp_disparity": (".inference", "warp_disparity"),
    "infer_scene_flow": (".inference", "infer_scene_flow"),
    "SceneFlowRunner": (".inference", "SceneFlowRunner"),
    "validate_scene_flow": (".evaluation", "validate_scene_flow"),
    "create_scene_flow_submission": (".submission", "create_scene_flow_submission"),
    "DepthFusionRunner": (".inference", "DepthFusionRunner"),
    "TSDFVolume": (".fusion", "TSDFVolume"),
    "fuse_depths": (".fusion", "fuse_depths"),
    "write_ply": (".fusion", "write_ply"),
    "read_ply": (".fusion", "read_ply"),
    "nearest_neighbors": (".fusion", "nearest_neighbors"),
    "voxel_down_sample": (".fusion", "voxel_down_sample"),
    "reconstruction_metrics": (".evaluation", "reconstruction_metrics"),
    "render_mesh": (".fusion", "render_mesh"),
    "visible_points": (".fusion", "visible_points"),
    "depth_metrics": (".evaluation", "depth_metrics"),
    "sequence_sources": (".fusion", "sequence_sources"),
    "filter_depths": (".fusion", "filter_depths"),
    "depth_points": (".fusion", "depth_points"),
    "validate_flow": (".evaluation", "validate_flow"),
    "validate_stereo": (".evaluation", "validate_stereo"),
    "validate_depth": (".evaluation", "validate_depth"),
    "tapvid_metrics": (".evaluation", "tapvid_metrics"),
    "create_flow_submission": (".submission", "create_flow_submission"),
    "create_stereo_submission": (".submission", "create_stereo_submission"),
    "inference_flow": (".inference_io", "inference_flow"),
    "inference_stereo": (".inference_io", "inference_stereo"),
    "inference_depth": (".inference_io", "inference_depth"),
}

__all__ = ["UniMatch", "ops", "WORKLOADS", "BASELINE_CONFIGS", "param_spec", "InputPadder", "infer_flow", "infer_stereo",
           "infer_depth", "BatchedFlowRunner", "forward_backward_consistency_check", "infer_flow_video", "VideoFlowRunner",
           "VideoTrackRunner", "chain_tracks", "PointTrackRunner", "track_points", "MultiFlowTrackRunner",
           "multi_flow_tracks", "multi_flow_sources", "flow_to_image", "infer_depth_sequence", "DepthSequenceRunner", "StereoRunner",
           "MixedSizeStereoRunner", "MixedSizeFlowRunner", "MixedSizeDepthRunner", "disparity_to_image", "depth_to_image",
           "validate_flow", "validate_stereo", "validate_depth", "tapvid_metrics", "create_flow_submission", "create_stereo_submission",
           "inference_flow", "inference_stereo", "inference_depth", "warp_disparity", "infer_scene_flow", "SceneFlowRunner",
           "validate_scene_flow", "create_scene_flow_submission", "DepthFusionRunner", "TSDFVolume", "fuse_depths", "write_ply",
           "read_ply", "nearest_neighbors", "voxel_down_sample", "reconstruction_metrics",
           "render_mesh", "visible_points", "depth_metrics", "sequence_sources", "filter_depths", "depth_points"]


def __getattr__(name):
    if name in _LAZY:
        mod, attr = _LAZY[name]
        m = importlib.import_module(mod, __name__)
        val = m if attr is None else getattr(m, attr)
        globals()[name] = val
        return val
    raise AttributeError("module %r has no attribute %r" % (__name__, name))

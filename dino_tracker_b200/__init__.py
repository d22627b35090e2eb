"""dino_tracker_b200 -- H100 (sm_90a) implementation of the DINO-Tracker inference hot path.

Host side mirrors the reference's ``models/tracker.py`` + ``models/model_inference.py`` call surface
(SURVEY.md 8b); all arithmetic runs in hand-written CUDA kernels behind the C ABI of
``include/dinotrk.h`` (``libdinotrk.so``, loaded with ctypes).  There is no CPU fallback.

(The importable package name uses an underscore; ``dino-tracker_b200`` is not a valid Python module
name.)
"""
from .range_normalizer import RangeNormalizer  # noqa: F401
from .tracker import Tracker  # noqa: F401
from .model_inference import (ModelInference, generate_trajectory_input, generate_trajectory,  # noqa: F401
                              generate_trajectories)

from .vit import DinoV2Features, get_dino_features_video  # noqa: F401
from .pipeline import build_tracker_from_video, track_video, save_dino_embed_video, preprocess_best_buddies  # noqa: F401
from .benchmark import infer_query_frames, save_predictions, run_videos  # noqa: F401
from .trajectories import extract_trajectories, save_trajectories  # noqa: F401
from .best_buddies import of_filter, run_of_filter  # noqa: F401
from .trainer import DinoTrackerTrainer  # noqa: F401

__all__ = ["DinoTrackerTrainer", "extract_trajectories", "save_trajectories", "of_filter", "run_of_filter", "preprocess_best_buddies",
           "infer_query_frames", "save_predictions", "run_videos", "DinoV2Features", "get_dino_features_video", "build_tracker_from_video", "track_video", "save_dino_embed_video","Tracker", "ModelInference", "RangeNormalizer", "generate_trajectory_input", "generate_trajectory",
           "generate_trajectories"]

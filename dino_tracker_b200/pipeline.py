"""In-process per-video pipeline: frames -> DINOv2 features (a1) -> delta-DINO refinement (a2) -> tracker.

The reference splits this over separate processes and a disk round trip
(``preprocessing/save_dino_embed_video.py`` -> ``dino_embed_video.pt`` -> ``Tracker.load_dino_embed_video``);
here the ViT writes token-major features that the tracker adopts without a copy.  ``save_dino_embed_video`` keeps
the on-disk format (T x C x h x w fp32) for existing tooling (SURVEY.md 8f-1).
"""
import os

import torch

from .model_inference import ModelInference
from .tracker import Tracker
from .vit import DinoV2Features


def build_tracker_from_video(video01, vit: DinoV2Features, device="cuda:0", ckpt_path="", delta_channels=None,
                             corr_precision="fp16x3") -> Tracker:
    """video01: T x 3 x H x W in [0, 1].  Runs the ViT stage in-process and hands its [T][P][C] output to a Tracker."""
    tpc = vit(video01)                                   # [T][P][C] on the GPU
    T, P, C = tpc.shape
    model = Tracker(video=video01.to(device), ckpt_path=ckpt_path, device=device, delta_channels=delta_channels,
                    corr_precision=corr_precision, dino_embed_video=torch.empty(0), _adopt_tpc=tpc)
    return model


@torch.no_grad()
def track_video(video01, vit: DinoV2Features, query_points, head_state_dict=None, delta_state_dict=None,
                device="cuda:0", anchor_th=0.7, cos_th=0.6, batch_size=None):
    """frames + query points -> (trajectories N x T x 2 px, occlusion N x T bool)."""
    model = build_tracker_from_video(video01, vit, device=device)
    if head_state_dict is not None:
        model.tracker_head.load_state_dict(head_state_dict)
    if delta_state_dict is not None:
        model.delta_dino.load_state_dict(delta_state_dict)
    mi = ModelInference(model, model.range_normalizer, anchor_th, cos_th)
    return mi.infer(query_points, batch_size)


@torch.no_grad()
def preprocess_best_buddies(features_chw, video01, dino_bb_dir, traj_path, h, w, stride=7, flow_fn=None, threshold=1.0,
                            min_trajectory_length=2, box_size=50, iou_thresh=0.2, device="cuda:0"):
    """preprocessing_dino_bb/main_dino_bb_preprocessing.py in one process: best buddies of the features (T x C x h' x w'),
    optical-flow trajectories of the video (T x 3 x h x w in [0, 1], no direct-flow filtering), the flow filter of the
    best buddies, then their NMS.  Features and trajectories stay on the GPU.  Writes the reference's three files:
    ``dino_bb_dir``/dino_best_buddies.pt, ``traj_path`` and ``dino_bb_dir``/dino_best_buddies_filtered.pt.  Returns
    (best buddies, trajectories, filtered best buddies)."""
    from . import best_buddies as bbm
    from .trajectories import extract_trajectories
    dev = torch.device(device)
    pk = bbm.PackedFeatures(features_chw, stride=stride, device=dev)
    bb = bbm.best_buddies(features_chw, h, w, stride=stride, device=dev)
    os.makedirs(dino_bb_dir, exist_ok=True)
    torch.save(bb, os.path.join(dino_bb_dir, "dino_best_buddies.pt"))
    traj = extract_trajectories(video01, flow_fn, threshold, min_trajectory_length, device=dev)
    os.makedirs(os.path.dirname(traj_path) or ".", exist_ok=True)
    torch.save(traj.cpu(), traj_path)
    filtered = bbm.nms_dict(bbm.of_filter(bb, traj, h, w, stride), pk, stride, box_size, iou_thresh)
    torch.save(filtered, os.path.join(dino_bb_dir, "dino_best_buddies_filtered.pt"))
    return bb, traj, filtered


@torch.no_grad()
def save_dino_embed_video(video01, vit: DinoV2Features, path):
    """preprocessing/save_dino_embed_video.py:9-25: writes T x C x h x w fp32 (CPU tensor) to ``path``."""
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    torch.save(vit.features_chw(video01).contiguous().cpu(), path)

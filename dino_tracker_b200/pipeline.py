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
    """video01: T x 3 x H x W in [0, 1].  Runs the ViT stage in-process and hands its [T][P][C] output to a Tracker with
    the backbone's patch and stride (the token centres: 8-pixel patches put them at 4 + 7 c, 14-pixel ones at 7 + 7 c)."""
    tpc = vit(video01)                                   # [T][P][C] on the GPU
    T, P, C = tpc.shape
    model = Tracker(video=video01.to(device), ckpt_path=ckpt_path, device=device, delta_channels=delta_channels,
                    corr_precision=corr_precision, dino_embed_video=torch.empty(0), _adopt_tpc=tpc,
                    dino_patch_size=vit.patch, stride=vit.stride)
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
                            min_trajectory_length=2, box_size=50, iou_thresh=0.2, device="cuda:0", flows=None):
    """preprocessing_dino_bb/main_dino_bb_preprocessing.py in one process: best buddies of the features (T x C x h' x w'),
    optical-flow trajectories of the video (T x 3 x h x w in [0, 1], no direct-flow filtering), the flow filter of the
    best buddies, then their NMS.  Features and trajectories stay on the GPU.  ``flows``: the consecutive flows
    (fwd, bwd, None) of ``trajectories.video_flows`` when already computed.  Writes the reference's three files:
    ``dino_bb_dir``/dino_best_buddies.pt, ``traj_path`` and ``dino_bb_dir``/dino_best_buddies_filtered.pt.  Returns
    (best buddies, trajectories, filtered best buddies)."""
    from . import best_buddies as bbm
    from .trajectories import extract_trajectories
    dev = torch.device(device)
    pk = bbm.PackedFeatures(features_chw, stride=stride, device=dev)
    bb = bbm.best_buddies(features_chw, h, w, stride=stride, device=dev)
    os.makedirs(dino_bb_dir, exist_ok=True)
    torch.save(bb, os.path.join(dino_bb_dir, "dino_best_buddies.pt"))
    traj = extract_trajectories(video01, flow_fn, threshold, min_trajectory_length, device=dev, flows=flows)
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


PREPROCESSING_DEFAULTS = dict(threshold=1.5, min_trajectory_length=2, filter_using_direct_flow=True, direct_flow_threshold=2.5,
                              fg_mask_threshold=0.6, dino_bb_box_size=30, dino_bb_iou_threshold=0.2)   # preprocessing.yaml


@torch.no_grad()
def preprocess_video(video01, vit: DinoV2Features, mask_vit: DinoV2Features, data_path, flow_fn=None, device="cuda:0",
                     **config):
    """preprocessing/main_preprocessing.py in one process, for a video T x 3 x H x W in [0, 1] and the paths of
    utils.add_config_paths(data_path):
      1. optical-flow trajectories -> of_trajectories/trajectories.pt;
      2. the features of ``vit`` -> dino_embeddings/dino_embed_video.pt;
      3. unless ``data_path``/masks exists: the features of ``mask_vit`` (layer 23 in the reference) go straight from the
         ViT into the mask kernels (no feature file) -> masks/{idx:05d}.jpg;
      4. the fg / bg split of the trajectories by the masks READ BACK from masks/ (JPEG is lossy, and ``> 0`` turns its
         ringing near mask edges into foreground; the re-read masks are what the trainer's load_fg_masks sees), resized
         to H x W -> of_trajectories/fg_trajectories.pt, bg_trajectories.pt;
      5. preprocess_best_buddies -> dino_best_buddies/*, of_trajectories/trajectories_wo_direct_filter.pt.
    A ``flow_fn`` with a ``video_flows`` method (``raft.RaftLarge``) encodes the frames once, and the consecutive flows
    of steps 1 and 5 are computed once.  ``config`` overrides PREPROCESSING_DEFAULTS.  Returns the trajectories, fg, bg and the masks [T][H][W] uint8."""
    from . import fg_masks as fgm
    from .trajectories import extract_trajectories, video_flows
    cfg = dict(PREPROCESSING_DEFAULTS, **config)
    dev = torch.device(device)
    T, _, H, W = video01.shape
    of_dir = os.path.join(data_path, "of_trajectories")
    os.makedirs(of_dir, exist_ok=True)
    flows = bb_flows = None
    if hasattr(flow_fn, "video_flows"):
        flows = video_flows(video01, flow_fn, cfg["filter_using_direct_flow"], device=dev)
        bb_flows = (flows[0], flows[1], None)
    traj = extract_trajectories(video01, flow_fn, cfg["threshold"], cfg["min_trajectory_length"],
                                cfg["filter_using_direct_flow"], cfg["direct_flow_threshold"], device=dev, flows=flows)
    torch.save(traj.cpu(), os.path.join(of_dir, "trajectories.pt"))
    features_chw = vit.features_chw(video01)
    os.makedirs(os.path.join(data_path, "dino_embeddings"), exist_ok=True)
    torch.save(features_chw.contiguous().cpu(), os.path.join(data_path, "dino_embeddings", "dino_embed_video.pt"))
    masks_path = os.path.join(data_path, "masks")
    if not os.path.exists(masks_path):
        tpc = mask_vit(video01)
        h, w = features_chw.shape[-2:]
        masks = fgm.fg_masks(tpc.view(T, h, w, tpc.shape[-1]), (H, W), fg_mask_threshold=cfg["fg_mask_threshold"])
        del tpc
        fgm.save_mask_frames(masks, masks_path)
    masks = torch.from_numpy(fgm.load_masks(masks_path, H, W)).to(dev)
    fg, bg = fgm.split_trajectories(traj, masks)
    torch.save(fg.cpu(), os.path.join(of_dir, "fg_trajectories.pt"))
    torch.save(bg.cpu(), os.path.join(of_dir, "bg_trajectories.pt"))
    preprocess_best_buddies(features_chw, video01, os.path.join(data_path, "dino_best_buddies"),
                            os.path.join(of_dir, "trajectories_wo_direct_filter.pt"), H, W, flow_fn=flow_fn,
                            threshold=cfg["threshold"], min_trajectory_length=cfg["min_trajectory_length"],
                            box_size=cfg["dino_bb_box_size"], iou_thresh=cfg["dino_bb_iou_threshold"], device=dev,
                            flows=bb_flows)
    return traj, fg, bg, masks

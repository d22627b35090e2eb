"""Optical-flow trajectories (``preprocessing/extract_trajectories.py``) over libdinotrk.

The flow network comes in through ``flow_fn(a, b)``: frames a, b [B][3][H][W] in [0, 1] -> flows a -> b [B][2][H][W].
The default is torchvision's RAFT (``raft_large``, as in the reference); ``raft.RaftLarge`` runs the same network on the
library, and as a provider with a ``video_flows`` method it encodes every frame once and batches the consecutive and
the direct pairs (``video_flows`` below).  Everything done with the flows runs in the library
(include/dinotrk.h: dinotrk_flow_masks, dinotrk_traj_chain / _emit): one thread walks one pixel through the frames,
and only the number of kept trajectories of each start frame is read back, to size its output.
"""
import ctypes
import os
from pathlib import Path

import torch

from . import _lib


def raft_flow_fn(device="cuda:0", num_flow_updates=24):
    """The reference's flow network: torchvision ``raft_large(weights=DEFAULT)``, frames replicate-padded to a multiple
    of 8 (``InputPadder``, sintel mode) and normalised by the weights' transforms, 24 updates."""
    from torchvision.models.optical_flow import Raft_Large_Weights, raft_large
    model = raft_large(weights=Raft_Large_Weights.DEFAULT, progress=False).to(device).eval()
    transforms = Raft_Large_Weights.DEFAULT.transforms()

    @torch.no_grad()
    def flow_fn(a, b):
        ht, wd = a.shape[-2:]
        ph, pw = (((ht // 8) + 1) * 8 - ht) % 8, (((wd // 8) + 1) * 8 - wd) % 8
        pad = [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]
        a, b = (torch.nn.functional.pad(x.to(device), pad, mode="replicate") for x in (a, b))
        a, b = transforms(a, b)
        f = model(a, b, num_flow_updates=num_flow_updates)[-1]
        return f[..., pad[2]:f.shape[-2] - pad[3], pad[0]:f.shape[-1] - pad[1]]
    return flow_fn


def _flow_video(fwd, bwd):
    fv = _lib.FlowVideo()
    fv.fwd, fv.bwd = fwd.data_ptr(), bwd.data_ptr()
    fv.T, fv.H, fv.W = fwd.shape[0] + 1, fwd.shape[2], fwd.shape[3]
    fv._keep = (fwd, bwd)
    return fv


def flow_masks(fwd, bwd, threshold=1.0):
    """get_flows_with_masks (extract_trajectories.py:74-95) on given flows [T-1][2][H][W]: masks [T+1][H][W] bool."""
    fwd, bwd = fwd.float().contiguous(), bwd.float().contiguous()
    T, H, W = fwd.shape[0] + 1, fwd.shape[2], fwd.shape[3]
    masks = torch.empty(T + 1, H, W, device=fwd.device, dtype=torch.uint8)
    with torch.cuda.device(fwd.device):
        _lib.check(_lib.load().dinotrk_flow_masks(ctypes.byref(_flow_video(fwd, bwd)), float(threshold), _lib.ptr(masks),
                                                  _lib.stream_ptr()), "flow_masks")
    return masks.bool()


@torch.no_grad()
def chain_trajectories(fwd, bwd, direct=None, threshold=1.0, min_trajectory_length=2, direct_flow_threshold=None):
    """extract_trajectories.py:195-266 on given flows: fwd / bwd [T-1][2][H][W] (CUDA), ``direct``: None or a callable
    s -> (flows s -> s+1+k, flows s+1+k -> s), each [T-1-s][2][H][W].  Returns [M][T][2] fp32, NaN where a trajectory
    does not exist, ordered by start frame, then row-major start pixel."""
    if int(min_trajectory_length) < 1:
        raise ValueError("min_trajectory_length must be >= 1")
    if direct is not None and direct_flow_threshold is None:
        raise ValueError("filtering with direct flows needs direct_flow_threshold")
    lib = _lib.load()
    dev = _lib.require_cuda(fwd.device)
    fwd, bwd = fwd.to(dev, torch.float32).contiguous(), bwd.to(dev, torch.float32).contiguous()
    T, H, W = fwd.shape[0] + 1, fwd.shape[2], fwd.shape[3]
    with torch.cuda.device(dev):
        fv = _flow_video(fwd, bwd)
        st = _lib.stream_ptr()
        masks = torch.empty(T + 1, H, W, device=dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_flow_masks(ctypes.byref(fv), float(threshold), _lib.ptr(masks), st), "flow_masks")
        nb = lib.dinotrk_traj_workspace_bytes(T, H, W)
        ws = torch.zeros(nb, device=dev, dtype=torch.uint8)       # the occupancy bitmap starts empty
        n_kept = torch.empty(1, device=dev, dtype=torch.int32)
        parts = []
        dthr = float(direct_flow_threshold) if direct is not None else 0.0
        for s in range(T - (int(min_trajectory_length) - 1)):
            dfwd = dbwd = None
            if direct is not None and s < T - 1:
                dfwd, dbwd = (x.to(dev, torch.float32).contiguous() for x in direct(s))
            _lib.check(lib.dinotrk_traj_chain(ctypes.byref(fv), _lib.ptr(masks), s, float(threshold), int(min_trajectory_length),
                                              _lib.ptr(dfwd), _lib.ptr(dbwd), dthr, _lib.ptr(n_kept), _lib.ptr(ws), nb, st),
                       "traj_chain")
            n = int(n_kept.item())                                  # the one read-back of the start frame
            if n == 0:
                continue
            out = torch.empty(n, T, 2, device=dev)
            _lib.check(lib.dinotrk_traj_emit(ctypes.byref(fv), s, _lib.ptr(out), _lib.ptr(ws), nb, st), "traj_emit")
            parts.append(out)
    return torch.cat(parts) if parts else torch.full((0, T, 2), float("nan"), device=dev)


@torch.no_grad()
def video_flows(video01, flow_fn=None, filter_using_direct_flow=False, device="cuda:0", direct_batch=16):
    """The flows ``extract_trajectories`` chains: (fwd, bwd, direct) with fwd / bwd [T-1][2][H][W] the consecutive flows
    and ``direct`` None or the callable s -> (flows s -> s+1+k, flows s+1+k -> s) of ``chain_trajectories``.  A provider
    with a ``video_flows(video01, groups)`` method (``raft.RaftLarge``) gets the consecutive pairs as one group and each
    start frame's direct pairs as one more, in chaining order; a plain ``flow_fn`` is called pair by pair as
    extract_trajectories.py does (the direct flows in batches of ``direct_batch``)."""
    dev = _lib.require_cuda(device)
    flow_fn = flow_fn or raft_flow_fn(dev)
    video01 = video01.to(dev, torch.float32)
    T = video01.shape[0]
    if hasattr(flow_fn, "video_flows"):
        groups = [[(i, i + 1) for i in range(T - 1)] + [(i + 1, i) for i in range(T - 1)]]
        if filter_using_direct_flow:
            groups += [[(s, t) for t in range(s + 1, T)] + [(t, s) for t in range(s + 1, T)] for s in range(T - 1)]
        it = flow_fn.video_flows(video01, groups)
        f = next(it)
        pending = iter(range(T - 1))

        def direct_provider(s):
            if next(pending) != s:
                raise RuntimeError("direct flows are produced in start-frame order")
            g = next(it)
            return g[:T - 1 - s], g[T - 1 - s:]
        return f[:T - 1], f[T - 1:], direct_provider if filter_using_direct_flow else None

    fwd, bwd = [], []
    for i in range(T - 1):
        pair = video01[i:i + 2]
        f = flow_fn(pair, pair.flip(0))                 # one batch: flow i -> i+1 and i+1 -> i (:63-65)
        fwd.append(f[0])
        bwd.append(f[1])
    fwd, bwd = torch.stack(fwd), torch.stack(bwd)

    def direct(s):
        src = video01[s:s + 1].expand(T - 1 - s, -1, -1, -1)
        dst = video01[s + 1:]
        ff, bf = [], []
        for i in range(0, T - 1 - s, direct_batch):
            ff.append(flow_fn(src[i:i + direct_batch], dst[i:i + direct_batch]))
            bf.append(flow_fn(dst[i:i + direct_batch], src[i:i + direct_batch]))
        return torch.cat(ff), torch.cat(bf)

    return fwd, bwd, direct if filter_using_direct_flow else None


@torch.no_grad()
def extract_trajectories(video01, flow_fn=None, threshold=1.0, min_trajectory_length=2, filter_using_direct_flow=False,
                         direct_flow_threshold=None, device="cuda:0", direct_batch=16, flows=None):
    """``save_trajectories`` of extract_trajectories.py:163-268 on a video [T][3][H][W] in [0, 1]: flows of consecutive
    frames (both directions), with ``filter_using_direct_flow`` the direct flows of every start frame to the later frames
    (``video_flows``), then the chaining.  ``flows``: the (fwd, bwd, direct) of ``video_flows`` when already computed.
    Returns [M][T][2] fp32 on ``device``."""
    if flows is None:
        flows = video_flows(video01, flow_fn, filter_using_direct_flow, device, direct_batch)
    fwd, bwd, direct = flows
    return chain_trajectories(fwd, bwd, direct if filter_using_direct_flow else None, threshold, min_trajectory_length,
                              direct_flow_threshold)


def load_frames(frames_path, infer_res_size=None):
    """The frames of a folder (*.jpg then *.png, sorted) as [T][3][H][W] in [0, 1]; ``infer_res_size`` (h, w): Lanczos
    resize as data_utils.resize_tensor_frames_lanczos."""
    import numpy as np
    from PIL import Image
    images = sorted(list(Path(frames_path).glob("*.jpg")) + list(Path(frames_path).glob("*.png")))
    frames = []
    for f in images:
        img = torch.from_numpy(np.array(Image.open(f)).astype(np.uint8)).permute(2, 0, 1).float() / 255
        if infer_res_size is not None:
            from torchvision import transforms
            pil = transforms.ToPILImage()(img).resize((infer_res_size[1], infer_res_size[0]), resample=Image.LANCZOS)
            img = transforms.ToTensor()(pil)
        frames.append(img)
    return torch.stack(frames)


def save_trajectories(args, flow_fn=None):
    """Drop-in for ``extract_trajectories.save_trajectories`` (same argparse namespace: frames_path, output_path,
    infer_res_size, threshold, min_trajectory_length, filter_using_direct_flow, direct_flow_threshold)."""
    video = load_frames(args.frames_path, args.infer_res_size)
    traj = extract_trajectories(video, flow_fn, args.threshold, args.min_trajectory_length, args.filter_using_direct_flow,
                                args.direct_flow_threshold)
    os.makedirs(os.path.dirname(args.output_path), exist_ok=True)
    torch.save(traj.cpu(), args.output_path)
    print(f"Saved {args.output_path}, shape: {traj.shape}")
    return traj

"""Foreground masks from DINO features (``preprocessing/create_fg_mask.py``) and the fg / bg split of the trajectories
(``preprocessing/split_trajectories_to_fg_bg.py``) over libdinotrk.

The reference runs ``torch.pca_lowrank(q, niter=20)`` on normalised, centred copies of the T*h*w x C layer-23 features.
Here the features stay as the ViT wrote them, token-major [M][C] fp32, and every pass over them is a library kernel
(include/dinotrk.h: dinotrk_pca_stats, dinotrk_pca_power, dinotrk_fg_mask): the row scales and the column mean are
applied on the fly, and one pass gives both ``X = Â P`` and ``W = Âᵀ X``, so that ``Âᵀ Q = W R⁻¹`` with ``Q R = X``.  The
small linear algebra (m x q and C x q QRs, the triangular solve, the q x C SVD) stays the ``torch.linalg`` calls of
``torch/_lowrank.py``, on the device, so signs follow the reference's conventions.
"""
import ctypes
import os
from pathlib import Path

import numpy as np
import torch

from . import _lib


def _token_major(feature_map):
    """(T, h, w, C) -> contiguous fp32 [T*h*w][C] on its device (a view when the input is already token-major)."""
    if feature_map.dim() == 3:
        feature_map = feature_map[None]
    return feature_map.reshape(-1, feature_map.shape[-1]).to(torch.float32).contiguous(), tuple(feature_map.shape[:3])


class PcaPasses:
    """The passes of the PCA over one feature matrix a [M][C] (CUDA, fp32, contiguous)."""

    def __init__(self, a, normalize=True):
        self.lib = _lib.load()
        self.a = a
        self.M, self.C = a.shape
        self.dev = a.device
        self.ws_bytes = self.lib.dinotrk_pca_workspace_bytes(self.M, self.C, 4)
        self.ws = torch.empty(self.ws_bytes, device=self.dev, dtype=torch.uint8)
        self.s = torch.empty(self.M, device=self.dev, dtype=torch.float32)
        self.c = torch.empty(self.C, device=self.dev, dtype=torch.float32)
        _lib.check(self.lib.dinotrk_pca_stats(_lib.ptr(a), self.M, self.C, 1 if normalize else 0, _lib.ptr(self.s),
                                              _lib.ptr(self.c), _lib.ptr(self.ws), self.ws_bytes, _lib.stream_ptr()),
                   "pca_stats")

    def power(self, P):
        """(X = Â P [M][q], W = Âᵀ X [C][q]) for P [C][q]."""
        q = P.shape[1]
        P = P.to(self.dev, torch.float32).contiguous()
        X = torch.empty(self.M, q, device=self.dev, dtype=torch.float32)
        W = torch.empty(self.C, q, device=self.dev, dtype=torch.float32)
        _lib.check(self.lib.dinotrk_pca_power(_lib.ptr(self.a), self.M, self.C, q, _lib.ptr(self.s), _lib.ptr(self.c),
                                              _lib.ptr(P), _lib.ptr(X), _lib.ptr(W), _lib.ptr(self.ws), self.ws_bytes,
                                              _lib.stream_ptr()), "pca_power")
        return X, W


def _adjoint_times_q(passes, P):
    """Âᵀ Q with Q = qr(Â P).Q, from one pass: W R⁻¹."""
    X, W = passes.power(P)
    R = torch.linalg.qr(X, mode="r").R
    return torch.linalg.solve_triangular(R, W, upper=True, left=False)


def pca_directions(passes, q, niter=20, R=None):
    """V [C][q] of ``torch.pca_lowrank(Â, q, niter)[2]`` (torch/_lowrank.py, m > n branch).  The random start R [C][q] is
    drawn as ``get_approximate_basis`` draws it (``torch.randn`` on the features' device) unless given."""
    if not 1 <= q <= 4:
        raise ValueError(f"q = {q}: the mask kernels take 1 <= q <= 4")
    if R is None:
        R = torch.randn(passes.C, q, dtype=torch.float32, device=passes.dev)
    Y = _adjoint_times_q(passes, R)                      # Âᵀ Q after Q = qr(Â R).Q
    for _ in range(niter):
        Y = _adjoint_times_q(passes, torch.linalg.qr(Y).Q)
    # B = Qᵀ Â = Yᵀ; U, S, Vh = svd(B); V = Vh.mH
    return torch.linalg.svd(Y.mT, full_matrices=False)[2].mH


@torch.no_grad()
def fg_masks(features, img_size, q=3, normalize=True, fg_mask_threshold=0.4, niter=20, R=None, return_all=False):
    """features: (T, h, w, C) on a CUDA device (``DinoV2Features.forward(...).view(T, h, w, C)`` is read in place).
    Returns the masks [T][H][W] uint8 0/255 on the device (``img_size`` = (H, W)); with ``return_all``, also
    (token mask [T][h][w] bool, V [C][q])."""
    dev = _lib.require_cuda(features.device)
    with torch.cuda.device(dev):
        a, (T, h, w) = _token_major(features)
        passes = PcaPasses(a, normalize)
        V = pca_directions(passes, q, niter, R).contiguous()
        H, W = int(img_size[0]), int(img_size[1])
        colors = torch.empty(a.shape[0], q, device=dev, dtype=torch.float32)
        tm = torch.empty(T, h, w, device=dev, dtype=torch.uint8)
        out = torch.empty(T, H, W, device=dev, dtype=torch.uint8)
        ws = torch.empty(256, device=dev, dtype=torch.uint8)
        _lib.check(passes.lib.dinotrk_fg_mask(_lib.ptr(a), T, h, w, a.shape[1], q, _lib.ptr(passes.s), _lib.ptr(V),
                                              float(fg_mask_threshold), H, W, _lib.ptr(colors), _lib.ptr(tm), _lib.ptr(out),
                                              _lib.ptr(ws), 256, _lib.stream_ptr()), "fg_mask")
    return (out, tm.bool(), V) if return_all else out


def upsample_mask(token_mask, size):
    """F.interpolate(token_mask[None].float(), size, mode="nearest") of a [T][h][w] 0/1 mask, as [T][H][W] uint8 0/255."""
    dev = _lib.require_cuda(token_mask.device)
    tm = token_mask.to(torch.uint8).contiguous()
    T, h, w = tm.shape
    out = torch.empty(T, int(size[0]), int(size[1]), device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().dinotrk_mask_upsample(_lib.ptr(tm), T, h, w, out.shape[1], out.shape[2], _lib.ptr(out),
                                                     _lib.stream_ptr()), "mask_upsample")
    return out


def get_fg_mask_from_pca(feature_map, img_size, q=3, interpolation="nearest", normalize=True, fg_mask_threshold=0.4):
    """Drop-in for create_fg_mask.py:11-43: feature_map (T, h, w, C) or (h, w, C) on a CUDA device -> numpy float32
    (T, H, W) of 0 / 1.  A non-token-major input (the reference passes a permuted view) gets one contiguous copy."""
    if interpolation != "nearest":
        raise ValueError(f"interpolation={interpolation!r}: only 'nearest' is supported")
    m = fg_masks(feature_map, img_size, q=q, normalize=normalize, fg_mask_threshold=fg_mask_threshold)
    return (m > 0).float().cpu().numpy()


def save_mask_frames(masks, mask_path):
    """{idx:05d}.jpg per frame of masks [T][H][W] uint8 (the reference's save_video_frames; PIL's JPEG encoder)."""
    from PIL import Image
    path = Path(mask_path)
    path.mkdir(exist_ok=True, parents=True)
    for idx, frame in enumerate(masks.cpu().numpy()):
        Image.fromarray(frame).save(path / f"{idx:05d}.jpg")
    return path


@torch.no_grad()
def run(args):
    """Drop-in for create_fg_mask.py:51-60 (args: dino_embed_video_path, h, w, mask_path, q, fg_mask_threshold)."""
    dino_embed_video = torch.load(args.dino_embed_video_path, map_location="cuda:0")    # T x C x h x w
    masks = fg_masks(dino_embed_video.permute(0, 2, 3, 1), (args.h, args.w), q=args.q,
                     fg_mask_threshold=args.fg_mask_threshold)
    frames_path = save_mask_frames(masks, args.mask_path)
    print(f"Saved fg. mask to {frames_path}")


# ---- split_trajectories_to_fg_bg.py -----------------------------------------------------------------------------------
@torch.no_grad()
def split_trajectories(traj, masks):
    """traj [N][T][2] fp32 (NaN where missing), masks [Tm][H][W] (> 0 = foreground), both on one CUDA device ->
    (fg, bg): the trajectories whose rounded first valid position lies on the mask, and the others, in order.
    Raises DinotrkError when a trajectory has no valid step or starts outside the masks."""
    dev = _lib.require_cuda(traj.device)
    lib = _lib.load()
    traj = traj.to(dev, torch.float32).contiguous()
    masks = masks.to(dev, torch.uint8).contiguous()
    N, T = traj.shape[0], traj.shape[1]
    if N == 0:
        return traj.clone(), traj.clone()
    Tm, H, W = masks.shape
    with torch.cuda.device(dev):
        nb = lib.dinotrk_traj_split_workspace_bytes(N)
        ws = torch.empty(nb, device=dev, dtype=torch.uint8)
        st = _lib.stream_ptr()
        n_fg = ctypes.c_int(0)
        _lib.check(lib.dinotrk_traj_split_count(_lib.ptr(traj), N, T, _lib.ptr(masks), Tm, H, W, ctypes.byref(n_fg),
                                                _lib.ptr(ws), nb, st), "traj_split_count")
        fg = torch.empty(n_fg.value, T, 2, device=dev)
        bg = torch.empty(N - n_fg.value, T, 2, device=dev)
        _lib.check(lib.dinotrk_traj_split_emit(_lib.ptr(traj), N, T, _lib.ptr(fg) if fg.numel() else None,
                                               _lib.ptr(bg) if bg.numel() else None, _lib.ptr(ws), nb, st), "traj_split_emit")
    return fg, bg


def load_masks(masks_path, h_resize=476, w_resize=854):
    """split_trajectories_to_fg_bg.py:38-52: the *.jpg then *.png files of a folder (sorted), grayscale, nearest-resized
    -> numpy uint8 [T][h_resize][w_resize]."""
    from PIL import Image
    from torch.nn.functional import interpolate
    files = sorted(list(Path(masks_path).glob("*.jpg")) + list(Path(masks_path).glob("*.png")))
    masks = np.stack([np.array(Image.open(f).convert("L")) for f in files])
    h_resize = masks.shape[1] if h_resize is None else h_resize
    w_resize = masks.shape[2] if w_resize is None else w_resize
    masks = interpolate(torch.from_numpy(masks).unsqueeze(1), size=(h_resize, w_resize), mode="nearest")
    return masks[:, 0].numpy()


def mask_filter_trajectories(traj_path, masks_path, out_path, filter_bg=False, device="cuda:0"):
    """split_trajectories_to_fg_bg.py:55-78: writes the fg (or, with ``filter_bg``, the bg) trajectories of
    ``traj_path`` to ``out_path`` (CPU tensor)."""
    traj = torch.load(traj_path, map_location="cpu")
    masks = torch.from_numpy(load_masks(masks_path)).to(device)
    fg, bg = split_trajectories(traj.to(device), masks)
    out = (bg if filter_bg else fg).cpu()
    torch.save(out, out_path)
    print(f"Saved {out_path}, shape: {out.shape}")
    return out


def split_trajectories_to_fg_bg(args, device="cuda:0"):
    """split_trajectories_to_fg_bg.py:80-82 (args: traj_path, fg_masks_path, fg_traj_path, bg_traj_path), with one
    classification for both files."""
    traj = torch.load(args.traj_path, map_location="cpu")
    masks = torch.from_numpy(load_masks(args.fg_masks_path)).to(device)
    fg, bg = split_trajectories(traj.to(device), masks)
    for t, p in ((fg, args.fg_traj_path), (bg, args.bg_traj_path)):
        os.makedirs(os.path.dirname(p) or ".", exist_ok=True)
        torch.save(t.cpu(), p)
        print(f"Saved {p}, shape: {t.shape}")
    return fg, bg

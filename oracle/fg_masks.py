"""Plain-torch, device-agnostic restatement of the foreground masks (``preprocessing/create_fg_mask.py:11-43``) and of
the fg / bg split of the trajectories (``preprocessing/split_trajectories_to_fg_bg.py:9-78``), plus the seeded inputs
of their tests."""
import numpy as np
import torch
import torch.nn.functional as F


def fg_mask_tokens(feature_map, q=3, normalize=True, fg_mask_threshold=0.4):
    """create_fg_mask.py:22-35: feature_map (T, h, w, C) or (h, w, C) -> (token mask (T, h, w) bool, V [C][q],
    normalised first component (M,)).  Runs torch.pca_lowrank (q, niter=20) as the reference does: the random start
    is drawn from the default generator of the features' device."""
    if len(feature_map.shape) == 3:
        feature_map = feature_map[None]                                          # :22-24
    if normalize:
        feature_map = F.normalize(feature_map, dim=-1)                           # :25-26
    features = feature_map.reshape(-1, feature_map.shape[-1])                    # :27
    reduction_mat = torch.pca_lowrank(features, q=q, niter=20)[2]                # :28
    colors = features @ reduction_mat                                            # :29
    colors_min = colors.min(dim=0).values                                        # :31-33
    colors_max = colors.max(dim=0).values
    tmp_colors = (colors - colors_min) / (colors_max - colors_min)
    fg_mask = tmp_colors[..., 0] < fg_mask_threshold                             # :34
    return fg_mask.reshape(feature_map.shape[:3]), reduction_mat, tmp_colors[..., 0]


def get_fg_mask_from_pca(feature_map, img_size, q=3, interpolation="nearest", normalize=True, fg_mask_threshold=0.4):
    """create_fg_mask.py:11-43: numpy float32 (T, H, W) of 0 / 1."""
    fg_mask, _, _ = fg_mask_tokens(feature_map, q, normalize, fg_mask_threshold)
    fg_mask = F.interpolate(fg_mask.unsqueeze(0).float(), size=img_size, mode=interpolation).squeeze(0)   # :37-41
    return fg_mask.cpu().numpy()


def pca_directions_from(A, R, niter=20):
    """torch/_lowrank.py pca_lowrank(A, q, center=True, niter)[2] (m > n branch) from a given random start R [n][q], in
    A's dtype: get_approximate_basis on A - mean, B = Qᵀ Â, V = svd(B).Vh.mH."""
    A = A - A.mean(dim=-2, keepdim=True)
    Q = torch.linalg.qr(A @ R).Q
    for _ in range(niter):
        Q = torch.linalg.qr(A.mH @ Q).Q
        Q = torch.linalg.qr(A @ Q).Q
    return torch.linalg.svd(Q.mH @ A, full_matrices=False)[2].mH


def first_steps(trajectories):
    """split_trajectories_to_fg_bg.py:9-35 + :67 (generate_start_end, argmax of the first-step mask): the index of each
    trajectory's first step with no NaN coordinate (0 for a trajectory without one)."""
    mask = trajectories.isnan().any(dim=-1)
    mask_shifted_right = mask.roll(1, dims=1)
    mask_shifted_right[:, 0] = True
    first_timestep_mask = ~mask & mask_shifted_right
    return first_timestep_mask.int().argmax(dim=1)


def mask_filter(trajectories, masks, filter_bg=False):
    """split_trajectories_to_fg_bg.py:62-76 on tensors: trajectories [N][T][2], masks [Tm][H][W] on one device -> the
    trajectories whose rounded start position is on the mask (> 0), or off it (== 0) with ``filter_bg``."""
    start_indices = first_steps(trajectories)
    traj_start_points = trajectories[torch.arange(trajectories.shape[0], device=trajectories.device), start_indices].round().int()
    masks_at_start = masks[start_indices, traj_start_points[:, 1], traj_start_points[:, 0]]
    is_valid_traj = masks_at_start == 0 if filter_bg else masks_at_start > 0
    return trajectories[is_valid_traj]


# ---- seeded inputs ------------------------------------------------------------------------------------------------
def planted_features(T, h, w, C, seed, noise=0.3, radius=0.25, device="cpu"):
    """(features (T, h, w, C) fp32, planted foreground (T, h, w) bool): a disc of radius ``radius`` * min(h, w) moving
    across the frames; foreground and background tokens are two random unit directions, plus two more random unit
    directions with Gaussian weights of std 0.3 and 0.15 per token (so that the top three principal directions are well
    separated), plus Gaussian noise of ``noise`` per channel (times 1 / sqrt(C)), times a random positive scale per
    token.  Generated frame by frame on
    ``device`` from a generator of that device, so large videos never exist on the host."""
    g = torch.Generator(device=device).manual_seed(seed)
    mu = F.normalize(torch.randn(4, C, generator=g, device=device), dim=-1)
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=device),
                            torch.arange(w, dtype=torch.float32, device=device), indexing="ij")
    feats = torch.empty(T, h, w, C, device=device)
    plant = torch.empty(T, h, w, dtype=torch.bool, device=device)
    r = radius * min(h, w)
    for t in range(T):
        cx = r + (w - 2 * r) * (t + 0.5) / T
        cy = h / 2 + (h / 2 - r) * 0.5 * np.sin(2 * np.pi * t / max(T, 2))
        fg = (xx - cx) ** 2 + (yy - cy) ** 2 <= r * r
        x = torch.where(fg[..., None], mu[0], mu[1]) + noise / np.sqrt(C) * torch.randn(h, w, C, generator=g, device=device)
        k = torch.randn(h, w, 2, generator=g, device=device) * torch.tensor([0.3, 0.15], device=device)
        x = x + k[..., :1] * mu[2] + k[..., 1:] * mu[3]
        feats[t] = x * (0.5 + torch.rand(h, w, 1, generator=g, device=device))
        plant[t] = fg
    return feats, plant


def split_case_inputs(N, T, H, W, seed):
    """(trajectories [N][T][2], masks [T][H][W] uint8): chain-style rows (NaN, then a run of valid steps, then NaN; a
    start step never NaN in one coordinate only), start positions on a half-pixel lattice (exact .5 ties for
    torch.round), later steps anywhere in the frame; masks of random discs with values 0, 1, 128 and 255."""
    g = torch.Generator().manual_seed(seed)
    traj = torch.full((N, T, 2), float("nan"))
    start = torch.randint(0, T, (N,), generator=g)
    length = torch.randint(1, T + 1, (N,), generator=g)
    pos = torch.rand(N, T, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    pos[:, :, 0] = (pos[:, :, 0] * 2).round() / 2
    pos[:, :, 1] = (pos[:, :, 1] * 2).round() / 2
    t = torch.arange(T)[None]
    valid = (t >= start[:, None]) & (t < (start + length).clamp(max=T)[:, None])
    traj[valid] = pos[valid]
    half = torch.rand(N, T, generator=g) < 0.05                      # NaN in one coordinate only, after the start
    half &= valid & (t > start[:, None])
    traj[..., 1][half] = float("nan")
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    masks = torch.zeros(T, H, W, dtype=torch.uint8)
    for k in range(T):
        for _ in range(3):
            c = torch.rand(2, generator=g) * torch.tensor([W, H])
            r = float(torch.rand(1, generator=g)) * min(H, W) / 3 + 4
            v = [1, 128, 255][int(torch.randint(0, 3, (1,), generator=g))]
            masks[k][(xx - c[0]) ** 2 + (yy - c[1]) ** 2 <= r * r] = v
    return traj, masks

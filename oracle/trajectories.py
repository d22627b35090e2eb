"""Device-agnostic PyTorch restatement of ``preprocessing/extract_trajectories.py`` on given flows.

Test infrastructure (see ``oracle/__init__.py``).  The reference computes the flows with RAFT inside the same
functions; here they come in as tensors so that tests can pass synthetic ones:
  fwd, bwd: [T-1][2][H][W]  flows frame i -> i+1 and i+1 -> i (``get_flows_with_masks``, :61-73);
  direct(s) -> (dfwd, dbwd) [T-1-s][2][H][W] flows s -> s+1+k and s+1+k -> s (``compute_direct_flows_for_start_frame``,
  :128-141).
Everything after the flows follows the reference op for op; the result is the ``[M][T][2]`` tensor it saves.
"""
import torch
import torch.nn.functional as F


def coords_grid(h, w, device):
    """data/data_utils.py:55-58 (one batch, channels last): [h][w][2] = (x, y)."""
    ys, xs = torch.meshgrid(torch.arange(h, device=device), torch.arange(w, device=device), indexing="ij")
    return torch.stack((xs, ys), dim=-1).float()


def bilinear_sampler(img, coords):
    """data/data_utils.py:62-76: img [1][C][H][W], coords [1][h][w][2] pixels -> [1][C][h][w]."""
    H, W = img.shape[-2:]
    xgrid, ygrid = coords.split([1, 1], dim=-1)
    xgrid = 2 * xgrid / (W - 1) - 1
    ygrid = 2 * ygrid / (H - 1) - 1
    return F.grid_sample(img, torch.cat([xgrid, ygrid], dim=-1), align_corners=True, mode="bilinear")


def bilinear_interpolate_video(video, points, h, w, t):
    """utils.py:75-101 with normalize_h = normalize_w = normalize_t = True."""
    samples = points[None, None, :, None].clone()
    samples[..., 0] = samples[..., 0] / (w - 1)
    samples[..., 0] = samples[..., 0] * 2 - 1
    samples[..., 1] = samples[..., 1] / (h - 1)
    samples[..., 1] = samples[..., 1] * 2 - 1
    if t > 1:
        samples[..., 2] = samples[..., 2] / (t - 1)
    samples[..., 2] = samples[..., 2] * 2 - 1
    return F.grid_sample(video, samples, align_corners=True, padding_mode="border")


def flow_masks(fwd, bwd, threshold=1.0):
    """extract_trajectories.py:74-95: masks [T+1][h][w][1] bool."""
    T1, _, h, w = fwd.shape
    dev = fwd.device
    upper_bound = torch.tensor([[w, h]], device=dev) - 1
    err_array = torch.zeros((T1 + 2, h, w), device=dev)
    missing_forward_warp = torch.ones((T1 + 2, h, w), device=dev, dtype=torch.bool)
    coords = coords_grid(h, w, dev)[None]
    for idx in range(T1):
        flow12, flow21 = fwd[idx:idx + 1], bwd[idx:idx + 1]
        coords1 = coords + flow21.permute(0, 2, 3, 1)
        coords2 = coords1 + bilinear_sampler(flow12, coords1).permute(0, 2, 3, 1)
        err_array[idx + 1] = (coords - coords2).norm(dim=3)
        g = (coords + flow12.permute(0, 2, 3, 1)).round().long().flatten(0, -2)
        g = g[((g >= 0) & (g <= upper_bound)).all(dim=-1)]
        missing_forward_warp[idx + 1, g[:, 1], g[:, 0]] = False
    masks = err_array.unsqueeze(-1) < threshold
    masks[0] = False
    masks = masks & ~missing_forward_warp.unsqueeze(-1)
    masks[0] = False
    return masks


def direct_flow_masks(dfwd, dbwd, threshold=1.0):
    """extract_trajectories.py:142-160 on given direct flows: (positions [D][h][w][2], mask [D][h][w] float32)."""
    D, _, h, w = dfwd.shape
    dev = dfwd.device
    upper_bound = torch.tensor([[w, h]], device=dev) - 1
    coords = coords_grid(h, w, dev)[None].repeat(D, 1, 1, 1)
    forward_flows = dfwd.permute(0, 2, 3, 1)
    coords1 = coords + forward_flows
    time_grid = torch.arange(D, device=dev)[:, None, None, None].repeat(1, h, w, 1)
    coords1_3d = torch.cat((coords1, time_grid), dim=-1).reshape(-1, 3)
    back = bilinear_interpolate_video(dbwd.permute(1, 0, 2, 3)[None], coords1_3d, h=h, w=w, t=D)
    back = back.squeeze().permute(1, 0).reshape((D, h, w, 2))
    err = (coords - (coords1 + back)).norm(dim=-1)
    mask = (err < threshold) & ((coords1 >= 0) & (coords1 <= upper_bound)).all(dim=-1)
    return forward_flows, mask.to(torch.float32)


def extract_trajectories(fwd, bwd, direct=None, threshold=1.0, min_trajectory_length=2, direct_flow_threshold=None):
    """extract_trajectories.py:195-266 (look-behind on).  ``direct``: None, or a callable s -> (dfwd, dbwd)."""
    T = fwd.shape[0] + 1
    h, w = fwd.shape[-2:]
    dev = fwd.device
    masks = flow_masks(fwd, bwd, threshold)
    upper_bound = torch.tensor([w, h], device=dev) - 1
    lower_bound = torch.tensor([0, 0], device=dev)
    kept = torch.full((0, T, 2), float("nan"), device=dev)
    for s in range(T - (min_trajectory_length - 1)):
        traj = torch.zeros((T - s, h, w, 2), device=dev)
        coords = coords_grid(h, w, dev)[None]
        orig_coords = coords.clone()
        mask = ~masks[s]
        past = kept[:, s]
        past = past[past.isnan().any(dim=-1).logical_not()].round().long()
        past = past[((past >= 0) & (past <= upper_bound)).all(dim=-1)]
        not_passed_through = torch.ones_like(mask)
        not_passed_through[past[:, 1], past[:, 0]] = False
        mask |= not_passed_through
        traj[0] = torch.where(mask, coords.double(), float("nan"))
        if direct is not None:
            dflows, dmasks = direct_flow_masks(*direct(s), threshold)
        for idx in range(T - 1 - s):
            flow12, flow21 = fwd[s + idx:s + idx + 1], bwd[s + idx:s + idx + 1]
            warped = bilinear_sampler(flow12, coords).permute(0, 2, 3, 1)
            coords1 = coords + warped
            coords2 = coords1 + bilinear_sampler(flow21, coords1).permute(0, 2, 3, 1)
            err = (coords - coords2).norm(dim=3)
            mask = mask & (err.unsqueeze(-1) < threshold) & (coords1 <= upper_bound) & (coords1 >= lower_bound)
            coords += warped
            if direct is not None:
                err_d = (coords - (orig_coords + dflows[idx].unsqueeze(0))).norm(dim=3)
                err_d = err_d * (dmasks[idx] > 0.2).float()
                mask = mask & (err_d.unsqueeze(-1) < direct_flow_threshold)
            traj[idx + 1] = torch.where(mask, coords.double(), float("nan"))
        padded = F.pad(traj.permute(1, 2, 3, 0), (s, 0), mode="constant", value=float("nan"))
        padded = padded.permute(0, 1, 3, 2).reshape(h * w, T, 2)
        padded[padded.isnan().any(dim=-1)[..., None].expand(-1, -1, 2)] = float("nan")
        kept = torch.cat([kept, padded[padded.isnan().any(dim=-1).logical_not().sum(dim=-1) >= min_trajectory_length]])
    return kept


def smooth_flows(T, H, W, seed, amplitude=3.0, integer=False, device="cpu", noise=True):
    """Seeded flows for tests: a smooth random motion field per frame (low-frequency cosines; with ``noise``, per-pixel
    noise on about half of the frames), forward and backward flows of every ordered frame pair from it.  Per-pixel noise
    amplifies last-bit differences along a walk; tests that compare positions with a tolerance use ``noise=False``.
    ``integer``: whole-pixel values, |v| <= 4;
    walks then stay on the pixel lattice and, for H - 1 and W - 1 powers of two, every sample, sum and norm is exact in
    fp32, so any two correct implementations agree bit for bit.
    Returns flow(a, b) -> [2][H][W] on ``device``: the flow from frame a to frame b."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    fields = []
    for _ in range(T):
        f = torch.zeros(2, H, W, dtype=torch.float64)
        for c in range(2):
            for _k in range(3):
                a, fx, fy, ph = torch.rand(4, generator=g, dtype=torch.float64).tolist()
                f[c] += amplitude * (a - 0.5) * torch.cos(2 * torch.pi * (fx * xs / W * 2 + fy * ys / H * 2) + 6.3 * ph)
        if noise:
            f = f + 0.25 * amplitude * (torch.rand(2, H, W, generator=g, dtype=torch.float64) - 0.5) * (torch.rand(1, generator=g).item() < 0.5)
        fields.append(f)
    cache = {}

    def flow(a, b):
        if (a, b) not in cache:
            v = fields[b] - fields[a]
            v = v.clamp(-4, 4).round() if integer else v
            cache[(a, b)] = v.float().to(device)
        return cache[(a, b)]
    return flow


def stack_flows(flow, T):
    """Consecutive forward / backward flows [T-1][2][H][W] and the direct-flow callable of ``extract_trajectories``."""
    fwd = torch.stack([flow(i, i + 1) for i in range(T - 1)])
    bwd = torch.stack([flow(i + 1, i) for i in range(T - 1)])

    def direct(s):
        return (torch.stack([flow(s, s + 1 + k) for k in range(T - 1 - s)]),
                torch.stack([flow(s + 1 + k, s) for k in range(T - 1 - s)]))
    return fwd, bwd, direct

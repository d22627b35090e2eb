"""Device-agnostic PyTorch restatement of ``preprocessing_dino_bb/of_filter_dino_best_buddies.py``.

Test infrastructure (see ``oracle/__init__.py``).  ``of_filter`` is ``run`` (:36-112) on in-memory inputs: the best-buddy
dict and the ``[M][T][2]`` trajectories in, the filtered dict out.
"""
import torch


def create_meshgrid(h, w, step=7, patch_size=14, device="cpu"):
    """preprocessing_dino_bb/dino_bb_utils.py:5-15 with return_hw: (grid [G][2] (x, y), rows, columns)."""
    x = torch.arange(patch_size // 2, w, step=step, device=device).float()
    y = torch.arange(patch_size // 2, h, step=step, device=device).float()
    yy, xx = torch.meshgrid(y, x, indexing="ij")
    return torch.stack([xx.reshape(-1), yy.reshape(-1)], dim=-1), len(y), len(x)


def closest_traj_idx(trajectories, points, t, batch_size=30):
    """get_closest_traj_idx_batch (:9-29)."""
    at_t = trajectories[:, t, :]
    out = []
    for i in range(0, len(points), batch_size):
        d = torch.norm(at_t[None, ...] - points[i:i + batch_size][:, None, :], dim=2)
        out.append(torch.nan_to_num(d, nan=torch.inf).argmin(dim=-1))
    return torch.cat(out, dim=0)


def nearest_grid(traj, h, w, stride):
    """:51-56: [T][rows][columns] index of the nearest trajectory of every grid point."""
    grid, gh, gw = create_meshgrid(h, w, step=stride, device=traj.device)
    return torch.stack([closest_traj_idx(traj, grid, t).reshape(gh, gw) for t in range(traj.shape[1])])


def of_filter(bb_data, traj, h, w, stride=7):
    """:45-108."""
    nearest = nearest_grid(traj, h, w, stride)
    invalid = traj.isnan().any(dim=-1)
    T = traj.shape[1]
    out = {}
    for s in range(T):
        for t in range(T):
            if s == t:
                continue
            bb = bb_data[f"{s}_{t}"]
            src, tgt = bb["source_coords"], bb["target_coords"]
            sg = ((src - 7) // stride).long()
            tg = ((tgt - 7) // stride).long()
            si = nearest[s][sg[:, 1], sg[:, 0]]
            ti = nearest[t][tg[:, 1], tg[:, 0]]
            keep = (invalid[si, t] & invalid[ti, s]).to(src.device)
            any_ = bool(keep.any())
            f = {k: None for k in ("source_coords", "target_coords", "cos_sims", "peak_coords", "peak_affs", "r")}
            for k in f:
                if bb.get(k, None) is not None and any_:
                    f[k] = bb[k][keep]
            out[f"{s}_{t}"] = f
    return out

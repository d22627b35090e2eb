"""Plain-torch restatement of the training-batch sampler, ``data/dataset.py:56-258`` (``LongRangeSampler`` and
``DinoTrackerSampler``), for any device.

It makes the reference's random draws with the same torch calls, arguments and order, on the device of the sampled
set, so that a seeded run gives the reference's samples bit for bit:
  per set (fg, then bg): ``randperm(T)[:num_frames]`` until at least 2 trajectories are candidates
  (``dataset.py:167-175``), ``randperm(n)[:batch]`` (``:177``), ``multinomial(2, replacement=False)`` (``:183``).
The frame-set mapping keeps the reference's per-point ``.nonzero()`` loops (``:240-241``).  The windowed mode
(``keep_in_cpu``) samples from windows of ``MAX_TRAJ_SIZE`` valid trajectories moved to ``window_device`` (the
reference's ``.cuda()``; default: the trajectories' own device), advanced by ``load_next_batch`` (``:108-131``).
"""
import math

import torch

MAX_TRAJ_SIZE = 200_000


def get_valid_trajectories(trajectories):
    """dataset.py:100-106: the rows with more than one step where neither coordinate is NaN, and their [N'][T] mask."""
    can_sample = ~trajectories.isnan().any(dim=-1)
    keep = can_sample.sum(dim=1) > 1
    return trajectories[keep], can_sample[keep]


def point_correspondences(valid, can_sample, num_frames, batch_size, frame_draws=None):
    """dataset.py:162-190: (t1_points, t2_points) [min(batch, n)][3] = (x, y, t) of one set.  ``frame_draws`` (a list)
    gets the number of frame draws the call made."""
    T, dev = valid.shape[1], valid.device
    draws = 0
    while True:
        draws += 1
        frame_indices = torch.arange(T, device=dev)[torch.randperm(T, device=dev)[:num_frames]]
        candidates = can_sample.float()[:, frame_indices].sum(dim=1) >= 2
        rows = candidates.nonzero()[:, 0]
        if rows.shape[0] >= 2:
            break
    if frame_draws is not None:
        frame_draws.append(draws)
    rows = rows[torch.randperm(rows.shape[0], device=dev)[:batch_size]]
    weights = torch.zeros(rows.shape[0], T, dtype=torch.bool, device=dev)
    weights[:, frame_indices] = can_sample[rows][:, frame_indices]
    t1, t2 = weights.float().multinomial(2, replacement=False).unbind(dim=1)
    p1 = torch.cat([valid[rows, t1], t1.unsqueeze(-1)], dim=-1)
    p2 = torch.cat([valid[rows, t2], t2.unsqueeze(-1)], dim=-1)
    return p1, p2


class LongRangeSampler(torch.nn.Module):
    def __init__(self, batch_size, fg_trajectories=None, bg_trajectories=None, fg_traj_ratio=0.5, num_frames=None,
                 keep_in_cpu=False, window_device=None):
        super().__init__()
        self.batch_size, self.num_frames, self.fg_traj_ratio = batch_size, num_frames, fg_traj_ratio
        self.keep_in_cpu = keep_in_cpu
        self.gpu_batch_index = 0
        self.frame_draws = []
        self.sets = {}
        for name, traj in (("fg", fg_trajectories), ("bg", bg_trajectories)):
            valid, can = get_valid_trajectories(traj)
            s = {"valid": valid, "can": can}
            if keep_in_cpu:
                s["device"] = window_device or traj.device
                s["n_batches"] = math.ceil(valid.shape[0] / MAX_TRAJ_SIZE)
                self._load_window(s, 0)
            else:
                s["window"] = (valid, can)
            self.sets[name] = s

    @staticmethod
    def _load_window(s, index):
        start, end = index * MAX_TRAJ_SIZE, min((index + 1) * MAX_TRAJ_SIZE, s["valid"].shape[0])
        s["window"] = (s["valid"][start:end].to(s["device"]), s["can"][start:end].to(s["device"]))

    def load_next_batch(self):
        if not self.keep_in_cpu:
            return
        self.gpu_batch_index += 1
        for s in self.sets.values():
            self._load_window(s, self.gpu_batch_index % s["n_batches"])

    def get_fg_batch_size(self):
        return int(self.batch_size * self.fg_traj_ratio)

    def forward(self):
        assert self.num_frames is not None, "num_frames must be specified"
        fg_batch = self.get_fg_batch_size()
        fg = point_correspondences(*self.sets["fg"]["window"], self.num_frames, fg_batch, self.frame_draws)
        bg = point_correspondences(*self.sets["bg"]["window"], self.num_frames, self.batch_size - fg_batch, self.frame_draws)
        return torch.cat([fg[0], bg[0]], dim=0), torch.cat([fg[1], bg[1]], dim=0)


class DinoTrackerSampler(LongRangeSampler):
    def __init__(self, batch_size, range_normalizer, dst_range, fg_trajectories=None, bg_trajectories=None,
                 fg_traj_ratio=0.5, num_frames=None, keep_in_cpu=False, window_device=None):
        super().__init__(batch_size, fg_trajectories=fg_trajectories, bg_trajectories=bg_trajectories,
                         fg_traj_ratio=fg_traj_ratio, num_frames=num_frames, keep_in_cpu=keep_in_cpu,
                         window_device=window_device)
        self.range_normalizer = range_normalizer
        self.dst_range = dst_range

    def forward(self):
        """dataset.py:233-258."""
        t1_points, t2_points = super().forward()
        frames_set_t = torch.cat((t1_points[:, 2], t2_points[:, 2])).unique().int()
        source_frame_indices = torch.cat([(frames_set_t == i).nonzero() for i in t1_points[:, 2]])[:, 0]
        target_frame_indices = torch.cat([(frames_set_t == i).nonzero() for i in t2_points[:, 2]])[:, 0]
        t1_points_normalized = self.range_normalizer(t1_points, dst=self.dst_range)
        t2_points_normalized = self.range_normalizer(t2_points, dst=self.dst_range)
        t1_points[:, 2] = t1_points_normalized[:, 2]
        return {"frames_set_t": frames_set_t, "source_frame_indices": source_frame_indices,
                "target_frame_indices": target_frame_indices, "t1_points_normalized": t1_points_normalized,
                "t2_points_normalized": t2_points_normalized, "t1_points": t1_points, "target_times": t2_points[:, 2]}


class RangeNormalizer(torch.nn.Module):
    """dataset.py:5-37 (forward only): x[:, dims] / (shape - 1), then (dst[1] - dst[0]) * . + dst[0]."""

    def __init__(self, shapes, device="cpu"):
        super().__init__()
        self.register_buffer("normalizer", torch.tensor(shapes).float().to(device) - 1)

    def forward(self, x, dst=(0, 1), dims=[0, 1, 2]):
        out = x.clone()
        out[:, dims] = x[:, dims] / self.normalizer[dims]
        out[:, dims] = (dst[1] - dst[0]) * out[:, dims] + dst[0]
        return out

"""The training-batch sampler (``data/dataset.py:56-258`` ``LongRangeSampler`` / ``DinoTrackerSampler``) over libdinotrk.

The reference keeps the valid trajectories and a [N'][T] bool ``can_sample``; every call builds ``can_sample.float()``
over the whole set, copies every candidate row twice by boolean indexing and maps the drawn times to frame-set slots
with one ``.nonzero()`` per point.  Here each set is compacted once into its valid rows and a bitmask of their valid
frames (include/dinotrk.h: dinotrk_sampler_*); a call counts the candidates of the drawn frames per block, finds the
selected ones by position and copies the drawn points.  The frame-set mapping is one ``searchsorted`` into the sorted
unique times (the same int64 slots: the values are unique).

The random draws are the reference's, with the same torch calls and arguments on the same device in the same order
(per set, fg then bg: ``randperm(T)[:num_frames]`` until at least 2 trajectories are candidates, ``randperm(n)[:batch]``,
``multinomial(2, replacement=False)`` on the identical 0/1 matrix), so a seeded run gives the reference's samples bit
for bit.  Syncs per set and call: one read-back of the candidate count per frame draw, as in the reference.

``keep_in_cpu=True`` samples from the reference's windows of 200,000 valid trajectories (``load_next_batch``).  The
valid rows then stay in pinned host memory and the kernels read only the drawn points through the device's mapping of
it; the device holds the window's frame bits, ceil(T / 32) words per row.  The only intended difference from the
reference: a set with fewer than 2 valid trajectories raises ``ValueError`` at construction (the reference's frame
draw loops forever on it).
"""
import ctypes
import math

import torch

from . import _lib

MAX_TRAJ_SIZE = 200_000


def _addr(t):
    """Address of a contiguous tensor in device or pinned host memory (the library maps the latter)."""
    assert t.is_contiguous() and (t.is_cuda or t.is_pinned())
    return ctypes.c_void_p(t.data_ptr())


class _TrajectorySet:
    """The valid rows [N'][T][2] of one trajectory set and their frame bits [N'][ceil(T / 32)] int32 (bit t % 32 of word
    t / 32 set where step t has both coordinates non-NaN), compacted by dinotrk_sampler_prepare_*."""

    def __init__(self, name, traj, keep_in_cpu):
        if not isinstance(traj, torch.Tensor):
            raise TypeError(f"{name}_trajectories must be a tensor, got {type(traj).__name__}")
        if traj.dtype != torch.float32:
            raise TypeError(f"{name}_trajectories must be float32, got {traj.dtype}")
        if traj.dim() != 3 or traj.shape[2] != 2 or traj.shape[1] < 1 or traj.shape[0] >= 2 ** 31 or traj.shape[1] > 65536:
            raise ValueError(f"{name}_trajectories must be [N][T][2] with N < 2^31 and 1 <= T <= 65536, got {tuple(traj.shape)}")
        if keep_in_cpu:
            if traj.device.type not in ("cpu", "cuda"):
                raise _lib.DinotrkError(f"{name}_trajectories on {traj.device}: expected a CPU or CUDA tensor")
            self.dev = traj.device if traj.is_cuda else _lib.require_cuda("cuda")
            if self.dev.index is None:
                self.dev = torch.device("cuda", torch.cuda.current_device())
        else:
            self.dev = _lib.require_cuda(traj.device)
        N, T = traj.shape[0], traj.shape[1]
        if N < 2:
            raise ValueError(f"{name}_trajectories: {N} trajectories, the sampler needs at least 2 valid ones")
        self.T, self.W = T, (T + 31) // 32
        lib = _lib.load()
        src = traj.contiguous() if traj.is_cuda else traj.contiguous().pin_memory()
        with torch.cuda.device(self.dev):
            ws = torch.empty(lib.dinotrk_sampler_workspace_bytes(N), device=self.dev, dtype=torch.uint8)
            st = _lib.stream_ptr()
            n = ctypes.c_int(0)
            _lib.check(lib.dinotrk_sampler_prepare_count(_addr(src), N, T, ctypes.byref(n), _lib.ptr(ws), ws.numel(), st),
                       "sampler_prepare_count")
            self.n = n.value
            if self.n < 2:
                raise ValueError(f"{name}_trajectories: {self.n} valid trajectories (more than one non-NaN step), the "
                                 "sampler needs at least 2")
            where = dict(device="cpu", pin_memory=True) if keep_in_cpu else dict(device=self.dev)
            self.rows = torch.empty(self.n, T, 2, dtype=torch.float32, **where)
            self.bits = torch.empty(self.n, self.W, dtype=torch.int32, **where)
            _lib.check(lib.dinotrk_sampler_prepare_emit(_addr(src), N, T, _addr(self.rows), _addr(self.bits), _lib.ptr(ws),
                                                        ws.numel(), st), "sampler_prepare_emit")
            if not traj.is_cuda:
                torch.cuda.current_stream().synchronize()   # the pinned copy of the input is read until here
        self.keep_in_cpu = keep_in_cpu
        self.n_batches = math.ceil(self.n / MAX_TRAJ_SIZE)
        self.load_window(0)

    def load_window(self, index):
        """dataset.py:120-131: valid rows [index * 200,000, min((index + 1) * 200,000, N')) (all of them when the set is
        kept on the device).  Only the window's frame bits move to the device."""
        if not self.keep_in_cpu:
            self.win_rows, self.win_bits = self.rows, self.bits
        else:
            start, end = index * MAX_TRAJ_SIZE, min((index + 1) * MAX_TRAJ_SIZE, self.n)
            self.win_rows = self.rows[start:end]
            self.win_bits = self.bits[start:end].to(self.dev)
        self.ws = torch.empty(_lib.load().dinotrk_sampler_workspace_bytes(self.win_rows.shape[0]), device=self.dev,
                              dtype=torch.uint8)

    def draw(self, num_frames, batch_size):
        """dataset.py:162-190: (t1_points, t2_points) [min(batch_size, n)][3] = (x, y, t) on the device."""
        lib, dev, T = _lib.load(), self.dev, self.T
        N = self.win_rows.shape[0]
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            n = ctypes.c_int(0)
            while True:
                frames = torch.arange(T, device=dev)[torch.randperm(T, device=dev)[:num_frames]]
                _lib.check(lib.dinotrk_sampler_count(_lib.ptr(self.win_bits), N, T, _lib.ptr(frames), frames.numel(),
                                                     ctypes.byref(n), _lib.ptr(self.ws), self.ws.numel(), st), "sampler_count")
                if n.value >= 2:
                    break
            perm = torch.randperm(n.value, device=dev)[:batch_size]
            m = perm.numel()
            row_ids = torch.empty(m, dtype=torch.int64, device=dev)
            weights = torch.empty(m, T, dtype=torch.float32, device=dev)
            if m:
                _lib.check(lib.dinotrk_sampler_select(_lib.ptr(self.win_bits), N, T, _lib.ptr(frames), frames.numel(),
                                                      _lib.ptr(perm), m, _lib.ptr(row_ids), _lib.ptr(weights),
                                                      _lib.ptr(self.ws), self.ws.numel(), st), "sampler_select")
            draws = weights.multinomial(2, replacement=False)
            t1 = torch.empty(m, 3, dtype=torch.float32, device=dev)
            t2 = torch.empty(m, 3, dtype=torch.float32, device=dev)
            if m:
                _lib.check(lib.dinotrk_sampler_gather(_addr(self.win_rows), T, _lib.ptr(row_ids), _lib.ptr(draws.contiguous()),
                                                      m, _lib.ptr(t1), _lib.ptr(t2), st), "sampler_gather")
        return t1, t2


class LongRangeSampler(torch.nn.Module):
    """dataset.py:56-208 with the reference's constructor; ``forward`` returns (t1_points, t2_points) [B][3]."""

    def __init__(self, batch_size, fg_trajectories=None, bg_trajectories=None, fg_traj_ratio=0.5, num_frames=None,
                 keep_in_cpu=False) -> None:
        super().__init__()
        self.batch_size = batch_size
        self.num_frames = num_frames
        self.fg_traj_ratio = fg_traj_ratio
        self.keep_in_cpu = keep_in_cpu
        self.max_traj_size = MAX_TRAJ_SIZE
        self.gpu_batch_index = 0
        self.fg = _TrajectorySet("fg", fg_trajectories, keep_in_cpu)
        self.bg = _TrajectorySet("bg", bg_trajectories, keep_in_cpu)
        self.vid_len = self.fg.T

    def load_next_batch(self):
        """dataset.py:108-131: the next window of each set (nothing when the sets are kept whole on the device)."""
        if not self.keep_in_cpu:
            return
        self.gpu_batch_index += 1
        for s in (self.fg, self.bg):
            s.load_window(self.gpu_batch_index % s.n_batches)

    def get_fg_batch_size(self):
        return int(self.batch_size * self.fg_traj_ratio)

    def forward(self):
        assert self.num_frames is not None, "num_frames must be specified"
        fg_batch_size = self.get_fg_batch_size()
        fg1, fg2 = self.fg.draw(self.num_frames, fg_batch_size)
        bg1, bg2 = self.bg.draw(self.num_frames, self.batch_size - fg_batch_size)
        return torch.cat([fg1, bg1], dim=0), torch.cat([fg2, bg2], dim=0)


class DinoTrackerSampler(LongRangeSampler):
    """dataset.py:211-258: the sample dict of one training iteration."""

    def __init__(self, batch_size, range_normalizer, dst_range, fg_trajectories=None, bg_trajectories=None,
                 fg_traj_ratio=0.5, num_frames=None, keep_in_cpu=False) -> None:
        super().__init__(batch_size, fg_trajectories=fg_trajectories, bg_trajectories=bg_trajectories,
                         fg_traj_ratio=fg_traj_ratio, num_frames=num_frames, keep_in_cpu=keep_in_cpu)
        self.range_normalizer = range_normalizer
        self.dst_range = dst_range

    def forward(self):
        t1_points, t2_points = super().forward()
        times = torch.cat((t1_points[:, 2], t2_points[:, 2])).unique()
        frames_set_t = times.int()
        source_frame_indices = torch.searchsorted(times, t1_points[:, 2].contiguous())
        target_frame_indices = torch.searchsorted(times, t2_points[:, 2].contiguous())
        t1_points_normalized = self.range_normalizer(t1_points, dst=self.dst_range)
        t2_points_normalized = self.range_normalizer(t2_points, dst=self.dst_range)
        t1_points[:, 2] = t1_points_normalized[:, 2]
        return {
            "frames_set_t": frames_set_t,
            "source_frame_indices": source_frame_indices,
            "target_frame_indices": target_frame_indices,
            "t1_points_normalized": t1_points_normalized,
            "t2_points_normalized": t2_points_normalized,
            "t1_points": t1_points,
            "target_times": t2_points[:, 2],
        }

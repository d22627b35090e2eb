"""Generate ``tests/golden/sampler_small.npz`` from the LIVE reference's ``DinoTrackerSampler`` (data/dataset.py) on the
CPU.

    python -m oracle.make_golden_sampler

Inputs are regenerated from seeds (``make_trajectories``), so the fixture holds only the configuration and the sample
dicts.  Two cases at T = 12 with train.yaml's 4 frames per draw:
  * ``small``: fg = 3,000 trajectories, bg = 60 trajectories confined to frames 0-2.  Both sets contain single-step
    rows (filtered out) and rows with NaN in one coordinate only; the bg set has fewer valid rows than its share of the
    batch, and most of its frame draws fail and are redrawn.  6 consecutive calls.
  * ``windowed``: ``keep_in_cpu=True`` with 450,000 fg and 300,000 bg trajectories (more than 200,000 valid each), calls
    interleaved with three ``load_next_batch``: the fg windows 0, 1, 2, 0 and the bg windows 0, 1, 0, 1.
The reference's ``.cuda()`` calls (dataset.py:88-131) are shimmed to the identity for the generation only.
"""
import contextlib
import os

import numpy as np
import torch

from . import ref_harness
from . import sampler as osm

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sampler_small.npz")
H, W = 476, 854
KEYS = ("frames_set_t", "source_frame_indices", "target_frame_indices", "t1_points_normalized", "t2_points_normalized",
        "t1_points", "target_times")
CASES = {
    "small": dict(T=12, fg=(3000, 11, None), bg=(60, 12, (0, 3)), batch=128, num_frames=4, ratio=0.5, keep_in_cpu=False,
                  seed=13, ops=["call"] * 6),
    "windowed": dict(T=12, fg=(450_000, 21, None), bg=(300_000, 22, None), batch=64, num_frames=4, ratio=0.5,
                     keep_in_cpu=True, seed=23, ops=["call", "call", "next", "call", "next", "call", "call", "next", "call"]),
}


def make_trajectories(N, T, seed, frames=None):
    """[N][T][2] positions in a 476 x 854 frame on one interval of steps each (inside ``frames`` = [lo, hi) when given),
    NaN elsewhere; about a sixth of the rows are single-step, and 10% get NaN in one coordinate at one step."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = frames or (0, T)
    xy = torch.rand(N, T, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    start = torch.randint(lo, hi, (N,), generator=g)
    length = torch.randint(1, hi - lo + 1, (N,), generator=g)
    length = torch.where(torch.rand(N, generator=g) < 0.1, torch.ones_like(length), length)
    end = torch.clamp(start + length, max=hi)
    t = torch.arange(T)
    xy[(t[None] < start[:, None]) | (t[None] >= end[:, None])] = float("nan")
    one = (torch.rand(N, generator=g) < 0.1).nonzero()[:, 0]
    step = torch.randint(0, T, (one.numel(),), generator=g)
    coord = torch.randint(0, 2, (one.numel(),), generator=g)
    xy[one, step, coord] = float("nan")
    return xy


def case_inputs(case):
    c = CASES[case]
    return tuple(make_trajectories(n, c["T"], seed, frames) for n, seed, frames in (c["fg"], c["bg"]))


def run_case(case, sampler_cls, normalizer_cls, device="cpu", fg=None, bg=None, **kw):
    """Build the sampler under the case's seed and run its ops -> {f"{case}/{i}/{key}": array} for every call i."""
    c = CASES[case]
    if fg is None:
        fg, bg = case_inputs(case)
    fg, bg = fg.to(device), bg.to(device)
    rn = normalizer_cls(shapes=(W, H, c["T"]), device=device)
    torch.manual_seed(c["seed"])
    s = sampler_cls(batch_size=c["batch"], range_normalizer=rn, dst_range=(-1, 1), fg_trajectories=fg, bg_trajectories=bg,
                    fg_traj_ratio=c["ratio"], num_frames=c["num_frames"], keep_in_cpu=c["keep_in_cpu"], **kw)
    out, i = {}, 0
    for op in c["ops"]:
        if op == "next":
            s.load_next_batch()
            continue
        sample = s()
        for k in KEYS:
            out[f"{case}/{i}/{k}"] = sample[k].cpu().numpy()
        i += 1
    return out, s


@contextlib.contextmanager
def cuda_is_identity():
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = orig


def generate():
    ref_harness.install("cpu")
    import data.dataset as ds
    out = {}
    for case in CASES:
        with cuda_is_identity():
            ref, _ = run_case(case, ds.DinoTrackerSampler, ds.RangeNormalizer)
        ora, s = run_case(case, osm.DinoTrackerSampler, osm.RangeNormalizer)
        assert set(ref) == set(ora) and all(np.array_equal(ref[k], ora[k]) and ref[k].dtype == ora[k].dtype for k in ref), case
        out.update(ref)
        out[f"{case}/frame_draws"] = np.array(s.frame_draws, dtype=np.int64)
    return out


if __name__ == "__main__":
    np.savez_compressed(OUT, **generate())
    print("wrote", OUT)

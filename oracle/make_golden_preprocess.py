"""Generate the trajectory and flow-filter fixtures of ``tests/golden/`` by running the LIVE reference (only where its
sources are present), next to ``oracle/make_golden.py``:

    python -m oracle.make_golden_preprocess

Inputs are seeded and regenerable (``oracle/trajectories.py``, ``oracle/of_filter.py``).  Outputs are whatever the
unmodified reference scripts return on CPU behind the shims of ``oracle/ref_harness.py`` plus two more, installed here
in memory only:
  1. ``raft_large`` of ``preprocessing/extract_trajectories.py`` is replaced by a stand-in returning pre-baked flows.
     ``save_trajectories`` builds the model from the module's globals, so patching that attribute is enough.  Frame k is
     written as a constant image of value 10 + 20 k; the stand-in reads k back from its (padded, normalised) input and
     returns the flow of the requested frame pair, padded as RAFT's output would be.
  2. ``torch.Tensor.cuda`` is the identity (extract_trajectories.py:265 calls ``.cuda()``).
"""
import argparse
import os
import tempfile

import numpy as np
import torch

from . import of_filter as oof
from . import ref_harness
from . import trajectories as otr
from .make_golden import GOLDEN_DIR

# name: video size, frames, flow seed, chaining parameters.  H - 1 and W - 1 are powers of two and the flows are
# whole pixels, so that every operation is exact (see oracle.trajectories.smooth_flows).
TRAJ_CASES = {
    "traj_chain_small": dict(H=33, W=65, T=7, seed=71, threshold=1.0, min_len=2, direct=False, dthr=None),
    "traj_direct_small": dict(H=33, W=65, T=6, seed=72, threshold=1.5, min_len=3, direct=True, dthr=2.5),
}
OF_CASE = dict(H=98, W=126, T=4, seed=73, stride=7, n_max=40)


def traj_case_flows(cfg, device="cpu"):
    return otr.smooth_flows(cfg["T"], cfg["H"], cfg["W"], cfg["seed"], amplitude=6.0, integer=True, device=device)


def of_case_inputs(cfg=OF_CASE, device="cpu"):
    """(trajectories [M][T][2], best-buddy dict) of the flow-filter case: chained smooth flows (min length 2) and random
    token pairs per ordered frame pair; peak fields on the pairs with an even source frame only."""
    flow = otr.smooth_flows(cfg["T"], cfg["H"], cfg["W"], cfg["seed"], amplitude=4.0)
    fwd, bwd, _ = otr.stack_flows(flow, cfg["T"])
    traj = otr.extract_trajectories(fwd, bwd, None, 1.0, 2).to(device)
    grid, _, _ = oof.create_meshgrid(cfg["H"], cfg["W"], step=cfg["stride"])
    g = torch.Generator().manual_seed(cfg["seed"])
    bb = {}
    for s in range(cfg["T"]):
        for t in range(cfg["T"]):
            if s == t:
                continue
            n = int(torch.randint(0, cfg["n_max"], (1,), generator=g))
            d = {"source_coords": grid[torch.randint(0, len(grid), (n,), generator=g)],
                 "target_coords": grid[torch.randint(0, len(grid), (n,), generator=g)],
                 "cos_sims": torch.rand(n, generator=g)}
            if s % 2 == 0:
                d["peak_coords"] = None
                d["peak_affs"] = torch.rand(n, 2, generator=g)
                d["r"] = torch.rand(n, generator=g)
            bb[f"{s}_{t}"] = {k: (v.to(device) if v is not None else None) for k, v in d.items()}
    return traj, bb


class _PrebakedRaft(torch.nn.Module):
    def __init__(self, flow, H, W):
        super().__init__()
        self.flow, self.H, self.W = flow, H, W

    def forward(self, a, b, num_flow_updates=12):
        def frame(x):
            v = ((x[0, 0, 0, 0].item() + 1) / 2 * 255 - 10) / 20
            assert abs(v - round(v)) < 1e-3, v
            return round(v)
        ht, wd = a.shape[-2:]
        top, left = (ht - self.H) // 2, (wd - self.W) // 2
        out = torch.zeros(a.shape[0], 2, ht, wd)
        for i in range(a.shape[0]):
            out[i, :, top:top + self.H, left:left + self.W] = self.flow(frame(a[i:i + 1]), frame(b[i:i + 1]))
        return [out]


def gen_traj_case(name, cfg):
    from PIL import Image
    ref_harness.install("cpu")
    from preprocessing import extract_trajectories as et
    flow = traj_case_flows(cfg)
    d = tempfile.mkdtemp()
    frames = os.path.join(d, "frames")
    os.makedirs(frames)
    for k in range(cfg["T"]):
        Image.fromarray(np.full((cfg["H"], cfg["W"], 3), 10 + 20 * k, dtype=np.uint8)).save(os.path.join(frames, f"{k:05d}.png"))
    args = argparse.Namespace(frames_path=frames, output_path=os.path.join(d, "out", "traj.pt"), infer_res_size=None,
                              threshold=cfg["threshold"], min_trajectory_length=cfg["min_len"],
                              filter_using_direct_flow=cfg["direct"], direct_flow_threshold=cfg["dthr"])
    real_raft, real_cuda = et.raft_large, torch.Tensor.cuda
    et.raft_large = lambda *a, **kw: _PrebakedRaft(flow, cfg["H"], cfg["W"])
    torch.Tensor.cuda = lambda self, *a, **kw: self
    try:
        et.save_trajectories(args)
    finally:
        et.raft_large, torch.Tensor.cuda = real_raft, real_cuda
    traj = torch.load(args.output_path)
    valid = ~traj.isnan().any(dim=-1)
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), trajectories=traj.numpy(),
                        cfg=np.array([cfg["H"], cfg["W"], cfg["T"], cfg["seed"], cfg["min_len"]]))
    print(name, "trajectories", tuple(traj.shape), "mean length", float(valid.sum(1).float().mean()))


def gen_of_case(name, cfg=OF_CASE):
    ref_harness.install("cpu")
    from preprocessing_dino_bb import of_filter_dino_best_buddies as off
    traj, bb = of_case_inputs(cfg)
    d = tempfile.mkdtemp()
    torch.save(bb, os.path.join(d, "bb.pt"))
    torch.save(traj, os.path.join(d, "traj.pt"))
    args = argparse.Namespace(dino_bb_path=os.path.join(d, "bb.pt"), traj_path=os.path.join(d, "traj.pt"),
                              out_path=os.path.join(d, "out", "bbf.pt"), dino_bb_stride=cfg["stride"], h=cfg["H"], w=cfg["W"])
    off.run(args)
    res = torch.load(args.out_path)
    out = {}
    for k, v in res.items():
        for kk, vv in v.items():
            if vv is not None:
                out[f"{k}.{kk}"] = vv.numpy()
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    print(name, "M", traj.shape[0], {k: (0 if v["source_coords"] is None else v["source_coords"].shape[0]) for k, v in res.items()})


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for name, cfg in TRAJ_CASES.items():
        gen_traj_case(name, cfg)
    gen_of_case("of_filter_small")


if __name__ == "__main__":
    main()

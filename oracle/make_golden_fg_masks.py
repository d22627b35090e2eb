"""Generate ``tests/golden/fg_mask_small.npz`` and ``tests/golden/traj_split_small.npz`` by running the LIVE reference
(only where its sources are present), next to ``oracle/make_golden_preprocess.py``:

    python -m oracle.make_golden_fg_masks

1. ``gen_fg_mask_case``: ``preprocessing/create_fg_mask.py::get_fg_mask_from_pca`` on the CPU, under a fixed seed, on
   seeded features with a planted foreground disc moving across the frames (``oracle.fg_masks.planted_features``).
2. ``gen_traj_split_case``: ``preprocessing/split_trajectories_to_fg_bg.py::mask_filter_trajectories`` on PNG masks in a
   temporary folder and seeded chain-style trajectories (``oracle.fg_masks.split_case_inputs``), with
   ``torch.Tensor.cuda`` the identity (:61 calls ``.cuda()``).  The masks are 476 x 854, the size ``load_masks``
   resizes to by default, so the resize is the identity.
"""
import os
import tempfile

import numpy as np
import torch

from . import fg_masks as ofg
from . import ref_harness
from .make_golden import GOLDEN_DIR

FG_CASE = dict(T=3, h=9, w=12, C=32, seed=41, torch_seed=42, H=61, W=86, q=3, threshold=0.6)
SPLIT_CASE = dict(N=3000, T=6, H=476, W=854, seed=43)


def fg_case_inputs(cfg=FG_CASE):
    return ofg.planted_features(cfg["T"], cfg["h"], cfg["w"], cfg["C"], cfg["seed"], noise=0.6)


def gen_fg_mask_case(name="fg_mask_small", cfg=FG_CASE):
    ref_harness.install("cpu")
    from preprocessing import create_fg_mask as cfm
    feats, plant = fg_case_inputs(cfg)
    torch.manual_seed(cfg["torch_seed"])
    mask = cfm.get_fg_mask_from_pca(feats, (cfg["H"], cfg["W"]), q=cfg["q"], interpolation="nearest",
                                    fg_mask_threshold=cfg["threshold"])
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), mask=mask.astype(np.uint8),
                        feat_checksum=np.array([feats.double().sum().item(), feats.double().abs().sum().item()]))
    print(name, mask.shape, "fg fraction", float(mask.mean()), "planted", float(plant.float().mean()))


def gen_traj_split_case(name="traj_split_small", cfg=SPLIT_CASE):
    from PIL import Image
    ref_harness.install("cpu")
    from preprocessing import split_trajectories_to_fg_bg as stf
    traj, masks = ofg.split_case_inputs(cfg["N"], cfg["T"], cfg["H"], cfg["W"], cfg["seed"])
    d = tempfile.mkdtemp()
    os.makedirs(os.path.join(d, "masks"))
    for k, m in enumerate(masks.numpy()):
        Image.fromarray(m).save(os.path.join(d, "masks", f"{k:05d}.png"))
    torch.save(traj, os.path.join(d, "traj.pt"))
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **kw: self
    try:
        out = {}
        for which, filter_bg in (("fg", False), ("bg", True)):
            p = os.path.join(d, which + ".pt")
            stf.mask_filter_trajectories(os.path.join(d, "traj.pt"), os.path.join(d, "masks"), p, filter_bg=filter_bg)
            out[which] = torch.load(p).numpy()
    finally:
        torch.Tensor.cuda = real_cuda
    np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
    print(name, {k: v.shape for k, v in out.items()})


def main():
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    gen_fg_mask_case()
    gen_traj_split_case()


if __name__ == "__main__":
    main()

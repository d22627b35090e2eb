"""Generate ``tests/golden/contrastive_small.npz`` from the LIVE reference's contrastive losses on the CPU.

    python -m oracle.make_golden_contrastive

The reference's ``DINOTracker.get_dino_bb_contrastive_loss`` / ``get_refined_bb_contrastive_loss`` (dino_tracker.py:159-330)
run on a trainer stand-in (``object.__new__(DINOTracker)`` + ``config``, ``fg_masks``, ``dino_bb_pairs``) and a tracker
stand-in (oracle/contrastive.py: ModelStandIn) over small seeded inputs: 6 frames of 98 x 126, C = 32, a frame set of 4,
24 points per pair, train.yaml's temperature and weights.  The reference calls ``.cuda()`` (models/utils.py:54,
dino_tracker.py:196-203) and builds its token grid on "cuda" (models/utils.py:87); both are shimmed to the CPU for the
generation only.  Per loss the fixture holds the loss, its gradient with respect to a leaf ``frame_embeddings`` and the
pairs and indices the oracle selects under the same seed (checked to give the reference's loss).  The seeds are the
first under which a refined pair is a self-pair and a dino-BB pair draws no foreground buddies.
"""
import contextlib
import os

import numpy as np
import torch

from . import contrastive as oc
from . import ref_harness

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "contrastive_small.npz")

CONFIG = {"cl_n_frames": 4, "cl_points_per_pair": 24, "cl_fg_points_ratio": 0.7, "cl_temp": 0.1, "cl_div_dino_bb": 700,
          "cl_div_ref_bb": 900, "bb_amb_sig_a": 27, "bb_amb_sig_b": -5.7, "dino_patch_size": 14}
T, H, W, C, STRIDE = 6, 98, 126, 32, 7
FRAMES = [0, 2, 3, 5]
EMPTY_MASK_FRAME = 5          # a frame without foreground: its pairs have no fg buddies


def make_inputs():
    g = torch.Generator().manual_seed(1234)
    h, w = (H - 14) // STRIDE + 1, (W - 14) // STRIDE + 1
    P = h * w
    # smooth shifted fields plus noise: realistic nearest neighbours, no exact ties
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    freq = torch.rand(C, 2, generator=g) * 0.6
    phase = torch.rand(C, generator=g) * 6.28
    emb = []
    for i in range(len(FRAMES)):
        f = torch.sin(freq[:, 0, None, None] * (xx + 0.7 * i) + freq[:, 1, None, None] * yy + phase[:, None, None])
        emb.append(f + 0.05 * torch.randn(C, h, w, generator=g))
    emb = torch.stack(emb).contiguous()
    masks = torch.zeros(T, H, W)
    for t in range(T):
        if t != EMPTY_MASK_FRAME:
            masks[t, 20 + 3 * t:70, 30:90 - 4 * t] = 1.0
    coords = oc.get_vit_feature_coords_from_mask(H, W, STRIDE, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s == t:
                continue
            n = int(torch.randint(40, 90, (1,), generator=g))
            src = torch.randperm(P, generator=g)[:n]
            tgt = torch.randint(P, (n,), generator=g)
            bb[f"{s}_{t}"] = {"source_coords": coords[src].clone(), "target_coords": coords[tgt].clone(),
                              "cos_sims": torch.rand(n, generator=g) * 0.6 + 0.4, "r": torch.rand(n, generator=g) * 0.4}
    return emb, masks, bb


@contextlib.contextmanager
def cpu_shims(dt_module):
    orig_cuda = torch.Tensor.cuda
    orig_coords = dt_module.get_vit_feature_coords_from_mask
    torch.Tensor.cuda = lambda self, *a, **k: self
    dt_module.get_vit_feature_coords_from_mask = lambda *a, **k: orig_coords(*a, **{**k, "device": "cpu"})
    try:
        yield
    finally:
        torch.Tensor.cuda = orig_cuda
        dt_module.get_vit_feature_coords_from_mask = orig_coords


def trainer_standin(cls, masks, bb):
    tr = object.__new__(cls)
    tr.config = dict(CONFIG)
    tr.fg_masks = masks
    tr.dino_bb_pairs = bb
    return tr


def run_loss(which, method_owner, tr, emb0, video, seed, record=None):
    emb = emb0.clone().requires_grad_(True)
    model = oc.ModelStandIn(video, emb, stride=STRIDE)
    fs = torch.tensor(FRAMES)
    torch.manual_seed(seed)
    kw = {} if record is None else {"record": record}
    if which == "dino":
        loss = method_owner.get_dino_bb_contrastive_loss(tr, model, fs, **kw)
    else:
        loss = method_owner.get_refined_bb_contrastive_loss(tr, model, fs, emb, batch_size=CONFIG["cl_n_frames"],
                                                            points_per_pair=CONFIG["cl_points_per_pair"],
                                                            fg_points_ratio=CONFIG["cl_fg_points_ratio"],
                                                            temp=CONFIG["cl_temp"], cl_div=CONFIG["cl_div_ref_bb"], **kw)
    loss.backward()
    return loss.detach(), emb.grad


def pack_record(rec):
    pairs = np.array([(s, t, len(a)) for s, t, a, _ in rec], dtype=np.int64).reshape(-1, 3)
    src = np.concatenate([a.numpy() for _, _, a, _ in rec]).astype(np.int64)
    tgt = np.concatenate([b.numpy() for _, _, _, b in rec]).astype(np.int64)
    return pairs, src, tgt


def generate():
    ref_harness.install("cpu")
    import dino_tracker as dt
    emb, masks, bb = make_inputs()
    video = torch.zeros(T, 3, H, W)
    tr = trainer_standin(dt.DINOTracker, masks, bb)
    out = {"emb": emb.numpy(), "masks": masks.numpy(), "frames": np.array(FRAMES, dtype=np.int64), "video_hw": np.array([H, W])}
    keys = sorted(bb)
    out["bb_keys"] = np.array(keys)
    for k in keys:
        for f, v in bb[k].items():
            out[f"bb/{k}/{f}"] = v.numpy()
    oracle_owner = type("OracleTrainer", (), {n: getattr(oc, n) for n in (
        "get_dino_bb_contrastive_loss", "get_refined_bb_contrastive_loss", "get_bb_pairs_contrastive_loss")})
    for which, ok in (("dino", lambda rec: any(FRAMES[s] == EMPTY_MASK_FRAME for s, _, _, _ in rec)),
                      ("refined", lambda rec: any(s == t for s, t, _, _ in rec))):
        for seed in range(100):
            rec = []
            run_loss(which, oracle_owner, tr, emb, video, seed, rec)
            if ok(rec):
                break
        else:
            raise RuntimeError(f"no seed gives the {which} case")
        with cpu_shims(dt):
            loss, grad = run_loss(which, dt.DINOTracker, tr, emb, video, seed)
        oloss, ograd = run_loss(which, oracle_owner, tr, emb, video, seed)
        assert torch.allclose(oloss, loss, rtol=1e-5) and torch.allclose(ograd, grad, rtol=1e-4, atol=1e-8), which
        pairs, src, tgt = pack_record(rec)
        out.update({f"{which}_seed": np.array(seed), f"{which}_loss": loss.numpy(), f"{which}_grad": grad.numpy(),
                    f"{which}_pairs": pairs, f"{which}_src": src, f"{which}_tgt": tgt})
    return out


def load_bb(z):
    return {str(k): {f: torch.from_numpy(z[f"bb/{k}/{f}"]) for f in ("source_coords", "target_coords", "cos_sims", "r")}
            for k in z["bb_keys"]}


if __name__ == "__main__":
    np.savez_compressed(OUT, **generate())
    print("wrote", OUT)

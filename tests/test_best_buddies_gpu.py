"""GPU parity: best-buddies (wgmma GEMM + top-2 epilogue + exact resolve) against the reference vectors
and the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import best_buddies as obb
from oracle import synth
from oracle.tracker import Geometry

from golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu


def check_against(res, ref, cos_tol=2e-6):
    assert set(res) == set(ref)
    for k in ref:
        assert np.array_equal(res[k]["source_coords"].cpu().numpy(), np.asarray(ref[k]["source_coords"])), k
        assert np.array_equal(res[k]["target_coords"].cpu().numpy(), np.asarray(ref[k]["target_coords"])), k
        assert np.abs(res[k]["cos_sims"].cpu().numpy() - np.asarray(ref[k]["cos_sims"])).max() <= cos_tol, k


def test_best_buddies_match_reference_vectors():
    from dino_tracker_b200.best_buddies import best_buddies
    g = dict(np.load(os.path.join(GOLDEN_DIR, "bb_small.npz")))
    H, W, T, C = (int(v) for v in g["HWTC"])
    feats = torch.from_numpy(g["features"])
    res = best_buddies(feats, H, W)
    ref = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                ref[f"{s}_{t}"] = {k: g[f"{s}_{t}.{k}"] for k in ("source_coords", "target_coords", "cos_sims")}
    check_against(res, ref)


def test_best_buddies_full_geometry_against_oracle():
    from dino_tracker_b200.best_buddies import best_buddies
    geo = Geometry()
    T, C = 3, 256
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=77, noise=0.6, max_shift=2)
    res = best_buddies(feats, geo.H, geo.W)
    ref = obb.best_buddies(feats, geo.H, geo.W)
    ref = {k: {kk: vv.numpy() for kk, vv in v.items()} for k, v in ref.items()}
    check_against(res, ref)
    n_bb = sum(v["cos_sims"].shape[0] for v in res.values())
    assert n_bb > 1000


def test_pair_sharding_covers_all_pairs():
    from dino_tracker_b200.best_buddies import best_buddies
    g = dict(np.load(os.path.join(GOLDEN_DIR, "bb_small.npz")))
    H, W, T, C = (int(v) for v in g["HWTC"])
    feats = torch.from_numpy(g["features"])
    full = best_buddies(feats, H, W)
    parts = {}
    for r in range(2):
        parts.update(best_buddies(feats, H, W, rank=r, world=2))
    assert set(parts) == set(full)
    for k in full:
        assert torch.equal(parts[k]["cos_sims"], full[k]["cos_sims"])


def test_bb_peak_filter_matches_reference_vectors():
    """SURVEY.md 8f-3: compute_bb_nms + compute_max_r on the GPU against the live compute_dino_bb_nms.py vectors."""
    from dino_tracker_b200.best_buddies import PackedFeatures, best_buddies, compute_bb_nms, compute_max_r
    g = dict(np.load(os.path.join(GOLDEN_DIR, "bb_nms_small.npz")))
    H, W, T, C = (int(v) for v in g["HWTC"])
    geo = Geometry(H=H, W=W)
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=int(g["seed"]), noise=0.5, max_shift=2)
    bbs = best_buddies(feats, H, W)
    pk = PackedFeatures(feats)
    for key in list(bbs):
        if "r" in bbs[key]:
            continue
        sf, tf = (int(x) for x in key.split("_"))
        a = compute_bb_nms(bbs[f"{sf}_{tf}"], sf, tf, pk)
        b = compute_bb_nms(bbs[f"{tf}_{sf}"], tf, sf, pk)
        bbs[key], bbs[f"{tf}_{sf}"] = compute_max_r(a, b)
    for key in bbs:
        assert np.array_equal(bbs[key]["source_coords"].cpu().numpy(), g[key + ".source_coords"]), key
        e_p = np.abs(bbs[key]["peak_affs"].cpu().numpy() - g[key + ".peak_affs"]).max()
        e_r = np.abs(bbs[key]["r"].cpu().numpy() - g[key + ".r"]).max()
        assert e_p <= 2e-6 and e_r <= 4e-6, (key, e_p, e_r)


def test_bb_peak_filter_full_geometry_against_oracle():
    from oracle import bb_nms as onms
    from dino_tracker_b200.best_buddies import PackedFeatures, best_buddies, compute_bb_nms
    geo = Geometry()
    T, C = 2, 128
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=78, noise=0.6, max_shift=2)
    bbs = best_buddies(feats, geo.H, geo.W)
    pk = PackedFeatures(feats)
    got = compute_bb_nms(bbs["0_1"], 0, 1, pk)
    sub = {k: v.cpu()[:200] for k, v in bbs["0_1"].items()}           # the oracle's Python NMS loop: 200 source points
    ref = onms.compute_bb_nms(sub, 0, 1, feats, obb.token_coords(geo.H, geo.W))
    assert (got["peak_affs"].cpu()[:200] - ref["peak_affs"]).abs().max().item() <= 2e-6
    assert (got["r"].cpu()[:200] - ref["r"]).abs().max().item() <= 4e-6

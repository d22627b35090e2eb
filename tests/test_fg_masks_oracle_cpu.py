"""CPU: the foreground-mask and trajectory-split oracles against the live reference's vectors, bit for bit, and the
fixtures regenerated from the reference where its sources are present."""
import os

import numpy as np
import pytest
import torch

from oracle import fg_masks as ofg
from oracle import make_golden_fg_masks as mgf
from oracle import ref_harness

from golden_util import GOLDEN_DIR


def _fg_oracle():
    cfg = mgf.FG_CASE
    feats, _ = mgf.fg_case_inputs()
    g = np.load(os.path.join(GOLDEN_DIR, "fg_mask_small.npz"))
    cs = np.array([feats.double().sum().item(), feats.double().abs().sum().item()])
    assert np.allclose(cs, g["feat_checksum"], rtol=1e-12), "seeded inputs drifted from fixture"
    torch.manual_seed(cfg["torch_seed"])
    mask = ofg.get_fg_mask_from_pca(feats, (cfg["H"], cfg["W"]), q=cfg["q"], fg_mask_threshold=cfg["threshold"])
    return mask, g["mask"]


def _split_oracle():
    cfg = mgf.SPLIT_CASE
    traj, masks = ofg.split_case_inputs(cfg["N"], cfg["T"], cfg["H"], cfg["W"], cfg["seed"])
    return {"fg": ofg.mask_filter(traj, masks), "bg": ofg.mask_filter(traj, masks, filter_bg=True)}


def test_fg_mask_oracle_matches_reference():
    mask, ref = _fg_oracle()
    assert mask.dtype == np.float32 and mask.shape == ref.shape
    assert np.array_equal(mask.astype(np.uint8), ref)
    assert 0 < ref.mean() < 1


def test_traj_split_oracle_matches_reference():
    got = _split_oracle()
    ref = np.load(os.path.join(GOLDEN_DIR, "traj_split_small.npz"))
    for k in ("fg", "bg"):
        assert np.array_equal(got[k].numpy(), ref[k], equal_nan=True), k
    assert len(ref["fg"]) > 0 and len(ref["bg"]) > 0
    assert len(ref["fg"]) + len(ref["bg"]) == mgf.SPLIT_CASE["N"]


@pytest.mark.skipif(not ref_harness.reference_available(), reason="the reference sources are not present")
def test_fixtures_regenerate_bit_for_bit(tmp_path, monkeypatch):
    monkeypatch.setattr(mgf, "GOLDEN_DIR", str(tmp_path))
    mgf.gen_fg_mask_case()
    mgf.gen_traj_split_case()
    for name in ("fg_mask_small", "traj_split_small"):
        new, old = np.load(tmp_path / (name + ".npz")), np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        assert set(new.files) == set(old.files)
        for k in old.files:
            assert np.array_equal(new[k], old[k], equal_nan=True), (name, k)

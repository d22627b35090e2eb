"""GPU parity of the preprocessing kernels: flow-consistency masks, trajectory chaining (with and without direct flow),
the nearest trajectory of every token centre, the best-buddies flow filter and the whole best-buddy preprocessing
(best buddies -> trajectories -> flow filter -> NMS), against the oracle and the live reference's vectors."""
import os

import numpy as np
import pytest
import torch

from oracle import best_buddies as obb
from oracle import bb_nms as onms
from oracle import make_golden_preprocess as mgp
from oracle import of_filter as oof
from oracle import synth
from oracle import trajectories as otr
from oracle.tracker import Geometry

from golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _close(a, b):
    """max |a - b| <= max(1e-4 px, 2 ulp of the coordinate): above x = 512 one fp32 ulp is 6.1e-5 px, and the walk's
    bilinear sums may round differently from ATen's in the last bit (FMA contraction of its accumulation)."""
    ulp = torch.nextafter(b.abs(), torch.full_like(b, float("inf"))) - b.abs()
    return bool(((a - b).abs() <= torch.clamp(2 * ulp, min=1e-4)).all())


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(-1.0), b.nan_to_num(-1.0))


@pytest.mark.parametrize("name", sorted(mgp.TRAJ_CASES))
def test_chaining_exact_on_integer_flows(name):
    """Whole-pixel flows on a (2^a + 1) x (2^b + 1) video: every operation is exact, so the kernels must agree with the
    oracle (run on the GPU) and with the reference's vectors bit for bit, counts included."""
    from dino_tracker_b200.trajectories import chain_trajectories, flow_masks
    cfg = mgp.TRAJ_CASES[name]
    fwd, bwd, direct = otr.stack_flows(mgp.traj_case_flows(cfg, device=DEV), cfg["T"])
    assert torch.equal(flow_masks(fwd, bwd, cfg["threshold"]).cpu(), otr.flow_masks(fwd, bwd, cfg["threshold"])[..., 0].cpu())
    d = direct if cfg["direct"] else None
    got = chain_trajectories(fwd, bwd, d, cfg["threshold"], cfg["min_len"], cfg["dthr"]).cpu()
    ora = otr.extract_trajectories(fwd, bwd, d, cfg["threshold"], cfg["min_len"], cfg["dthr"]).cpu()
    ref = torch.from_numpy(np.load(os.path.join(GOLDEN_DIR, name + ".npz"))["trajectories"])
    assert _same(got, ora), (got.shape, ora.shape)
    assert _same(got, ref)


def _by_start(traj, W):
    """{(start frame, start pixel): trajectory} (a start pixel starts at most one trajectory per start frame)."""
    valid = ~traj.isnan().any(dim=-1)
    s = valid.float().argmax(dim=1)
    p0 = traj[torch.arange(traj.shape[0]), s]
    keys = (s * 10_000_000 + p0[:, 1].long() * W + p0[:, 0].long()).tolist()
    return dict(zip(keys, range(len(keys))))


@pytest.mark.parametrize("direct", [False, True])
def test_chaining_smooth_flows_full_size(direct):
    """Smooth fractional flows at 476 x 854: positions agree within max(1e-4 px, 2 ulp) where both keep a trajectory; the survivor
    sets differ by at most 0.01 % (decisions at the threshold or at a .5 rounding may go either way in the last bit)."""
    from dino_tracker_b200.trajectories import chain_trajectories
    T, H, W = 6, 476, 854
    fwd, bwd, dfn = otr.stack_flows(otr.smooth_flows(T, H, W, seed=81, amplitude=3.0, device=DEV, noise=False), T)
    d = dfn if direct else None
    got = chain_trajectories(fwd, bwd, d, 1.0, 2, 2.0 if direct else None)
    ora = otr.extract_trajectories(fwd, bwd, d, 1.0, 2, 2.0 if direct else None)
    kg, ko = _by_start(got, W), _by_start(ora, W)
    common = sorted(set(kg) & set(ko))
    diff = len(set(kg) ^ set(ko))
    assert len(common) > 100_000
    assert diff <= 1e-4 * len(ko), (diff, len(ko))
    a = got[[kg[k] for k in common]]
    b = ora[[ko[k] for k in common]]
    both = ~(a.isnan() | b.isnan())
    err = (a[both] - b[both]).abs().max().item()
    print(f"smooth flows, direct={direct}: {len(ko)} trajectories, {diff} differ, max |dxy| {err:.3g} px")
    assert _close(a[both], b[both])
    # lengths may differ only where the survivor sets differ (a last-bit decision ends one walk earlier)
    assert (a.isnan() != b.isnan()).any(dim=-1).any(dim=-1).sum().item() <= 1e-4 * len(ko)


def test_nearest_built_cases():
    from dino_tracker_b200.best_buddies import nearest_trajectories
    from test_preprocess_oracle_cpu import nearest_cases
    traj = nearest_cases()
    assert torch.equal(nearest_trajectories(traj.to(DEV), 40, 40, 7).cpu(), oof.nearest_grid(traj, 40, 40, 7))


def test_nearest_full_size_with_nans_and_ties():
    """476 x 854, 8,107 token centres, 60,000 trajectories on a quarter-pixel lattice (many exact equidistant ties),
    a third of the positions NaN, frame 3 all NaN."""
    from dino_tracker_b200.best_buddies import nearest_trajectories
    g = torch.Generator().manual_seed(91)
    M, T, H, W = 60_000, 4, 476, 854
    traj = (torch.rand(M, T, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0]) * 4).round() / 4
    traj[torch.rand(M, T, generator=g) < 0.33] = float("nan")
    traj[:, 3] = float("nan")
    traj[5000:5100] = traj[100:200]                      # duplicates: identical distances at different indices
    got = nearest_trajectories(traj.to(DEV), H, W, 7)
    ref = oof.nearest_grid(traj.to(DEV), H, W, 7)
    assert got.shape == (T, 67, 121)
    assert torch.equal(got, ref)
    assert (got[3] == 0).all()


def _bb_equal(got, ref):
    assert list(got) == list(ref)
    for k in ref:
        assert set(got[k]) == set(ref[k]), k
        for f in ref[k]:
            if ref[k][f] is None:
                assert got[k][f] is None, (k, f)
            else:
                assert torch.equal(got[k][f].cpu(), ref[k][f].cpu()), (k, f)


@pytest.mark.parametrize("on_gpu", [False, True])
def test_of_filter_matches_oracle_and_reference(on_gpu):
    """Pass-through fields present on some pairs (peak_affs, r; peak_coords None) and absent on others."""
    from dino_tracker_b200.best_buddies import of_filter
    cfg = mgp.OF_CASE
    traj, bb = mgp.of_case_inputs(device=DEV if on_gpu else "cpu")
    got = of_filter(bb, traj.to(DEV), cfg["H"], cfg["W"], cfg["stride"])
    _bb_equal(got, oof.of_filter(bb, traj, cfg["H"], cfg["W"], cfg["stride"]))
    ref = dict(np.load(os.path.join(GOLDEN_DIR, "of_filter_small.npz")))
    flat = {f"{k}.{kk}": vv.cpu().numpy() for k, v in got.items() for kk, vv in v.items() if vv is not None}
    assert set(flat) == set(ref)
    for k in ref:
        assert np.array_equal(flat[k], ref[k]), k
    for k, v in got.items():
        if v["source_coords"] is not None:
            assert v["source_coords"].device == bb[k]["source_coords"].device


def test_preprocess_best_buddies_end_to_end(tmp_path):
    """best buddies -> trajectories (synthetic flow_fn) -> flow filter -> NMS in one process, against the oracle chain:
    the trajectories equal the oracle's (same survivors, positions within max(1e-4 px, 2 ulp)), and the filtered, NMS'd dict equals
    the oracles' flow filter and NMS run on them."""
    from dino_tracker_b200.pipeline import preprocess_best_buddies
    H, W, T, C = 154, 210, 3, 16
    geo = Geometry(H=H, W=W)
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=32, noise=0.5, max_shift=2)
    flow = otr.smooth_flows(T, H, W, seed=83, amplitude=6.0, integer=True, device=DEV)    # breaks enough walks
    video = torch.arange(T, dtype=torch.float32).view(T, 1, 1, 1).expand(T, 3, H, W).contiguous() / 8

    def flow_fn(a, b):   # the frames carry their index in their (constant) value
        ia, ib = (x[:, 0, 0, 0].mul(8).round().long().tolist() for x in (a, b))
        return torch.stack([flow(i, j) for i, j in zip(ia, ib)])

    bb_dir, traj_path = str(tmp_path / "bb"), str(tmp_path / "traj" / "trajectories.pt")
    bb, traj, filt = preprocess_best_buddies(feats, video, bb_dir, traj_path, H, W, flow_fn=flow_fn, threshold=1.5,
                                             box_size=50, iou_thresh=0.2)
    for f in ("dino_best_buddies.pt", "dino_best_buddies_filtered.pt"):
        assert os.path.exists(os.path.join(bb_dir, f))
    assert _same(torch.load(traj_path), traj.cpu())
    # step 1: best buddies against the oracle
    ref_bb = obb.best_buddies(feats, H, W)
    for k in ref_bb:
        assert torch.equal(bb[k]["source_coords"].cpu(), ref_bb[k]["source_coords"]), k
    # step 2: trajectories against the oracle
    fwd, bwd, _ = otr.stack_flows(flow, T)
    ora = otr.extract_trajectories(fwd, bwd, None, 1.5, 2)   # round-trip errors of whole-pixel flows sit near sqrt(n)
    assert traj.shape == ora.shape and torch.equal(traj.isnan(), ora.isnan())
    ok = ~traj.isnan()
    assert _close(traj[ok], ora[ok])
    # steps 3 + 4: the oracles' flow filter and NMS
    ref = oof.of_filter({k: {kk: vv.cpu() for kk, vv in v.items()} for k, v in bb.items()}, traj.cpu(), H, W, 7)
    coords = obb.token_coords(H, W)
    n_kept = 0
    for key in list(ref):
        if ref[key]["source_coords"] is None or ref[key]["r"] is not None:
            continue
        sf, tf = (int(x) for x in key.split("_"))
        a = onms.compute_bb_nms(ref[f"{sf}_{tf}"], sf, tf, feats, coords)
        b = onms.compute_bb_nms(ref[f"{tf}_{sf}"], tf, sf, feats, coords)
        ref[key], ref[f"{tf}_{sf}"] = onms.compute_max_r(a, b)
    assert list(filt) == list(ref)
    for k, v in ref.items():
        if v["source_coords"] is None:
            assert filt[k]["source_coords"] is None and filt[k]["r"] is None, k
            continue
        n_kept += len(v["source_coords"])
        assert torch.equal(filt[k]["source_coords"].cpu(), v["source_coords"]), k
        assert torch.equal(filt[k]["target_coords"].cpu(), v["target_coords"]), k
        assert (filt[k]["cos_sims"].cpu() - v["cos_sims"]).abs().max().item() <= 2e-6, k
        assert (filt[k]["peak_affs"].cpu() - v["peak_affs"]).abs().max().item() <= 2e-6, k
        assert (filt[k]["r"].cpu() - v["r"]).abs().max().item() <= 4e-6, k
    assert n_kept > 0

"""GPU: tracking on the token grids of DINOv3's 16-pixel patches (stride 8: 58 x 105 tokens at 476 x 854; stride 16:
29 x 53), modelled on test_tracker_patch8_gpu.py.

Token c sits at pixel 8 + s c.  No tracker kernel depends on the patch beyond make_geom and the coordinate affine, so
the checks are those of patch 8 at the new geometry, with the existing bars: `infer` within 1e-3 px and identical
occlusion against the oracle at Geometry(patch=16); one training step's reverse pass against float64
(test_train_backward_gpu.py's bound and pinned kappas); and a tracker built from a DinoV3Features extractor, pixels to
tracks, against the chained oracles.  C = 384 (ViT-S/16) and 1024 (ViT-L/16).  Delta-DINO's CNN alignment keeps the
reference's patch-14 call, as at patch 8 (DESIGN 4.10, 4.11)."""
import pytest
import torch

import oracle
from oracle import delta_dino as od
from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle import vit_dinov3 as ov3
from oracle.tracker import Geometry

import test_train_backward_gpu as tb
from test_tracker_patch8_gpu import XY_TOL, _run_production, _tracker

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GEOS = {8: Geometry(H=476, W=854, patch=16, stride=8), 16: Geometry(H=476, W=854, patch=16, stride=16)}
WIDTHS = (384, 1024)


def test_geometry_at_patch_16():
    from dino_tracker_b200 import _lib
    for s, geo in GEOS.items():
        g = _lib.make_geom(geo.H, geo.W, 16, s, 35)
        assert (g.h, g.w) == (geo.h, geo.w) == ((58, 105) if s == 8 else (29, 53))


@pytest.mark.parametrize("kind", ["sharp", "well"])
@pytest.mark.parametrize("stride", [8, 16])
@pytest.mark.parametrize("C", WIDTHS)
def test_infer_matches_oracle(C, stride, kind):
    from dino_tracker_b200 import ModelInference
    geo, T = GEOS[stride], 4
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=C + 5, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=C + 1)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=10.0, jitter_seed=C)
    m = _tracker(geo, feats, head)
    pn = m.normalize_points_for_sampling(q.to(DEV))
    assert torch.allclose(pn.cpu(), ot.normalize_points_for_sampling(q, geo), rtol=0, atol=1e-6)
    traj, occ = ModelInference(m, m.range_normalizer, 0.7, 0.6).infer(q.to(DEV))
    torch.cuda.synchronize()
    oracle.use_exact_fp32()
    with torch.no_grad():
        t_ref, o_ref = oi.infer(feats.to(DEV), q.to(DEV), {k: v.to(DEV) for k, v in head.items()}, geo, 0.7, 0.6)
    err = (traj - t_ref).abs().max().item()
    print(f"[patch 16 / stride {stride}, C={C}, {kind}] max |dxy| = {err:.2e} px")
    assert err <= XY_TOL
    assert torch.equal(occ.cpu(), o_ref.cpu())


@pytest.mark.parametrize("C", WIDTHS)
def test_training_step_reverse_against_float64(C):
    """The training step's reverse pass at 476 x 854, N = 4, B = 512, patch 16 / stride 8."""
    geo = GEOS[8]
    feats, _ = synth.shifted_field_features(4, C, geo.h, geo.w, seed=113, noise=0.2, max_shift=2)
    pts, tgt, gout = tb._batch(geo, 4, 512, tb._gen("patch16", C))
    _run_production(f"patch 16 C={C}", geo, feats, synth.head_weights("sharp", seed=113), pts, tgt, gout)


@pytest.mark.parametrize("C", WIDTHS)
def test_pixels_to_tracks_dinov3(C):
    """DINOv3 (C wide, C / 64 heads, 4 registers, 2 blocks) at stride 8 -> delta-DINO -> infer, against the chained
    oracles."""
    from dino_tracker_b200 import ModelInference, build_tracker_from_video
    from dino_tracker_b200.vit import DinoV3Features
    H, W, T = 98, 126, 4
    geo = Geometry(H=H, W=W, patch=16, stride=8)
    sd = ov3.random_state_dict(2, C, torch.Generator().manual_seed(C), registers=4, std=0.05 if C == 384 else 0.02)
    video = synth.random_video(T, H, W, seed=9)
    vit = DinoV3Features(sd, layer=1, stride=8, device=DEV)
    chans = [3, 64, 128, 256, C]
    model = build_tracker_from_video(video, vit, delta_channels=chans)
    assert model.dino_patch_size == 16 and (model._geom.h, model._geom.w) == (geo.h, geo.w) == (11, 14)
    ref_dino = ov3.dino_features_video(video.double(), {k: v.double() for k, v in sd.items()}, 1, stride=8).float()
    got_dino = model.dino_embed_video.cpu()
    assert (got_dino - ref_dino).abs().max().item() <= 5e-3 * ref_dino.abs().max().item()
    dsd = od.random_state_dict(chans, torch.Generator().manual_seed(10), last_std=0.05)
    model.delta_dino.load_state_dict(dsd)
    head = synth.head_weights("sharp", seed=3)
    model.tracker_head.load_state_dict(head)
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)   # refines the features
    ref_refined = od.refined_features(video, got_dino.contiguous(), dsd, patch=14, stride=8)
    assert (model.refined_features.cpu() - ref_refined).abs().max().item() <= 1e-4
    q = synth.lattice_query_points(2, 2, H, W, t_q=[0, 1, 2, 3], margin=10.0, jitter_seed=1)
    traj, occ = mi.infer(q.to(DEV))
    t_ref, o_ref = oi.infer(model.refined_features.cpu().contiguous(), q, head, geo, 0.7, 0.6)
    assert (traj.cpu() - t_ref).abs().max().item() <= XY_TOL
    assert torch.equal(occ.cpu(), o_ref)

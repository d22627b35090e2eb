"""GPU: tracking on the token grids of 8-pixel-patch backbones (DINO v1 ViT-S/8, ViT-B/8 at stride 7).

At 476 x 854 the grid is 67 x 121 as at patch 14, but token c sits at pixel 4 + 7 c instead of 7 + 7 c.  That offset
enters make_geom, normalize_points_for_sampling, the head's coordinate grid, the training step's reverse pass, the cycle
term and the contrastive coordinate grid (get_vit_feature_coords_from_mask with patch_size = config['dino_patch_size']).
Every check runs a Tracker(dino_patch_size=8) with the shipped delta-DINO channels [3, 64, 128, 256, C], C = 384 and
768, against the oracle at Geometry(patch=8) with the existing bars: |dxy| <= 1e-3 px and identical occlusion for
`infer`; the reverse pass against float64 (test_train_backward_gpu.py's bound and pinned kappas); the cycle preds and
their gradients as in test_cycle_gpu.py; both contrastive losses and their gradients as in test_contrastive_gpu.py.
Delta-DINO's CNN alignment and the best-buddy preprocessing keep the reference's patch 14 (DESIGN 4.10)."""
import numpy as np
import pytest
import torch

import oracle
from oracle import contrastive as oc
from oracle import delta_dino as od
from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle import vit_dino_v1 as ov1
from oracle.tracker import Geometry

import test_cycle_gpu as tcy
import test_train_backward_gpu as tb
import track_reverse as tr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XY_TOL = 1e-3
GEO8 = Geometry(H=476, W=854, patch=8)
WIDTHS = (384, 768)


def _tracker(geo, feats, head=None, **kw):
    from dino_tracker_b200 import Tracker
    T, C = feats.shape[:2]
    m = Tracker(video=kw.pop("video", torch.zeros(T, 3, geo.H, geo.W, device=DEV)), dino_embed_video=feats, device=DEV,
                dino_patch_size=geo.patch, stride=geo.stride, delta_channels=[3, 64, 128, 256, C], **kw)
    if head is not None:
        m.tracker_head.load_state_dict(head)
    return m


def test_geometry_at_patch_8():
    from dino_tracker_b200 import _lib
    g = _lib.make_geom(GEO8.H, GEO8.W, 8, 7, 35)
    assert (g.h, g.w) == (GEO8.h, GEO8.w) == (67, 121)
    assert (Geometry(H=480, W=856, patch=8).h, Geometry(H=480, W=856, patch=8).w) == (68, 122)


@pytest.mark.parametrize("kind", ["sharp", "well", "mixed"])
@pytest.mark.parametrize("C", WIDTHS)
def test_infer_matches_oracle(C, kind):
    from dino_tracker_b200 import ModelInference, _lib
    T = 4
    feats, _ = synth.shifted_field_features(T, C, GEO8.h, GEO8.w, seed=C + 3, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=C)
    q = synth.lattice_query_points(4, 3, GEO8.H, GEO8.W, t_q=[i % T for i in range(12)], margin=10.0, jitter_seed=C)
    m = _tracker(GEO8, feats, head)
    pn = m.normalize_points_for_sampling(q.to(DEV))
    assert torch.allclose(pn.cpu(), ot.normalize_points_for_sampling(q, GEO8), rtol=0, atol=1e-6)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    traj, occ = mi.infer(q.to(DEV))
    torch.cuda.synchronize()
    stats = _lib.infer_stats()
    oracle.use_exact_fp32()
    with torch.no_grad():
        t_ref, o_ref = oi.infer(feats.to(DEV), q.to(DEV), {k: v.to(DEV) for k, v in head.items()}, GEO8, 0.7, 0.6)
    err = (traj - t_ref).abs().max().item()
    print(f"[patch 8, C={C}, {kind}] max |dxy| = {err:.2e} px, {stats}")
    assert err <= XY_TOL
    assert torch.equal(occ.cpu(), o_ref.cpu())


def _run_production(label, geo, feats, head, pts, tgt_slot, gout):
    """test_train_backward_gpu.run_production on a Tracker at geo's patch."""
    from dino_tracker_b200 import _lib
    from dino_tracker_b200 import train as dtrain
    m = _tracker(geo, feats, corr_precision="fp16x3")
    wts = tr.normalized_weights(head, device=DEV)
    emb = tb._tpc(feats.to(DEV)).contiguous()
    out, hw, saved = dtrain.track_forward(m, emb, *wts, pts.to(DEV), tgt_slot.to(DEV))
    emb, norms, pts_sorted, desc, dn, tgt_sorted, maps, aux, order, slots = saved
    feat = _lib.make_features(emb, norms)
    return tb.check_track_backward(label, feats, slots, pts_sorted, tgt_sorted, wts, geo, gout.to(DEV)[order], maps, aux,
                                   feat, m._geom, hw, desc, dn)


@pytest.mark.parametrize("kind", ["sharp", "well"])
@pytest.mark.parametrize("C", WIDTHS)
def test_training_step_reverse_against_float64(C, kind):
    """The training step's reverse pass at 476 x 854, N = 4, B = 512, patch 8."""
    feats, _ = synth.shifted_field_features(4, C, GEO8.h, GEO8.w, seed=111, noise=0.2, max_shift=2)
    gen = tb._gen("patch8", C, kind)
    pts, tgt, gout = tb._batch(GEO8, 4, 512, gen)
    _run_production(f"patch 8 C={C} {kind}", GEO8, feats, synth.head_weights(kind, seed=111), pts, tgt, gout)


@pytest.mark.parametrize("C", WIDTHS)
def test_cycle_preds_match_per_pair_reference(C):
    T = 6
    feats, _ = synth.shifted_field_features(T, C, GEO8.h, GEO8.w, seed=91, noise=0.1, max_shift=2)
    m = _tracker(GEO8, feats, synth.head_weights("sharp", seed=93),
                 video=synth.random_video(T, GEO8.H, GEO8.W, seed=92).to(DEV), cyc_n_frames=4, cyc_batch_size_per_frame=256,
                 cyc_fg_points_ratio=0.7, cyc_thresh=4)
    m.delta_dino.load_state_dict(od.random_state_dict([3, 64, 128, 256, C], torch.Generator().manual_seed(94), last_std=0.02))
    m.train()
    fg = torch.zeros(T, GEO8.H, GEO8.W, device=DEV)
    fg[:, 100:380, 200:650] = 1
    fs = torch.tensor([0, 1, 2, 3], dtype=torch.int64)
    g = torch.Generator().manual_seed(95)
    B = 64
    pts = torch.rand(B, 3, generator=g) * torch.tensor([GEO8.W - 1.0, GEO8.H - 1.0, 0.0])
    m((pts.to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), fs))
    emb = m.frame_embeddings
    params = list(m.tracker_head.parameters())
    torch.manual_seed(6)
    got = m.get_cycle_consistent_preds(fs, fg)
    torch.manual_seed(6)
    _, want, _ = tcy._reference_preds(m, fs, fg)
    n = want["source_coords"].shape[0]
    assert n > 0 and got["source_coords"].shape[0] == n
    assert torch.equal(got["source_coords"], want["source_coords"])
    to_px = torch.tensor([GEO8.W - 1, GEO8.H - 1], device=DEV) / 2
    for k in ("source_target_coords", "target_source_coords"):
        assert ((got[k] - want[k]).abs() * to_px).max().item() <= XY_TOL, k
    g_got = torch.autograd.grad(tcy._cycle_loss(got), [emb] + params, retain_graph=True)
    g_want = torch.autograd.grad(tcy._cycle_loss(want), [emb] + params, retain_graph=True)
    for a, b in zip(g_got, g_want):
        assert b.abs().max().item() > 0 and tcy._rel(a, b) <= tcy.GRAD_TOL


@pytest.mark.parametrize("which", ["dino", "refined"])
@pytest.mark.parametrize("C", WIDTHS)
def test_contrastive_losses_match_oracle(C, which):
    """Both losses on the contrastive fixture's best buddies and masks (98 x 126: 13 x 17 tokens at patch 8 and 14),
    C-wide smooth embeddings, config['dino_patch_size'] = 8, against the oracle in float64 (same draws), with
    test_contrastive_gpu.py's bars at the shipped shape: loss 1.5e-5, gradient 1e-4 (relative to max |grad|)."""
    from dino_tracker_b200 import contrastive as c
    from oracle import make_golden_contrastive as mg
    from test_contrastive_gpu import smooth_frames
    z = np.load(mg.OUT)
    geo = Geometry(H=mg.H, W=mg.W, patch=8)
    emb0 = smooth_frames(mg.T, C, geo.h, geo.w, seed=C)
    video = torch.zeros(mg.T, 3, mg.H, mg.W)
    cfg = dict(mg.CONFIG, dino_patch_size=8)
    fs = torch.tensor(mg.FRAMES)
    kw = dict(batch_size=cfg["cl_n_frames"], points_per_pair=cfg["cl_points_per_pair"], fg_points_ratio=cfg["cl_fg_points_ratio"])
    res = {}
    for owner in (c, oc):
        trn = mg.trainer_standin(type("T", (), {}), torch.from_numpy(z["masks"]), mg.load_bb(z))
        trn.config = dict(cfg)
        dt = torch.float32 if owner is c else torch.float64
        emb = emb0.to(DEV, dt).clone().requires_grad_(True)
        model = oc.ModelStandIn(video.to(dt), emb, stride=mg.STRIDE, dino_patch_size=8)
        torch.manual_seed(7)
        if which == "dino":
            loss = owner.get_dino_bb_contrastive_loss(trn, model, fs)
        else:
            loss = owner.get_refined_bb_contrastive_loss(trn, model, fs, emb, temp=cfg["cl_temp"], cl_div=cfg["cl_div_ref_bb"], **kw)
        loss.backward()
        res[owner is c] = (loss.item(), emb.grad.clone())
    (l_got, g_got), (l_ref, g_ref) = res[True], res[False]
    le = abs(l_got - l_ref) / abs(l_ref)
    ge = float((g_got.double() - g_ref).abs().max() / g_ref.abs().max())
    print(f"patch 8 {which} C={C}: loss {l_got:.6g} vs {l_ref:.6g} (rel {le:.2e}), grad rel err {ge:.2e}")
    assert l_ref != 0 and le <= 1.5e-5 and ge <= 1e-4


def test_pixels_to_tracks_vits8():
    """ViT-S/8 (384 wide, 6 heads, 2 blocks) -> delta-DINO -> infer, against the chained oracles."""
    from dino_tracker_b200 import DinoV2Features, ModelInference, build_tracker_from_video
    H, W, T = 98, 126, 4
    geo = Geometry(H=H, W=W, patch=8)
    _, D, heads = ov1.CONFIGS["dino_vits8"]
    sd = ov1.random_state_dict(2, D, torch.Generator().manual_seed(8), std=0.05)
    video = synth.random_video(T, H, W, seed=9)
    vit = DinoV2Features.from_name("dino_vits8", sd, layer=1, device=DEV)
    chans = [3, 64, 128, 256, D]
    model = build_tracker_from_video(video, vit, delta_channels=chans)
    assert model.dino_patch_size == 8 and (model._geom.h, model._geom.w) == (geo.h, geo.w)
    dsd = od.random_state_dict(chans, torch.Generator().manual_seed(10), last_std=0.05)
    model.delta_dino.load_state_dict(dsd)
    head = synth.head_weights("sharp", seed=3)
    model.tracker_head.load_state_dict(head)
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)
    ref_dino = ov1.dino_features_video(video, sd, heads, 1)
    got_dino = model.dino_embed_video.cpu()
    assert (got_dino - ref_dino).abs().max().item() <= 5e-3 * ref_dino.abs().max().item()
    ref_refined = od.refined_features(video, got_dino.contiguous(), dsd)
    assert (model.refined_features.cpu() - ref_refined).abs().max().item() <= 1e-4
    q = synth.lattice_query_points(2, 2, H, W, t_q=[0, 1, 2, 3], margin=10.0, jitter_seed=1)
    traj, occ = mi.infer(q.to(DEV))
    t_ref, o_ref = oi.infer(model.refined_features.cpu().contiguous(), q, head, geo, 0.7, 0.6)
    assert (traj.cpu() - t_ref).abs().max().item() <= XY_TOL
    assert torch.equal(occ.cpu(), o_ref)

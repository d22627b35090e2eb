"""GPU parity on BASELINE.json's own configurations, against the fp32 oracle running on the same GPU.

The oracle (``oracle/``) is device-agnostic PyTorch; on ``cuda`` with TF32 disabled (``oracle.use_exact_fp32()``)
it is the reference's PyTorch-CUDA arithmetic (fp32 matmuls / convolutions, same op sequence) and finishes the
full-size configurations in seconds.  Bars (BASELINE.json north_star): |dxy| <= 1e-3 px on trajectories,
occlusion masks and anchor sets bit-exact.  Every test prints the numbers DESIGN.md quotes.

  * config 2: 854x476, T=50, C=1024, 256 query points exactly as bench.py builds it -- heads sharp / well / mixed
  * config 1: 8 frames, 16 grid query points, C=1024 (ViT-L/14@15) and C=768 (ViT-B/14)
  * delta-DINO at the shipped widths [3, 64, 128, 256, 1024] on 476x854 frames
  * ViT-L/14@block15 and ViT-B/14@block11 on an 854x476 frame, and the pixels -> tracks chain
  * regression tests for the round-1 advisor findings (split cache ABA, N x T x 2 trajectories, index validation)
"""
import numpy as np
import pytest
import torch

import oracle
from oracle import delta_dino as od
from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle import vit as ovit
from oracle.tracker import Geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XY_TOL = 1e-3


def _tracker(feats, head, precision="fp16x3", T=None):
    from dino_tracker_b200 import ModelInference, Tracker
    T = feats.shape[0]
    video = torch.zeros(T, 3, 476, 854, device=DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=[3, 4, 4, 4, feats.shape[1]],
                corr_precision=precision)
    m.tracker_head.load_state_dict(head)
    return m, ModelInference(m, m.range_normalizer, 0.7, 0.6)


def _compare_infer(r, sub, feats, q, head, geo, label):
    """CUDA result dict ``r`` (all query points) against the oracle on the query subset ``sub`` (same device)."""
    oracle.use_exact_fp32()
    head_dev = {k: v.to(DEV) for k, v in head.items()}
    with torch.no_grad():
        t_ref, o_ref, aux = oi.infer(feats, q[sub], head_dev, geo, 0.7, 0.6, return_all=True)
    traj, cos, occ = r["traj"][sub], r["cos_sims"][sub], r["occ"][sub].bool()
    e_traj = (traj - aux["trajs"]).abs().max().item()
    e_cos = (cos - aux["cos_sims"]).abs().max().item()
    vis_ref = aux["cos_sims"] >= 0.7
    same_sets = torch.equal(cos >= 0.7, vis_ref)
    # anchor tracks (intermediate): dense [N][T][T][2] rows of the anchor frames vs the oracle's {n: M_n x T x 2}
    worst, n_bad, n_tot = 0.0, 0, 0
    for j in range(len(sub)):
        got = r["anchors"][sub[j]][vis_ref[j]]
        d = (got - aux["anchors"][j]).abs().amax(dim=-1)
        worst = max(worst, d.max().item() if d.numel() else 0.0)
        n_bad += int((d > XY_TOL).sum().item())
        n_tot += d.numel()
    occ_same = torch.equal(occ, o_ref)
    print(f"[{label}] {len(sub)} query points vs the GPU fp32 oracle: traj max |dxy| = {e_traj:.2e} px, cos-sims {e_cos:.2e}, "
          f"anchor sets {'identical' if same_sets else 'DIFFER'}, anchor tracks max {worst:.2e} px "
          f"({n_bad} of {n_tot} beyond {XY_TOL} px), occlusion {'identical' if occ_same else 'DIFFERS'}")
    assert e_traj <= XY_TOL
    assert e_cos <= 1e-4      # intermediate: sampled AT the predicted points, so it inherits d(cos)/d(px) * the track difference
    assert same_sets
    assert occ_same
    # intermediate anchor tracks: an arg-max near-tie between two tokens (a < 1e-6 gap in cosine) may legitimately
    # resolve differently under a different fp32 summation order; the outputs above are what the bar is stated on
    assert n_bad <= max(2, n_tot // 20000), f"{n_bad} of {n_tot} anchor tracks differ by more than {XY_TOL} px"
    return e_traj


@pytest.mark.parametrize("kind", ["sharp", "well", "mixed"])
def test_config2_full_size_against_gpu_oracle(kind):
    """BASELINE configs[1] exactly as bench.py builds it: T=50, C=1024, 256 lattice query points at t=0."""
    import bench
    from bench_inputs import sharp_head
    T, C, nq = 50, 1024, 256
    feats = bench.synth_video_features(T, C, DEV, 1234, 0.25)
    q = bench.query_lattice(nq, 0).to(DEV)
    head = sharp_head(0) if kind == "sharp" else synth.head_weights(kind, seed=0)
    geo = Geometry()
    m, mi = _tracker(feats, head)
    r = mi.infer_all(q)
    torch.cuda.synchronize()
    assert torch.equal(m.refined_features, feats)          # default delta-DINO: zero residual
    # 32 query points spread over the 16 x 16 lattice (every row and column is hit); 256 for the bench head
    sub = list(range(nq)) if kind == "sharp" else [(i * 8 + (i // 2) % 8) % nq for i in range(32)]
    _compare_infer(r, sub, feats, q, head, geo, f"config 2, {kind} head")


@pytest.mark.parametrize("C", [1024, 768])
def test_config1_against_gpu_oracle(C):
    """BASELINE configs[0] shape: 8 frames, 16 grid query points, full 67 x 121 token geometry."""
    geo = Geometry()
    T = 8
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=70 + C, noise=0.2, max_shift=2)
    feats = feats.to(DEV)
    head = synth.head_weights("sharp", seed=70)
    q = synth.lattice_query_points(4, 4, geo.H, geo.W, t_q=0, margin=60.0, jitter_seed=70).to(DEV)
    for prec in ("fp16x3", "fp32"):
        m, mi = _tracker(feats, head, prec)
        r = mi.infer_all(q)
        _compare_infer(r, list(range(16)), feats, q, head, geo, f"config 1, C={C}, {prec}")


def test_delta_dino_shipped_widths_against_gpu_oracle():
    """a2 at the widths the reference ships ([3, 64, 128, 256, 1024], models/networks/delta_dino.py:10) on full frames:
    the convolution GEMM with 256-column tiles, K = 6400 and dilation 2 that bench.py times."""
    from dino_tracker_b200 import Tracker
    oracle.use_exact_fp32()
    channels = [3, 64, 128, 256, 1024]
    H, W, T = 476, 854, 2
    geo = Geometry()
    sd = od.random_state_dict(channels, torch.Generator().manual_seed(81), last_std=0.01)
    video = synth.random_video(T, H, W, seed=82).to(DEV)
    dino = synth.random_features(T, 1024, geo.h, geo.w, seed=83).to(DEV)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = od.refined_features(video, dino, sd_dev)
        ref_res = ref - dino
    for prec in ("fp16x3", "fp32"):
        m = Tracker(video=video, dino_embed_video=dino, device=DEV, delta_channels=channels)
        m.delta_dino.conv_precision = prec
        m.delta_dino.load_state_dict(sd)
        m.cache_refined_embeddings()
        got = m.refined_features
        err = (got - ref).abs().max().item()
        res_scale = ref_res.abs().max().item()
        print(f"[delta-DINO shipped widths, {prec}] max |refined - oracle| = {err:.2e} (residual scale {res_scale:.3f})")
        assert err <= 5e-5
        assert torch.allclose(m._refined_norms, got.flatten(2).norm(dim=1), rtol=1e-5)
        del m


VIT_CASES = {"dinov2_vitl14": dict(layer=15), "dinov2_vitb14": dict(layer=11)}


def _vit_sd(name, seed):
    depth, dim, heads = ovit.CONFIGS[name]
    layer = VIT_CASES[name]["layer"]
    sd = ovit.random_state_dict(layer + 1, dim, torch.Generator().manual_seed(seed), n_pos=37, std=0.02)
    return sd, dim, heads, layer


@pytest.mark.parametrize("name", sorted(VIT_CASES))
def test_vit_full_size_against_gpu_oracle(name):
    """a1 on one 854x476 frame (8108 tokens, 127 key tiles) for the shipped backbones, fused attention + fp16-operand GEMMs
    (the timed configuration) against the fp32 oracle.  The arithmetic is narrower than the reference's fp32; the error is
    reported and bounded here, its effect on the tracks is measured in test_pixels_to_tracks_full_size."""
    from dino_tracker_b200.vit import DinoV2Features
    oracle.use_exact_fp32()
    sd, dim, heads, layer = _vit_sd(name, 90)
    frame = synth.random_video(1, 476, 854, seed=91).to(DEV)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = ovit.dino_features_video(frame, sd_dev, heads, layer)           # 1 x C x 67 x 121
    ex = DinoV2Features(sd, heads=heads, layer=layer, device=DEV)
    got = ex.features_chw(frame)
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    rms = ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    cos = torch.nn.functional.cosine_similarity(got.flatten(2), ref.flatten(2), dim=1).min().item()
    print(f"[{name}@block{layer}, 854x476] max |diff| = {err:.3e} = {err / scale:.2e} of the feature scale {scale:.2f}; "
          f"relative RMS {rms:.2e}; min token cosine {cos:.7f}")
    assert err <= 5e-3 * scale
    assert cos > 0.9999


def test_vit_full_size_frames_per_call_invariance():
    """ViT-B/14@11 on three 854x476 frames with frames_per_call = 2 (a 2-frame call of 16216 rows, then a 1-frame call)
    must equal each frame run alone bit for bit: a token's row lands in another tile and another CTA of the pair, with
    the same arithmetic."""
    from dino_tracker_b200.vit import DinoV2Features
    sd, dim, heads, layer = _vit_sd("dinov2_vitb14", 92)
    video = synth.random_video(3, 476, 854, seed=93).to(DEV)
    alone = DinoV2Features(sd, heads=heads, layer=layer, device=DEV, frames_per_call=1)(video).clone()
    batched = DinoV2Features(sd, heads=heads, layer=layer, device=DEV, frames_per_call=2)(video)
    assert torch.equal(batched, alone), f"frames_per_call changes the features: {(batched - alone).abs().max().item()}"


def test_vit_full_size_cta_pairs_bit_identical():
    """ViT-L/14@15 on two 854x476 frames: the linear layers on CTA pairs and on single CTAs issue the same wgmma sequence
    per output row and share their epilogue arithmetic, so the features are bit-identical."""
    from dino_tracker_b200.vit import DinoV2Features
    sd, dim, heads, layer = _vit_sd("dinov2_vitl14", 94)
    video = synth.random_video(2, 476, 854, seed=95).to(DEV)
    pairs = DinoV2Features(sd, heads=heads, layer=layer, device=DEV, cta_pairs=True)(video).clone()
    single = DinoV2Features(sd, heads=heads, layer=layer, device=DEV, cta_pairs=False)(video)
    assert torch.equal(pairs, single), f"CTA pairs change the features: {(pairs - single).abs().max().item()}"


def _arg_max_tie(feats, query, frame, p_a, p_b, geo):
    """|difference| between the float64 correlation peaks nearest to the two candidate track points p_a, p_b (px) of
    `query` (x, y, t) in `frame`."""
    pn = ot.normalize_points_for_sampling(query[None].float(), geo)
    desc = ot.sample_descriptors(feats, torch.cat([pn[:, :2], query[None, 2:3].float()], 1)).double()[0]
    f = feats[frame].double().reshape(feats.shape[1], -1)
    corr = (desc @ f) / (desc.norm() * f.norm(dim=0)).clamp_min(1e-8)
    corr = corr.reshape(geo.h, geo.w)
    peaks = []
    for p in (p_a, p_b):
        c = int(round((float(p[0]) - geo.patch // 2) / geo.stride)); rr = int(round((float(p[1]) - geo.patch // 2) / geo.stride))
        peaks.append(corr[max(rr - 5, 0):rr + 6, max(c - 5, 0):c + 6].max().item())
    return abs(peaks[0] - peaks[1])


def test_pixels_to_tracks_full_size():
    """ViT-L/14@15 -> delta-DINO (shipped widths) -> infer on an 854x476, T=6 clip, chained CUDA stages vs chained oracle
    stages from the SAME pixels.  Reports the track deviation caused by the fp16-operand ViT; the tracker stage itself is
    held to the parity bar on identical features."""
    from dino_tracker_b200 import DinoV2Features, ModelInference, build_tracker_from_video
    oracle.use_exact_fp32()
    name, T = "dinov2_vitl14", 6
    sd, dim, heads, layer = _vit_sd(name, 95)
    geo = Geometry()
    # a translating textured clip: smooth noise shifted by whole pixels per frame
    g = torch.Generator().manual_seed(96)
    base = torch.rand(3, 476 + 64, 854 + 64, generator=g)
    base = torch.nn.functional.avg_pool2d(base[None], 5, 1, 2)[0]
    video = torch.stack([base[:, 32 + 3 * t: 32 + 3 * t + 476, 32 + 5 * t: 32 + 5 * t + 854] for t in range(T)]).to(DEV)
    channels = [3, 64, 128, 256, dim]
    dsd = od.random_state_dict(channels, torch.Generator().manual_seed(97), last_std=0.01)
    head = synth.head_weights("sharp", seed=98)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=0, margin=80.0, jitter_seed=99).to(DEV)

    vit = DinoV2Features(sd, heads=heads, layer=layer, device=DEV)
    model = build_tracker_from_video(video, vit, device=DEV, delta_channels=channels)
    model.delta_dino.load_state_dict(dsd)
    model.tracker_head.load_state_dict(head)
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)
    r = mi.infer_all(q)

    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    dsd_dev = {k: v.to(DEV) for k, v in dsd.items()}
    head_dev = {k: v.to(DEV) for k, v in head.items()}
    with torch.no_grad():
        ref_dino = ovit.dino_features_video(video, sd_dev, heads, layer)
        ref_refined = od.refined_features(video, ref_dino, dsd_dev)
        t_ref, o_ref, aux = oi.infer(ref_refined, q, head_dev, geo, 0.7, 0.6, return_all=True)
        # tracker stage on OUR refined features (identical inputs): the parity bar proper
        ours = model.refined_features.contiguous()
        t_same, o_same, aux_same = oi.infer(ours, q, head_dev, geo, 0.7, 0.6, return_all=True)
    e_feat = (model.refined_features - ref_refined).abs().max().item() / ref_refined.abs().max().item()
    e_pix = (r["traj"][..., :2] - t_ref).abs().max().item()
    e_same = (r["traj"][..., :2] - t_same).abs().max().item()
    occ_pix = int((r["occ"].bool() != o_ref).sum().item())
    print(f"[pixels -> tracks, {name}@{layer}, T={T}, {q.shape[0]} query points] refined features {e_feat:.2e} of scale; "
          f"tracks vs chained oracle from pixels: max |dxy| = {e_pix:.3e} px, occlusion flags differing {occ_pix}; "
          f"tracker stage on identical features: max |dxy| = {e_same:.2e} px")
    # The features of a random-weight ViT are smooth enough for a correlation map to hold two far-apart peaks of equal
    # height: which one is the arg-max (tracker_head.py:115-116) then depends on the fp32 summation order.  A trajectory point
    # beyond the bar is accepted only if float64 shows exactly that: the peaks under the two answers differ by < 5e-6, the
    # near-tie bound delta of DESIGN.md 3.1 (tests/test_fp16_range_gpu.py drives it with twin peaks).
    dev = (r["traj"][..., :2] - t_same).abs().amax(-1)
    far = (dev > XY_TOL).nonzero().tolist()
    assert len(far) <= max(1, dev.numel() // 50), far
    for n, t in far:
        assert _arg_max_tie(ours, q[n], t, r["traj"][n, t, :2], t_same[n, t], geo) < 5e-6, (n, t)
    ok = dev <= XY_TOL
    e_pix = ((r["traj"][..., :2] - t_ref).abs().amax(-1) * ok).max().item()
    print(f"    arg-max ties (float64-verified): {len(far)} of {dev.numel()} trajectory points")
    assert torch.equal(r["occ"].bool(), o_same)
    assert e_pix <= 0.5          # the fp16-operand ViT moves tracks by a small fraction of a token (7 px); reported above


# ---------------------------------------------------------------------------- advisor regressions (round 1)
def test_uncached_forward_twice_uses_fresh_split():
    """ADVICE r1 (medium): forward() without cached embeddings, called twice with different frame sets in fp16x3 mode,
    must not correlate against the fp16 split of the previous frame set (stale cache keyed by a recycled address)."""
    from dino_tracker_b200 import Tracker
    geo = Geometry(H=98, W=126)
    T, C, B = 6, 64, 40
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=51, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=51)
    video = torch.zeros(T, 3, geo.H, geo.W, device=DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=[3, 4, 4, 4, C], corr_precision="fp16x3")
    m.tracker_head.load_state_dict(head)
    g = torch.Generator().manual_seed(52)
    scale = torch.tensor([geo.W - 1, geo.H - 1]) / 2
    for fs in ([0, 1, 2], [3, 4, 5], [5, 0, 3]):
        frames_set = torch.tensor(fs, dtype=torch.int32)
        pts = torch.rand(B, 3, generator=g) * torch.tensor([geo.W - 1.0, geo.H - 1.0, 0.0])
        src = torch.randint(0, 3, (B,), generator=g)
        tgt = torch.full((B,), 1, dtype=torch.long)          # > 8 maps on one frame: tensor-core GEMM path
        inp = (pts.to(DEV), src.to(DEV), tgt.to(DEV), frames_set.to(DEV))
        with torch.no_grad():        # the inference kernels (with gradients enabled forward() builds the training graph)
            out = m(inp).cpu()
        ref = ot.tracker_forward(feats, (pts, src, tgt, frames_set), head, geo)
        assert ((out - ref).abs() * scale).max().item() <= XY_TOL, fs
        # training-style consumers read the refined embeddings of the frame set (models/tracker.py:319-322)
        assert torch.equal(m.frame_embeddings.cpu(), feats[frames_set.long()])
        assert m.residual_embeddings.abs().max().item() == 0.0


def test_occlusion_accepts_xy_trajectories_and_validates():
    """ADVICE r1 (low): compute_occlusion with N x T x 2 trajectories (what infer returns) == N x T x 3; bad shapes and
    out-of-range frame indices raise instead of reading out of bounds."""
    from dino_tracker_b200 import ModelInference, Tracker
    geo = Geometry(H=98, W=126)
    T, C = 5, 32
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=61, noise=0.15, max_shift=2)
    head = synth.head_weights("sharp", seed=61)
    m = Tracker(video=torch.zeros(T, 3, geo.H, geo.W, device=DEV), dino_embed_video=feats, device=DEV,
                delta_channels=[3, 4, 4, 4, C])
    m.tracker_head.load_state_dict(head)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    q = synth.lattice_query_points(3, 2, geo.H, geo.W, t_q=[0, 1, 2, 3, 4, 0], margin=12.0, jitter_seed=61).to(DEV)
    traj3 = mi.compute_trajectories(q)
    cos = mi.compute_trajectory_cos_sims(traj3, q)
    anchors = mi.compute_anchor_trajectories(traj3, cos)
    occ3 = mi.compute_occlusion(traj3, cos, anchors)
    occ2 = mi.compute_occlusion(traj3[..., :2].contiguous(), cos, anchors)
    assert torch.equal(occ3, occ2)
    assert torch.equal(occ3, mi.infer(q)[1])
    with pytest.raises(ValueError):
        mi.compute_occlusion(traj3[..., :1], cos, anchors)
    with pytest.raises(IndexError):
        m((q[:, :3], torch.zeros(6, dtype=torch.long), torch.ones(6, dtype=torch.long), torch.tensor([0, T])))
    with pytest.raises(IndexError):
        m((q[:, :3], torch.zeros(6, dtype=torch.long), torch.full((6,), 2), torch.tensor([0, 1])))

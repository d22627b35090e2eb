"""Token grids beyond 128 x 128 and 8,192 tokens, up to the supported envelope (h, w <= 256, h * w <= 32,768): the head
(full-map kernel for wide / tall grids, both fast paths), inference on both anchor pipelines, the training step's
reverse pass (map buffers in global memory), the cycle term, the contrastive node and the feature stages, against
the oracle on the same GPU in exact fp32 (float64 where the suites of those stages use it).  Bars as everywhere: |dxy| <= 1e-3 px, identical occlusion, gradients within
2e-3 of the largest oracle entry.

Shapes: 98 x 1792 (13 x 255 tokens: wide only), 1792 x 98 (255 x 13: tall only), 966 x 546 (77 x 137 = 10,549 tokens,
beyond the old 64-tile coarse-pass limit), 1274 x 714 / 714 x 1274 (18,281 tokens) and 1274 x 1274 (32,761 tokens).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

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
GRAD_TOL = 2e-3
DINOTRK_EINVAL = -22


def _tracker(geo, feats, head, delta_channels=None):
    from dino_tracker_b200 import Tracker
    T, C = feats.shape[:2]
    video = torch.zeros(T, 3, geo.H, geo.W, device=DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=delta_channels or [3, 4, 4, 4, C])
    m.tracker_head.load_state_dict(head)
    return m


def _head_call(geo, maps, head, fast):
    """dinotrk_head on maps [n][P] -> (out [n][2] normalised, aux [n][2], maps sent to the full-map kernel or None)."""
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    n = maps.shape[0]
    g = _lib.make_geom(geo.H, geo.W)
    m = _tracker(geo, torch.zeros(1, 8, geo.h, geo.w), head)
    buf = torch.zeros(n, lib.dinotrk_map_stride(ctypes.byref(g)), device=DEV)
    buf[:, : geo.P] = maps.to(DEV)
    out = torch.empty(n, 2, device=DEV)
    aux = torch.empty(n, 2, device=DEV, dtype=torch.int32)
    scratch = torch.zeros(n + 1, device=DEV, dtype=torch.int32) if fast else None
    rc = lib.dinotrk_head(_lib.ptr(buf), n, ctypes.byref(g), ctypes.byref(m.head_weights()), None, _lib.ptr(out), 2, 1,
                          _lib.ptr(aux), _lib.ptr(scratch), _lib.stream_ptr())
    _lib.check(rc, "head")
    torch.cuda.synchronize()
    return out, aux, (int(scratch[0]) if fast else None)


def _border_maps(geo, n, seed):
    """Relu'd maps with a peak per map: at the right / bottom borders and corners, an exact duplicate of the peak far
    away (first index wins), a flat map, and interior peaks."""
    g = torch.Generator().manual_seed(seed)
    h, w = geo.h, geo.w
    maps = torch.rand(n, h, w, generator=g) * 0.4
    spots = [(h // 2, w - 1), (h - 1, w // 2), (h - 1, w - 1), (0, w - 1), (h - 1, 0), (h // 2, w - 2), (h - 2, w - 3)]
    for i in range(n):
        if i == n - 1:
            maps[i] = 0.25
            continue
        r, c = spots[i] if i < len(spots) else (int(torch.randint(0, h, (1,), generator=g)), int(torch.randint(0, w, (1,), generator=g)))
        rr = torch.arange(h)[:, None].float()
        cc = torch.arange(w)[None, :].float()
        maps[i] = torch.maximum(maps[i], 0.95 * torch.exp(-((rr - r) ** 2 + (cc - c) ** 2) / 3.0))
        maps[i, r, c] = 0.99
        if i % 3 == 1:   # duplicate peak in the opposite quadrant: a tie the window certificate cannot settle alone
            maps[i, (r + h // 2) % h, (c + w // 2) % w] = 0.99
    return maps.reshape(n, h * w)


@pytest.mark.parametrize("H,W", [(98, 1792), (1792, 98), (546, 966), (98, 1799), (714, 1274), (1274, 1274)])
@pytest.mark.parametrize("kind", ["sharp", "well", "mixed", "default"])
@pytest.mark.parametrize("fast", [False, True])
def test_head_matches_oracle(H, W, kind, fast):
    """Every map through the full-map kernel (no scratch) or the window kernel with its queue, on maps built to defeat
    the fast path; the "default" head puts maps on the stability branch (whole-map softmax)."""
    oracle.use_exact_fp32()
    geo = Geometry(H=H, W=W)
    n = 24
    maps = _border_maps(geo, n, seed=H + W)
    head = synth.head_weights(kind, seed=7)
    out, aux, n_slow = _head_call(geo, maps, head, fast)
    head_dev = {k: v.to(DEV) for k, v in head.items()}
    ref, raux = ot.head_forward(maps.to(DEV).reshape(n, 1, geo.h, geo.w), head_dev, geo, return_aux=True)
    assert torch.equal(aux[:, 0].long(), raux["argmax"])
    assert torch.equal(aux[:, 1].bool(), raux["fallback"])
    scale = torch.tensor([geo.W - 1, geo.H - 1], device=DEV) / 2
    err = ((out - ref).abs() * scale).max().item()
    print(f"[head {geo.h}x{geo.w} {kind} {'window+queue' if fast else 'full map'}] max |dxy| = {err:.2e} px"
          + (f", {n_slow}/{n} maps queued" if fast else ""))
    assert err <= XY_TOL
    if fast and kind == "default":
        assert n_slow > 0


def _infer_both_paths(geo, T, C, nq, kind, seed):
    from dino_tracker_b200 import ModelInference, _lib
    lib = _lib.load()
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.2, max_shift=2)
    feats = feats.to(DEV)
    head = synth.head_weights(kind, seed=seed)
    nx = max(2, int(round((nq * geo.W / geo.H) ** 0.5)))
    ny = max(1, nq // nx)
    margin = min(20.0, geo.H / 4, geo.W / 4)
    q = synth.lattice_query_points(nx, ny, geo.H, geo.W, t_q=[i % T for i in range(nx * ny)], margin=margin,
                                   jitter_seed=seed).to(DEV)
    m = _tracker(geo, feats, head)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    res = {}
    try:
        for path in (0, 1):
            lib.dinotrk_infer_set_path(path)
            traj, occ = mi.infer(q)
            torch.cuda.synchronize()
            res[path] = (traj.clone(), occ.clone(), _lib.infer_stats())
    finally:
        lib.dinotrk_infer_set_path(-1)
    oracle.use_exact_fp32()
    head_dev = {k: v.to(DEV) for k, v in head.items()}
    with torch.no_grad():
        t_ref, o_ref = oi.infer(feats, q, head_dev, geo, 0.7, 0.6)
    return res, t_ref, o_ref


@pytest.mark.parametrize("H,W,T,C,nq,kind", [
    (98, 1792, 4, 64, 12, "sharp"),
    (1792, 98, 4, 64, 12, "well"),
    (546, 966, 5, 64, 16, "mixed"),
    (714, 1274, 6, 128, 16, "sharp"),
    (1274, 714, 6, 128, 16, "well"),
    (1274, 1274, 6, 128, 12, "mixed"),
    (714, 1274, 4, 1024, 8, "sharp"),
])
def test_infer_both_pipelines_match_oracle(H, W, T, C, nq, kind):
    geo = Geometry(H=H, W=W)
    res, t_ref, o_ref = _infer_both_paths(geo, T, C, nq, kind, seed=H * 3 + W + C)
    for path, (traj, occ, st) in res.items():
        err = (traj - t_ref).abs().max().item()
        print(f"[infer {geo.h}x{geo.w} T={T} C={C} {kind}, path {path}] max |dxy| = {err:.2e} px; {st}")
        assert err <= XY_TOL
        assert torch.equal(occ.bool(), o_ref.bool())
    assert (res[0][0] - res[1][0]).abs().max().item() <= XY_TOL
    assert torch.equal(res[0][1], res[1][1])
    st = res[1][2]
    assert st["pipeline"] == "exact-window"
    if geo.P >= 18281 and kind != "mixed":   # the mixed-sign head's logit bound leaves most small-T maps uncertified
        assert st["exact_window"] > 0


def test_infer_duplicate_tokens_queue_to_full_map():
    """Every frame carries an exact copy of the query tokens' features at the far side of a 255-wide grid: coarse
    candidates far apart, so the maps leave the exact window for the full-map path and must still meet the bar."""
    from dino_tracker_b200 import ModelInference, _lib
    lib = _lib.load()
    geo = Geometry(H=98, W=1792)
    T, C = 4, 64
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=31, noise=0.2, max_shift=1)
    half = geo.w // 2
    feats[:, :, :, half:2 * half] = feats[:, :, :, :half]
    feats = feats.to(DEV)
    head = synth.head_weights("sharp", seed=31)
    q = synth.lattice_query_points(8, 1, geo.H, geo.W, t_q=[i % T for i in range(8)], margin=20.0, jitter_seed=31).to(DEV)
    m = _tracker(geo, feats, head)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    try:
        lib.dinotrk_infer_set_path(1)
        traj, occ = mi.infer(q)
        torch.cuda.synchronize()
        st = _lib.infer_stats()
    finally:
        lib.dinotrk_infer_set_path(-1)
    oracle.use_exact_fp32()
    with torch.no_grad():
        t_ref, o_ref = oi.infer(feats, q, {k: v.to(DEV) for k, v in head.items()}, geo, 0.7, 0.6)
    err = (traj - t_ref).abs().max().item()
    print(f"[duplicate tokens {geo.h}x{geo.w}] max |dxy| = {err:.2e} px; {st}")
    assert st["full_map"] > 0
    assert err <= XY_TOL
    assert torch.equal(occ.bool(), o_ref.bool())


def _loss(coords, labels):
    return F.huber_loss(coords, labels, reduction="none", delta=1 / 32).mean()


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("H,W,kind", [(1792, 98, "well"), (714, 1274, "mixed"), (1274, 714, "sharp"), (1274, 1274, "well"),
                                      (714, 1274, "default"), (756, 1274, "sharp"), (1050, 917, "well")])
def test_training_step_gradients_match_oracle_autograd(H, W, kind):
    """Tracker.forward with gradients and dinotrk_track_backward (map buffers in the workspace beyond 11,560 tokens, the
    token list beyond 19,366) against autograd through the oracle; "default" puts the maps on the stability branch."""
    oracle.use_exact_fp32()
    geo = Geometry(H=H, W=W)
    N, C, B = 3, 64, 24
    feats, _ = synth.shifted_field_features(N, C, geo.h, geo.w, seed=41, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=41)
    g = torch.Generator().manual_seed(42)
    pts = torch.rand(B, 3, generator=g) * torch.tensor([geo.W - 1.0, geo.H - 1.0, 0.0])
    src, tgt = torch.randint(0, N, (B,), generator=g), torch.randint(0, N, (B,), generator=g)
    labels = torch.rand(B, 2, generator=g) * 2 - 1
    fs = torch.arange(N, dtype=torch.int32)
    inp = (pts.to(DEV), src.to(DEV), tgt.to(DEV), fs.to(DEV))
    f_o = feats.to(DEV).requires_grad_(True)
    head_o = {k: v.to(DEV).requires_grad_(True) for k, v in head.items()}
    c_o = ot.tracker_forward(f_o, inp, head_o, geo)
    _loss(c_o, labels.to(DEV)).backward()
    m = _tracker(geo, feats, head)
    emb = feats.to(DEV).clone().requires_grad_(True)
    c = m.get_point_predictions(inp, emb)
    _loss(c, labels.to(DEV)).backward()
    scale = torch.tensor([geo.W - 1, geo.H - 1], device=DEV) / 2
    err = ((c.detach() - c_o.detach()).abs() * scale).max().item()
    tol = 2e-2 if kind == "default" else GRAD_TOL   # stability branch: logits ~1e3 (as in test_train_gpu.py)
    ge = _rel(emb.grad, f_o.grad)
    w1 = _rel(m.tracker_head.cnn_refiner[0].weight.grad, head_o["cnn_refiner.0.weight"].grad)
    w2 = _rel(m.tracker_head.cnn_refiner[2].weight.grad, head_o["cnn_refiner.2.weight"].grad)
    print(f"[training step {geo.h}x{geo.w} {kind}] max |dxy| = {err:.2e} px, gradients: embeddings {ge:.1e}, "
          f"w1 {w1:.1e}, w2 {w2:.1e}")
    assert err <= XY_TOL
    assert ge <= tol and w1 <= tol and w2 <= tol


def test_cycle_term_matches_per_pair_reference_at_large_grid():
    """The cycle-consistency term at 1274 x 714 (train.yaml's counts: 4 pairs x 256 points, foreground ratio 0.7,
    threshold 4) against the per-pair restatement of models/tracker.py:182-301 on the public get_point_predictions
    (tests/test_cycle_gpu.py): same pixels and survivors, leg coordinates within the bar, and the cycle loss's gradients
    for the embeddings and the refiner within GRAD_TOL."""
    from dino_tracker_b200 import Tracker
    from test_cycle_gpu import _cycle_loss, _reference_preds
    geo = Geometry(H=714, W=1274)
    T, C = 6, 128
    chans = [3, 16, 16, 16, C]
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=51, noise=0.1, max_shift=2)
    m = Tracker(video=synth.random_video(T, geo.H, geo.W, seed=52).to(DEV), dino_embed_video=feats, device=DEV,
                delta_channels=chans, cyc_n_frames=4, cyc_batch_size_per_frame=256, cyc_fg_points_ratio=0.7, cyc_thresh=4)
    m.tracker_head.load_state_dict(synth.head_weights("sharp", seed=53))
    m.delta_dino.load_state_dict(od.random_state_dict(chans, torch.Generator().manual_seed(54), last_std=0.02))
    m.train()
    fg = torch.zeros(T, geo.H, geo.W, device=DEV)
    fg[1] = 1                                   # all foreground
    fg[2, 300:310, 600:610] = 1                 # 100 foreground pixels (< 179)
    fg[3:, 150:560, 300:1000] = 1               # frame 0: no foreground
    fs = torch.tensor([0, 1, 2, 3], dtype=torch.int64, device=DEV)
    g = torch.Generator().manual_seed(55)
    B = 64
    pts = torch.rand(B, 3, generator=g) * torch.tensor([geo.W - 1.0, geo.H - 1.0, 0.0])
    m((pts.to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), fs))
    emb = m.frame_embeddings
    params = list(m.tracker_head.parameters())
    torch.manual_seed(6)
    got = m.get_cycle_consistent_preds(fs, fg)
    torch.manual_seed(6)
    cyc, want, _ = _reference_preds(m, fs, fg)
    n = want["source_coords"].shape[0]
    assert n > 0 and got["source_coords"].shape[0] == n                          # same survivors
    assert torch.equal(got["source_coords"], want["source_coords"])               # same pixels
    to_px = torch.tensor([geo.W - 1, geo.H - 1], device=DEV) / 2
    errs = {k: ((got[k] - want[k]).abs() * to_px).max().item() for k in ("source_target_coords", "target_source_coords")}
    assert (got["cycle_consistency_dists"] <= m.cyc_thresh).all()
    g_got = torch.autograd.grad(_cycle_loss(got), [emb] + params, retain_graph=True)
    g_want = torch.autograd.grad(_cycle_loss(want), [emb] + params, retain_graph=True)
    gerr = [_rel(a, b) for a, b in zip(g_got, g_want)]
    print(f"[cycle term {geo.h}x{geo.w}] {n} survivors; legs max |dxy| {max(errs.values()):.2e} px; gradients {max(gerr):.1e}")
    assert max(errs.values()) <= XY_TOL
    for b, e in zip(g_want, gerr):
        assert b.abs().max().item() > 0 and e <= GRAD_TOL


def test_contrastive_node_at_1274x714_against_float64():
    """The best-buddy contrastive node (dinotrk_bb_contrastive_*: correlation GEMM over every token of the target frame,
    softmax, backward) on 101 x 181 token frames against float64 autograd, at the bars of the shipped shape."""
    from test_contrastive_gpu import BARS_SHIPPED, check, run_both, smooth_frames, tok
    oracle.use_exact_fp32()
    N, C, h, w = 4, 1024, 101, 181
    E = tok(smooth_frames(N, C, h, w, 7)).to(DEV)
    P = h * w
    g = torch.Generator().manual_seed(8)
    groups = [(0, 1, 0, 256), (2, 2, 256, 256), (3, 0, 512, 256), (1, 3, 768, 256)]
    S = torch.cat([E[s][torch.randint(P, (n,), generator=g).to(DEV)] for s, _, _, n in groups])
    U = torch.cat([E[t][torch.randint(P, (n,), generator=g).to(DEV)] for _, t, _, n in groups])
    check(run_both(E, S, U, groups, 0.1), BARS_SHIPPED, "1274x714")


def test_envelope_edges():
    """One token inside the envelope works; one token over returns DINOTRK_EINVAL with the envelope in the message from
    the head, inference and the training backward, never a fault."""
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    head = synth.head_weights("sharp", seed=3)
    geo = Geometry(H=98, W=1799)                  # 13 x 256
    assert geo.w == 256
    maps = _border_maps(geo, 4, seed=3)
    out, aux, _ = _head_call(geo, maps, head, fast=False)
    ref = ot.head_forward(maps.to(DEV).reshape(4, 1, geo.h, geo.w), {k: v.to(DEV) for k, v in head.items()}, geo)
    assert ((out - ref).abs() * torch.tensor([geo.W - 1, geo.H - 1], device=DEV) / 2).max().item() <= XY_TOL
    for H, W in [(98, 1806), (1806, 98), (1281, 1281)]:
        g = _lib.make_geom(H, W)
        assert max(g.h, g.w) > 256 or g.h * g.w > 32768
        stride = lib.dinotrk_map_stride(ctypes.byref(g))
        buf = torch.zeros(2, stride, device=DEV)
        o = torch.empty(2, 2, device=DEV)
        m = _tracker(Geometry(H=98, W=126), torch.zeros(1, 8, 13, 17), head)
        rc = lib.dinotrk_head(_lib.ptr(buf), 2, ctypes.byref(g), ctypes.byref(m.head_weights()), None, _lib.ptr(o), 2, 1, None,
                              None, _lib.stream_ptr())
        assert rc == DINOTRK_EINVAL and b"envelope" in lib.dinotrk_last_error(), (H, W, rc)
        # inference: rejected before the workspace is touched
        T, C, N = 2, 8, 1
        tpc = torch.zeros(T, g.h * g.w, C, device=DEV)
        norms = torch.ones(T, g.h * g.w, device=DEV)
        feat = _lib.make_features(tpc, norms)
        qp = torch.zeros(N, 3, device=DEV)
        traj = torch.empty(N, T, 2, device=DEV)
        ws = torch.empty(1 << 20, device=DEV, dtype=torch.uint8)
        rc = lib.dinotrk_infer(ctypes.byref(feat), ctypes.byref(g), ctypes.byref(m.head_weights()), _lib.ptr(qp), N, 0.7, 0.6,
                               0, 0, 0, 0, _lib.ptr(traj), None, None, None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        assert rc == DINOTRK_EINVAL and b"envelope" in lib.dinotrk_last_error(), (H, W, rc)
        rc = lib.dinotrk_track_backward(ctypes.byref(feat), ctypes.byref(g), ctypes.byref(m.head_weights()), _lib.ptr(qp),
                                        _lib.ptr(torch.zeros(1, device=DEV, dtype=torch.int32)), 1, _lib.ptr(tpc),
                                        _lib.ptr(norms), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(buf), _lib.ptr(o), 1,
                                        _lib.ptr(o), None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        assert rc == DINOTRK_EINVAL and b"envelope" in lib.dinotrk_last_error(), (H, W, rc)
    torch.cuda.synchronize()


def test_delta_dino_at_714x1274_against_gpu_oracle():
    """delta-DINO's inference forward (cached refined features, no graph) on 714 x 1274 frames."""
    from dino_tracker_b200 import Tracker
    oracle.use_exact_fp32()
    channels = [3, 64, 128, 256, 1024]
    H, W, T = 714, 1274, 2
    geo = Geometry(H=H, W=W)
    sd = od.random_state_dict(channels, torch.Generator().manual_seed(61), last_std=0.01)
    video = synth.random_video(T, H, W, seed=62).to(DEV)
    dino = synth.random_features(T, 1024, geo.h, geo.w, seed=63).to(DEV)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = od.refined_features(video, dino, sd_dev)
    m = Tracker(video=video, dino_embed_video=dino, device=DEV, delta_channels=channels)
    m.delta_dino.load_state_dict(sd)
    m.cache_refined_embeddings()
    err = (m.refined_features - ref).abs().max().item()
    print(f"[delta-DINO 714x1274] max |refined - oracle| = {err:.2e}")
    assert err <= 5e-5


def test_delta_dino_training_node_at_714x1274_against_float64():
    """delta-DINO's training node (train-mode BatchNorm forward and backward, tests/test_delta_train_gpu.py) on one
    714 x 1274 frame at the shipped widths: every parameter gradient against float64 autograd at the shipped bars."""
    from test_delta_train_gpu import TRAIN_TOL, _backward_case, _check_grads
    m, sd64 = _backward_case(714, 1274, 1, True, 80)
    _check_grads(m, sd64, "backward train 1x714x1274", TRAIN_TOL)


def test_vit_l_at_714x1274_against_gpu_oracle():
    """ViT-L/14@15 on one 714 x 1274 frame (18,282 tokens with the class token), fused attention against the fp32
    oracle, and the materialized attention (a 73 KiB softmax row) likewise."""
    from dino_tracker_b200.vit import DinoV2Features
    oracle.use_exact_fp32()
    depth, dim, heads = ovit.CONFIGS["dinov2_vitl14"]
    layer = 15
    sd = ovit.random_state_dict(layer + 1, dim, torch.Generator().manual_seed(71), n_pos=37, std=0.02)
    frame = synth.random_video(1, 714, 1274, seed=72).to(DEV)
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        ref = ovit.dino_features_video(frame, sd_dev, heads, layer)
    scale = ref.abs().max().item()
    for attention in ("fused", "materialized"):
        got = DinoV2Features(sd, heads=heads, layer=layer, device=DEV, attention=attention).features_chw(frame)
        err = (got - ref).abs().max().item()
        cos = F.cosine_similarity(got.flatten(2), ref.flatten(2), dim=1).min().item()
        print(f"[ViT-L/14@15 714x1274 {attention}] max |diff| = {err / scale:.2e} of the feature scale; min cosine {cos:.7f}")
        assert err <= 5e-3 * scale
        assert cos > 0.9999
        del got

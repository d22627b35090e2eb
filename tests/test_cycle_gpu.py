"""The cycle-consistency term (models/tracker.py:182-301) on the CUDA path against a per-pair restatement of the
algorithm on the public ``get_point_predictions`` and ``torch.randperm``, at train.yaml's shape (476 x 854, C = 1024, a
4-frame set, 4 pairs x 256 points, foreground ratio 0.7, threshold 4): same pixels, survivors and generator states, the
same leg coordinates, and the cycle loss's gradients for the embeddings and the refiner.  Source frames cover the edge
cases: no foreground, all foreground, fewer foreground pixels than a pair draws, and pairs with source slot = target slot.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import delta_dino as od
from oracle import synth
from oracle.tracker import Geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XY_TOL = 1e-3
GRAD_TOL = 2e-3
GEO = Geometry(H=476, W=854)
CHANS = [3, 16, 16, 16, 1024]


def _model():
    from dino_tracker_b200 import Tracker
    T, C = 6, 1024
    feats, _ = synth.shifted_field_features(T, C, GEO.h, GEO.w, seed=91, noise=0.1, max_shift=2)
    m = Tracker(video=synth.random_video(T, GEO.H, GEO.W, seed=92).to(DEV), dino_embed_video=feats, device=DEV,
                delta_channels=CHANS, cyc_n_frames=4, cyc_batch_size_per_frame=256, cyc_fg_points_ratio=0.7, cyc_thresh=4)
    m.tracker_head.load_state_dict(synth.head_weights("sharp", seed=93))
    m.delta_dino.load_state_dict(od.random_state_dict(CHANS, torch.Generator().manual_seed(94), last_std=0.02))
    m.train()
    fg = torch.zeros(T, GEO.H, GEO.W, device=DEV)
    fg[1] = 1                                   # all foreground
    fg[2, 200:210, 300:310] = 1                 # 100 foreground pixels (< 179)
    fg[3:, 100:380, 200:650] = 1                # frame 0: no foreground
    return m, fg


def _reference_coords(m, frames_set_t, fg_masks):
    """The per-pair algorithm (models/tracker.py:183-267) on public calls."""
    n_set = frames_set_t.shape[0]
    src_sel = torch.randint(n_set, (m.cyc_n_frames,), device=frames_set_t.device)
    tgt_sel = torch.randint(n_set, (m.cyc_n_frames,), device=frames_set_t.device)
    H, W = fg_masks.shape[-2:]
    yy, xx = torch.meshgrid(torch.arange(H, device=fg_masks.device).float(), torch.arange(W, device=fg_masks.device).float(),
                            indexing="ij")
    grid = torch.stack([xx.reshape(-1), yy.reshape(-1)], dim=-1)
    n_fg = int(m.cyc_batch_size_per_frame * m.cyc_fg_points_ratio)
    n_bg = m.cyc_batch_size_per_frame - n_fg
    emb = m.frame_embeddings
    fs = frames_set_t.to(DEV)
    keys = ("source_points", "target_points", "cycle_points", "source_frame_indices", "target_frame_indices")
    rows = {k: [] for k in keys}
    for s, t in zip(src_sel.to(DEV), tgt_sel.to(DEV)):
        t_src, t_tgt = fs[s], fs[t]
        is_fg = (fg_masks[int(t_src)] > 0).reshape(-1)
        fg_px, bg_px = grid[is_fg], grid[~is_fg]
        px = torch.cat([fg_px[torch.randperm(fg_px.shape[0])[:n_fg]], bg_px[torch.randperm(bg_px.shape[0])[:n_bg]]]).to(DEV)
        start = torch.cat([px, torch.ones(px.shape[0], 1, device=DEV) * t_src], dim=-1)
        n = start.shape[0]
        with torch.no_grad():
            there = m.range_normalizer.unnormalize(m.get_point_predictions((start, s.repeat(n), t.repeat(n), frames_set_t), emb),
                                                   src=(-1, 1), dims=[0, 1])
            there = torch.cat([there, torch.ones(n, 1, device=DEV) * t_tgt], dim=-1)
            back = m.range_normalizer.unnormalize(m.get_point_predictions((there, t.repeat(n), s.repeat(n), frames_set_t), emb),
                                                  src=(-1, 1), dims=[0, 1])
        ok = torch.norm(start[:, :2] - back[:, :2], dim=1) <= m.cyc_thresh
        k = int(ok.sum())
        for key, v in zip(keys, (start[ok], there[ok], back[ok], s.repeat(k), t.repeat(k))):
            rows[key].append(v)
    return {k: torch.cat(v) for k, v in rows.items()}, (src_sel.tolist(), tgt_sel.tolist())


def _reference_preds(m, frames_set_t, fg_masks):
    while True:
        cyc, sel = _reference_coords(m, frames_set_t, fg_masks)
        if cyc["source_points"].shape[0] > 0:
            break
    emb = m.frame_embeddings
    fwd = m.get_point_predictions((cyc["source_points"], cyc["source_frame_indices"], cyc["target_frame_indices"], frames_set_t), emb)
    bwd = m.get_point_predictions((cyc["target_points"], cyc["target_frame_indices"], cyc["source_frame_indices"], frames_set_t), emb)
    return cyc, {"source_coords": m.range_normalizer(cyc["source_points"], dst=[-1, 1]),
                 "target_coords": m.range_normalizer(cyc["target_points"], dst=[-1, 1]),
                 "source_target_coords": fwd[:, :2], "target_source_coords": bwd[:, :2],
                 "cycle_consistency_dists": torch.norm(cyc["cycle_points"][:, :2] - cyc["source_points"][:, :2], dim=1),
                 "cycle_points": cyc["cycle_points"]}, sel


def _cycle_loss(p):
    w = 0.8 ** p["cycle_consistency_dists"]            # dino_tracker.py:346-353
    st = w[:, None] * F.huber_loss(p["source_target_coords"], p["target_coords"][:, :2], reduction="none", delta=1 / 32)
    ts = w[:, None] * F.huber_loss(p["target_source_coords"], p["source_coords"][:, :2], reduction="none", delta=1 / 32)
    return (st.mean() + ts.mean()) / 2


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("host_set", [True, False])
def test_cycle_term_matches_per_pair_reference(host_set):
    m, fg = _model()
    fs = torch.tensor([0, 1, 2, 3], dtype=torch.int64, device="cpu" if host_set else DEV)
    g = torch.Generator().manual_seed(95)
    B = 64
    pts = torch.rand(B, 3, generator=g) * torch.tensor([GEO.W - 1.0, GEO.H - 1.0, 0.0])
    inp = (pts.to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), torch.randint(0, 4, (B,), generator=g).to(DEV), fs)
    m(inp)                                             # the step's forward: its embeddings feed the cycle term
    emb = m.frame_embeddings
    params = list(m.tracker_head.parameters())
    # seed 6 draws source slots [2, 1, 3, 0] and target slots [2, 1, 3, 2] from the host generator
    torch.manual_seed(6)
    got = m.get_cycle_consistent_preds(fs, fg)
    states = torch.get_rng_state(), torch.cuda.get_rng_state()
    torch.manual_seed(6)
    cyc, want, sel = _reference_preds(m, fs, fg)
    assert torch.equal(torch.get_rng_state(), states[0]) and torch.equal(torch.cuda.get_rng_state(), states[1])
    if host_set:
        assert sel == ([2, 1, 3, 0], [2, 1, 3, 2])
    n = want["source_coords"].shape[0]
    assert n > 0 and got["source_coords"].shape[0] == n                          # same survivors
    assert torch.equal(got["source_coords"], want["source_coords"])               # same pixels
    coords = m.get_cycle_consistent_coords                                         # (the no-grad dict: same draw again)
    torch.manual_seed(6)
    lib_cyc = coords(fs, fg)
    for k in ("source_frame_indices", "target_frame_indices"):
        assert torch.equal(lib_cyc[k], cyc[k].to(lib_cyc[k].device)), k
    assert torch.equal(lib_cyc["source_points"], cyc["source_points"])
    to_px = torch.tensor([GEO.W - 1, GEO.H - 1], device=DEV) / 2
    assert ((lib_cyc["target_points"] - cyc["target_points"]).abs().max()).item() <= XY_TOL
    assert torch.equal(lib_cyc["target_points"][:, 2], cyc["target_points"][:, 2])
    assert ((lib_cyc["cycle_points"] - cyc["cycle_points"]).abs().max()).item() <= 2 * XY_TOL
    for k in ("source_target_coords", "target_source_coords"):
        assert ((got[k] - want[k]).abs() * to_px).max().item() <= XY_TOL, k
    assert (got["cycle_consistency_dists"] <= m.cyc_thresh).all()
    g_got = torch.autograd.grad(_cycle_loss(got), [emb] + params, retain_graph=True)
    g_want = torch.autograd.grad(_cycle_loss(want), [emb] + params, retain_graph=True)
    for a, b in zip(g_got, g_want):
        assert b.abs().max().item() > 0 and _rel(a, b) <= GRAD_TOL


def test_mask_scan_batches_frames():
    """dinotrk_cycle_mask_scan on 5 frames of 476 x 854 (1588 blocks of 256 pixels: each scan thread sums more than one
    count): every frame's block offsets and foreground count equal numpy's, from one count and one scan launch."""
    import numpy as np
    from dino_tracker_b200 import _lib
    T, P = 5, GEO.H * GEO.W
    nb = -(-P // 256)
    assert nb == 1588
    fg = np.zeros((T, P), np.uint8)                 # frame 0: all background
    fg[1] = 1                                       # all foreground
    fg[2] = np.random.default_rng(97).integers(0, 3, P)
    fg[3, -1] = 1                                   # only the last pixel
    fg[4, 0] = 2                                    # only pixel 0
    cnt = np.pad(fg != 0, ((0, 0), (0, nb * 256 - P))).reshape(T, nb, 256).sum(-1)
    lib = _lib.load()
    d_fg = torch.from_numpy(fg).to(DEV)
    off = torch.full((T, nb), -1, device=DEV, dtype=torch.int32)
    n_fg = torch.full((T,), -1, device=DEV, dtype=torch.int32)
    ws_bytes = lib.dinotrk_cycle_mask_workspace_bytes(T, P)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    before = _lib.launch_count()
    _lib.check(lib.dinotrk_cycle_mask_scan(_lib.ptr(d_fg), T, P, _lib.ptr(off), _lib.ptr(n_fg), _lib.ptr(ws), ws_bytes,
                                           _lib.stream_ptr()), "cycle_mask_scan")
    assert _lib.launch_count() - before == 2        # the count and one scan over all frames
    np.testing.assert_array_equal(off.cpu().numpy(), np.cumsum(cnt, 1) - cnt)
    np.testing.assert_array_equal(n_fg.cpu().numpy(), cnt.sum(1))


def test_keep_decides_as_torch_norm_at_the_threshold():
    """Points whose way back ends within a few ulps of the 4 px circle: the kernel's keep flags equal
    torch.norm(start - unnormalize(back), dim=1) <= 4 evaluated on the device."""
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.range_normalizer import RangeNormalizer
    H, W, R, thresh = GEO.H, GEO.W, 1000, 4.0
    rn = RangeNormalizer(shapes=(W, H, 4), device=DEV)
    g = torch.Generator().manual_seed(96)
    start = torch.cat([(torch.rand(R, 2, generator=g) * torch.tensor([W - 9.0, H - 9.0]) + 4).floor(),
                       torch.zeros(R, 1)], dim=1).to(DEV)
    ang = torch.rand(R, generator=g, dtype=torch.float64) * 6.283185307179586
    px = start[:, :2].double() + thresh * torch.stack([ang.cos(), ang.sin()], dim=1).to(DEV)
    back = (px / torch.tensor([W - 1.0, H - 1.0], device=DEV, dtype=torch.float64) * 2 - 1).float()
    back = back + (torch.randint(-3, 4, (R, 2), generator=g).float() * 1.2e-7).to(DEV) * back.abs()
    back = back.contiguous()
    want = torch.norm(start[:, :2] - rn.unnormalize(back, src=(-1, 1), dims=[0, 1]), dim=1) <= thresh
    assert 0 < int(want.sum()) < R
    keep_rows = torch.empty(R, device=DEV, dtype=torch.int32)
    cycle_px = torch.empty(R, 2, device=DEV)
    n = torch.empty(1, device=DEV, dtype=torch.int32)
    _lib.check(_lib.load().dinotrk_cycle_keep(_lib.ptr(start), _lib.ptr(back), R, H, W, thresh, _lib.ptr(keep_rows),
                                              _lib.ptr(cycle_px), _lib.ptr(n), _lib.stream_ptr()), "cycle_keep")
    k = int(n.item())
    assert torch.equal(keep_rows[:k].long(), want.nonzero()[:, 0])
    assert torch.equal(cycle_px[:k], rn.unnormalize(back, src=(-1, 1), dims=[0, 1])[want])

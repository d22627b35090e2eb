"""GPU: the fp16 tensor-core contractions across feature scale and at arg-max near-ties, against float64.

Cosine is scale-invariant, the kernels' fp16 operands are not: a video outside the split's faithful range (max |x| above
65504, a non-zero token norm below 2^-3 sqrt(C); csrc/corr.cuh) must be routed to the exact-fp32 path, visibly, and give
the same answers as at scale 1.  Near-ties: an arg-max that differs from the float64 one is accepted only when the float64
gap between the two is below DELTA (DESIGN.md 3.1); best buddies likewise below DELTA_BB (DESIGN.md 5)."""
import warnings

import numpy as np
import pytest
import torch

from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle.tracker import Geometry

from test_fp16_range_cpu import TWIN_DST, TWIN_GAPS, TWIN_SRC, ra_video, twin_video
from test_tracker_gpu import make_model, run_corr_maps

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XY_TOL = 1e-3
DELTA = 5e-6      # float64 gap below which the tracker's arg-max may differ from float64's
DELTA_BB = 4e-6   # best buddies: twice the 2e-6 bar on the exact-fp32 cosines
SCALES = (-14, -12, -8, 0, 8, 14, 16)


def _faithful(tpc, norms):
    from dino_tracker_b200 import _lib
    return _lib.split_range(tpc, norms, _lib.stream_ptr())


def _model(geo, feats, head, precision="fp16x3"):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        m = make_model(geo, feats, head, precision)
        m.features_struct(m._dino_tpc, m._dino_norms)
    routed = any("faithful range" in str(x.message) for x in w)
    return m, routed


@pytest.mark.parametrize("k", SCALES)
@pytest.mark.parametrize("C", [48, 1024])
def test_corr_maps_across_scales(k, C):
    """The bars of test_corr_maps_match_oracle (C = 48, vs the fp32 oracle) and test_corr_gemm_error_vs_float64 (C = 1024)
    at every scale; out-of-range videos must announce the exact-fp32 route."""
    if C == 48:
        geo = Geometry(H=98, W=126)
        torch.manual_seed(2)
        T, ms = 3, [150, 148, 151]
        feats = torch.randn(T, C, geo.h, geo.w)
        desc = torch.randn(sum(ms), C)
        frames = [2, 0, 1]
    else:
        geo = Geometry()
        torch.manual_seed(5)
        T, ms = 2, [200]
        feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=9, noise=0.2)
        desc = feats[0].reshape(C, -1).t()[torch.randint(0, geo.P, (200,))].contiguous() + 0.05 * torch.randn(200, C)
        frames = [1]
    fs, ds = synth.scaled(feats, k), synth.scaled(desc, k)
    m, routed = _model(geo, fs, synth.head_weights("well"))
    max_abs, min_norm, ok = _faithful(m._dino_tpc, m._dino_norms)
    assert routed == (not ok)
    maps = run_corr_maps(m, ds, frames, ms)[:, : geo.P].cpu()
    tgt = torch.tensor(sum([[f] * n for f, n in zip(frames, ms)], []))
    if C == 48:
        ref = torch.relu(ot.corr_maps(desc, feats, tgt))[:, 0].reshape(sum(ms), -1)
        err, bar = (maps - ref).abs().max().item(), 2e-6
    else:
        f = feats[1].reshape(C, -1).double()
        d = desc.double()
        ref = torch.relu((d @ f) / (d.norm(dim=1)[:, None] * f.norm(dim=0)[None]).clamp_min(1e-8))
        err, bar = (maps.double() - ref).abs().max().item(), 4e-5
    print(f"[corr_maps C={C} scale 2^{k}] max|x| {max_abs:.3g} min norm {min_norm:.3g} -> "
          f"{'fp16x3' if ok else 'fp32'}; max error {err:.3e}")
    assert err <= bar


def _infer(feats, head, q, geo, path, precision="fp16x3"):
    from dino_tracker_b200 import ModelInference, _lib
    lib = _lib.load()
    m, routed = _model(geo, feats, head, precision)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    try:
        assert lib.dinotrk_infer_set_path(path) == 0
        r = mi.infer_all(q.to(DEV))
        torch.cuda.synchronize()
        stats = _lib.infer_stats()
    finally:
        lib.dinotrk_infer_set_path(-1)
    return {k: v.cpu() for k, v in r.items()}, stats, routed


def _check_infer(r, ref):
    t_ref, o_ref, aux = ref
    assert (r["traj"][..., :2] - aux["trajs"][..., :2]).abs().max().item() <= XY_TOL
    assert torch.equal(r["occ"].bool(), o_ref)
    vis = aux["cos_sims"] >= 0.7
    assert torch.equal(r["cos_sims"] >= 0.7, vis)
    d = 0.0
    for n in range(vis.shape[0]):
        if vis[n].any():
            d = max(d, (r["anchors"][n][vis[n]] - aux["anchors"][n]).abs().max().item())
    assert d <= XY_TOL
    return d


@pytest.mark.parametrize("kind", ["scaled", "massive"])
def test_infer_across_scales(kind):
    geo = Geometry(H=98, W=126)
    T, C = 5, 64
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=31, noise=0.2, max_shift=2)
    if kind == "massive":
        feats = synth.massive_channels(feats, seed=31)
    head = synth.head_weights("sharp", seed=31)
    q = synth.lattice_query_points(3, 2, geo.H, geo.W, t_q=[0, 1, 2, 3, 4, 0], margin=14.0, jitter_seed=31)
    ref = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    scales = SCALES if kind == "scaled" else (-4, 0, 2)
    for k in scales:
        fs = synth.scaled(feats, k)
        for path, precision in ((0, "fp16x3"), (1, "fp16x3"), (-1, "fp16x3"), (-1, "fp32")):
            r, st, routed = _infer(fs, head, q, geo, path, precision)
            d = _check_infer(r, ref)
            print(f"[infer {kind} 2^{k} path {path} {precision}] anchors max |dxy| {d:.2e} px; {st}")
            tensor = precision == "fp16x3" and not routed
            assert st["contraction"] == ("fp16x3" if tensor else "fp32")
            if tensor and path == 1:
                assert st["pipeline"] == "exact-window" and st["exact_window"] > 0
    if kind == "massive":   # the massive-activation layout is inside the faithful range: no silent pass by falling back
        _, st, routed = _infer(feats, head, q, geo, 1)
        assert not routed and st["contraction"] == "fp16x3" and st["exact_window"] > 0


def _peak_gap64(feats, src_pt, frame, tok_a, tok_b):
    """float64 cosine gap between tokens tok_a and tok_b of `frame` for the descriptor at src_pt (x, y, t) px."""
    geo = Geometry(H=(feats.shape[2] - 1) * 7 + 14, W=(feats.shape[3] - 1) * 7 + 14)
    d = ot.sample_descriptors(feats.double(), ot.normalize_points_for_sampling(src_pt[None].float(), geo)).double()[0]
    f = feats[frame].double().reshape(feats.shape[1], -1)
    c = (d @ f) / (d.norm() * f.norm(dim=0)).clamp_min(1e-8)
    return abs(c[tok_a].item() - c[tok_b].item())


def _tok(geo, xy):
    c = int(round((float(xy[0]) - geo.patch // 2) / geo.stride)); r = int(round((float(xy[1]) - geo.patch // 2) / geo.stride))
    return min(max(r, 0), geo.h - 1) * geo.w + min(max(c, 0), geo.w - 1)


def _check_ties(got, want, src_pts, frames, feats, geo, what):
    """Every point within XY_TOL of the oracle, or a float64 near-tie (< DELTA) between the tokens under the two answers."""
    n_tie, worst = 0, 0.0
    for i in range(got.shape[0]):
        if (got[i] - want[i]).abs().max().item() <= XY_TOL:
            continue
        g = _peak_gap64(feats, src_pts[i], int(frames[i]), _tok(geo, got[i]), _tok(geo, want[i]))
        assert g < DELTA, (what, i, g)
        n_tie, worst = n_tie + 1, max(worst, g)
    return n_tie, worst


@pytest.mark.parametrize("k", [0, -14, 8])
def test_twin_peaks_through_both_pipelines(k):
    """Far-apart twins with float64 gaps from 1e-7 to 3e-3: the trajectory phase, and the anchor phase through the full-map
    (0) and exact-window (1) pipelines, on the oracle's own trajectories."""
    from dino_tracker_b200 import ModelInference, _lib
    lib = _lib.load()
    geo, feats = twin_video()
    T = feats.shape[0]
    head = synth.head_weights("sharp", seed=21)
    px = lambda rc, dx=0.0, dy=0.0: [geo.patch // 2 + geo.stride * rc[1] + dx, geo.patch // 2 + geo.stride * rc[0] + dy]
    q = torch.tensor([px(TWIN_SRC) + [float(T - 1)], px(TWIN_SRC, 2.0, -1.5) + [float(T - 1)],
                      px(TWIN_SRC, -3.0, 2.5) + [0.0], px((8, 3)) + [1.0]])
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    fs = synth.scaled(feats, k)
    m, routed = _model(geo, fs, head)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    traj = mi.compute_trajectories(q.to(DEV)).cpu()
    N = q.shape[0]
    src = q[:, None].expand(N, T, 3).reshape(-1, 3)
    frames = torch.arange(T).repeat(N)
    n_tie, worst = _check_ties(traj[..., :2].reshape(-1, 2), aux["trajs"][..., :2].reshape(-1, 2), src, frames, feats, geo,
                               "trajectory")
    print(f"[twins 2^{k}] trajectory phase: {n_tie} near-tie deviations (largest float64 gap {worst:.1e})")
    cos = aux["cos_sims"]
    for path in (0, 1):
        try:
            assert lib.dinotrk_infer_set_path(path) == 0
            anchors = mi.compute_anchor_trajectories(aux["trajs"].to(DEV), cos.to(DEV))
            torch.cuda.synchronize()
            st = _lib.infer_stats()
        finally:
            lib.dinotrk_infer_set_path(-1)
        n_tie, worst = 0, 0.0
        for n in range(N):
            a_frames = torch.nonzero(cos[n] >= 0.7).flatten()
            got = anchors[n].cpu()
            assert got.shape == aux["anchors"][n].shape
            for j, a in enumerate(a_frames.tolist()):
                c, g = _check_ties(got[j], aux["anchors"][n][j], aux["trajs"][n], torch.full((T,), a), feats, geo,
                                   f"anchor n={n} a={a} path={path}")
                n_tie, worst = n_tie + c, max(worst, g)
        print(f"[twins 2^{k}] anchor phase, path {path}: {n_tie} near-tie deviations (largest float64 gap {worst:.1e}); {st}")
        if path == 1 and not routed:
            assert st["pipeline"] == "exact-window" and st["exact_window"] > 0


@pytest.mark.parametrize("k", [0, 8])
@pytest.mark.parametrize("which", ["near", "far"])
def test_rounding_aligned_twins(which, k):
    """Twins whose single-pass fp16 cosines are ordered against the exact ones (test_fp16_range_cpu checks the reversal for
    every map below).  Every anchor map of the source token must still give the float64 arg-max's point, through both
    pipelines.  Near twins (one exact-window box) must be decided by the exact-window pipeline itself -- every map of the
    call finishes there -- far twins by the full-map queue."""
    from dino_tracker_b200 import ModelInference, _lib
    lib = _lib.load()
    geo, feats, src, dst, gap = ra_video(which)
    T = feats.shape[0]
    head = synth.head_weights("sharp", seed=23)
    px = [geo.patch // 2 + geo.stride * src[1], geo.patch // 2 + geo.stride * src[0]]
    traj = torch.tensor([[px + [float(i)] for i in range(T)]])     # the source token's centre in every frame
    cos = torch.ones(1, T)
    ref = oi.anchor_predictions(feats, traj[0], torch.arange(T), head, geo)
    m, routed = _model(geo, synth.scaled(feats, k), head)
    assert not routed
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    for path in (0, 1):
        try:
            assert lib.dinotrk_infer_set_path(path) == 0
            got = mi.compute_anchor_trajectories(traj.to(DEV), cos.to(DEV))[0].cpu()
            torch.cuda.synchronize()
            st = _lib.infer_stats()
        finally:
            lib.dinotrk_infer_set_path(-1)
        d = (got - ref).abs().max().item()
        print(f"[rounding-aligned {which} twins 2^{k}, float64 gap {gap:.1e}] path {path}: max |dxy| {d:.2e} px; {st}")
        assert d <= XY_TOL
        assert st["anchor_maps"] == T * T and st["contraction"] == "fp16x3"
        if path == 1:
            assert st["pipeline"] == "exact-window"
            assert (st["exact_window"], st["full_map"]) == ((T * T, 0) if which == "near" else (0, T * T))


def _bb_ladder_video(T=2, C=256, seed=41):
    """Frame 1 holds, for some source tokens n of frame 0, three far-apart near-copies of F0[n] at float64 cosines
    1 - g, 1 - g - s, 1 - g - 2 s (order shuffled; rungs s from 1e-7 to 1e-4): three-way near-ties of the row arg-max."""
    geo = Geometry()
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.6, max_shift=2)
    f = feats.double().reshape(T, C, -1)
    rs = np.random.RandomState(seed)
    P = geo.P
    used = set()
    for n, s in zip(rs.choice(P, 40, replace=False), [1e-7, 1e-6, 1e-5, 1e-4] * 10):
        o = f[0, :, n]
        gaps = [1e-4, 1e-4 + s, 1e-4 + 2 * s]
        rs.shuffle(gaps)
        for g in gaps:
            m = int(rs.randint(P))
            while m in used:
                m = int(rs.randint(P))
            used.add(m)
            v = torch.from_numpy(rs.standard_normal(C))
            v = v - o * (o @ v) / (o @ o)
            eta = 1.0 / (1.0 - g) ** 2 - 1.0
            f[1, :, m] = o + v * (o.norm() * np.sqrt(eta) / v.norm())
    return geo, f.reshape(T, C, geo.h, geo.w).float()


@pytest.mark.parametrize("k", [0, -14, -8, 8, 16])
def test_best_buddies_three_way_near_ties(k):
    from dino_tracker_b200.best_buddies import nearest_neighbours
    from dino_tracker_b200 import _lib
    geo, feats = _bb_ladder_video()
    T, C = feats.shape[:2]
    fs = synth.scaled(feats, k)
    chw = fs.to(DEV)
    tpc = chw.permute(0, 2, 3, 1).reshape(T, -1, C).contiguous()
    norms = tpc.norm(dim=2).contiguous()
    g = _lib.make_geom(geo.H, geo.W)
    nn_idx, nn_cos = nearest_neighbours(tpc, norms, g, [(0, 1), (1, 0)])
    f = feats.double().reshape(T, C, -1)
    worst_cos, n_tie = 0.0, 0
    for p, (s, t) in enumerate([(0, 1), (1, 0)]):
        a, b = f[s].t(), f[t].t()
        aff = (a @ b.t()) / (a.norm(dim=1)[:, None] * b.norm(dim=1)[None]).clamp_min(1e-8)
        top2 = aff.topk(2, dim=1)
        best, gap = top2.indices[:, 0], top2.values[:, 0] - top2.values[:, 1]
        got = nn_idx[p].long().cpu()
        wrong = (got != best) & (gap >= DELTA_BB)
        assert not wrong.any(), (k, p, wrong.nonzero()[:5].flatten().tolist(), gap[wrong][:5].tolist())
        n_tie += int((got != best).sum())
        worst_cos = max(worst_cos, (nn_cos[p].cpu().double() - top2.values[:, 0]).abs().max().item())
    print(f"[best buddies 2^{k}] max |nn_cos - float64| {worst_cos:.2e}; {n_tie} rows resolved to another near-tied token")
    assert worst_cos <= 2e-6


def test_best_buddies_warn_when_no_scale_fits():
    """A spread of token norms wider than the faithful range: no power-of-two rescaling brings the video inside, and the
    best-buddy search must say so instead of running the affinity GEMM outside its bound silently."""
    from dino_tracker_b200.best_buddies import nearest_neighbours
    from dino_tracker_b200 import _lib
    geo = Geometry(H=98, W=126)
    T, C = 2, 64
    feats = synth.random_features(T, C, geo.h, geo.w, seed=43)
    feats[1, :, 4, 5] *= 2.0 ** -24                      # one token of norm ~5e-7 next to components of ~4
    tpc = feats.to(DEV).permute(0, 2, 3, 1).reshape(T, -1, C).contiguous()
    norms = tpc.norm(dim=2).contiguous()
    with pytest.warns(RuntimeWarning, match="even after rescaling"):
        nearest_neighbours(tpc, norms, _lib.make_geom(geo.H, geo.W), [(0, 1)])

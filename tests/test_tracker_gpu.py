"""GPU parity suite: CUDA kernels (through the C ABI / the reference-facing classes) against the oracle
and the committed reference vectors.  Tolerances: |dxy| <= 1e-3 px (BASELINE.json north_star),
occlusion masks bit-exact."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle.tracker import Geometry

from golden_util import TRACK_CASES, load_track_case

pytestmark = pytest.mark.gpu
XY_TOL = 1e-3
DEV = "cuda:0"


PRECISIONS = ["fp16x3", "fp32"]  # split-fp16 wgmma tensor-core GEMM / exact-fp32 FFMA GEMM


def make_model(geo, feats, head, precision="fp16x3"):
    from dino_tracker_b200 import Tracker
    T = feats.shape[0]
    video = torch.zeros(T, 3, geo.H, geo.W, device=DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=[3, 4, 4, 4, feats.shape[1]],
                corr_precision=precision)
    m.tracker_head.load_state_dict(head)
    return m


def test_pack_unpack_and_norms():
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(0)
    chw = torch.randn(3, 40, 13 * 17, device=DEV)
    tpc = torch.empty(3, 13 * 17, 40, device=DEV)
    norms = torch.empty(3, 13 * 17, device=DEV)
    _lib.check(lib.dinotrk_pack_features(_lib.ptr(chw), _lib.ptr(tpc), _lib.ptr(norms), 3, 40, 221, _lib.stream_ptr()))
    assert torch.equal(tpc, chw.permute(0, 2, 1).contiguous())
    assert torch.allclose(norms, chw.norm(dim=1), rtol=2e-7, atol=0)
    back = torch.empty_like(chw)
    _lib.check(lib.dinotrk_unpack_features(_lib.ptr(tpc), _lib.ptr(back), 3, 40, 221, _lib.stream_ptr()))
    assert torch.equal(back, chw)


@pytest.mark.parametrize("geo", [Geometry(H=98, W=126), Geometry(H=476, W=854)])
def test_sample_descriptors_matches_oracle(geo):
    torch.manual_seed(1)
    T, C = 5, 64
    feats = torch.randn(T, C, geo.h, geo.w)
    m = make_model(geo, feats, synth.head_weights("well"))
    B = 300
    pts = torch.rand(B, 3) * torch.tensor([geo.W + 40.0, geo.H + 40.0, 1.0]) - torch.tensor([20.0, 20.0, 0.0])
    frames_set = torch.tensor([3, 0, 1, 2, 4, 2], dtype=torch.int32)
    pts[:, 2] = torch.randint(0, frames_set.shape[0], (B,)).float()
    desc, dn = m._sample(m._dino_tpc, pts, frames_set, normalized=False)
    pn = ot.normalize_points_for_sampling(pts, geo)
    ref = ot.sample_descriptors(feats[frames_set.long()], pn)
    assert (desc.cpu() - ref).abs().max().item() <= 2e-6
    assert torch.allclose(dn.cpu(), ref.norm(dim=1), rtol=1e-6)
    # Tracker.sample_embeddings semantics (already-normalised x, y; full frame set)
    pn2 = pn.clone(); pn2[:, 2] = torch.randint(0, T, (B,)).float()
    out = m.sample_embeddings(feats.to(DEV), pn2.to(DEV))
    assert (out.cpu() - ot.sample_descriptors(feats, pn2)).abs().max().item() <= 2e-6


def run_corr_maps(model, desc, frames, ms):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    total = sum(ms)
    C = desc.shape[1]
    row0 = np.cumsum([0] + list(ms[:-1])).astype(np.int32)
    grp = torch.tensor(np.stack([frames, row0, ms, row0]).astype(np.int32), device=DEV)
    d_dev = desc.to(DEV).contiguous()
    dn = d_dev.norm(dim=1).contiguous()
    stride = lib.dinotrk_map_stride(ctypes.byref(model._geom))
    maps = torch.zeros(total, stride, device=DEV)
    nb = lib.dinotrk_corr_maps_workspace_bytes(total, len(ms), C)
    ws = torch.empty(nb, device=DEV, dtype=torch.uint8)
    feat = model.features_struct(model._dino_tpc, model._dino_norms)
    _lib.check(lib.dinotrk_corr_maps(ctypes.byref(feat), ctypes.byref(model._geom), _lib.ptr(d_dev), _lib.ptr(dn),
                                     _lib.ptr(grp[0]), _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), len(ms),
                                     total, max(ms), _lib.ptr(maps), _lib.ptr(ws), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return maps


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("m_per_frame", [3, 8, 9, 150, 300])
def test_corr_maps_match_oracle(m_per_frame, precision):
    """stream kernel (<= 8 descriptors per frame) and grouped GEMM (> 8), incl. ragged tiles."""
    geo = Geometry(H=98, W=126)
    torch.manual_seed(2)
    T, C = 3, 48
    feats = torch.randn(T, C, geo.h, geo.w)
    model = make_model(geo, feats, synth.head_weights("well"), precision)
    frames = [2, 0, 1]
    ms = [m_per_frame, max(1, m_per_frame - 2), m_per_frame + 1]
    total = sum(ms)
    desc = torch.randn(total, C)
    desc[0] = 0  # zero descriptor: clamp(min=1e-8) path
    maps = run_corr_maps(model, desc, frames, ms)
    tgt = torch.tensor(sum([[f] * m for f, m in zip(frames, ms)], []))
    ref = torch.relu(ot.corr_maps(desc, feats, tgt))[:, 0].reshape(total, -1)
    got = maps[:, : geo.P].cpu()
    assert (got - ref).abs().max().item() <= 2e-6


@pytest.mark.parametrize("precision", PRECISIONS)
def test_corr_gemm_error_vs_float64(precision):
    """Full geometry, C=1024: error of the wide-group contraction against a float64 evaluation
    (the fp32 reference itself sits ~1e-7 away from it)."""
    geo = Geometry()
    torch.manual_seed(5)
    T, C, M = 2, 1024, 200
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=9, noise=0.2)
    model = make_model(geo, feats, synth.head_weights("well"), precision)
    desc = feats[0].reshape(C, -1).t()[torch.randint(0, geo.P, (M,))].contiguous() + 0.05 * torch.randn(M, C)
    maps = run_corr_maps(model, desc, [1], [M])[:, : geo.P].cpu().double()
    f = feats[1].reshape(C, -1).double()
    ref = torch.relu((desc.double() @ f) / (desc.double().norm(dim=1)[:, None] * f.norm(dim=0)[None]).clamp_min(1e-8))
    err = (maps - ref).abs().max().item()
    print(f"[{precision}] max |corr - float64| = {err:.3e}")
    # fp32 FFMA: sequential fp32 accumulation over K=1024; split fp16: three tensor-core passes whose accumulation
    # truncates (the bias is coherent across tokens, see DESIGN.md "Precision")
    assert err <= (3e-6 if precision == "fp32" else 4e-5)


@pytest.mark.parametrize("fast", [True, False])
@pytest.mark.parametrize("kind", ["well", "sharp", "mixed", "default"])
@pytest.mark.parametrize("geo", [Geometry(H=98, W=126), Geometry(H=476, W=854)])
def test_head_matches_oracle(kind, geo, fast):
    """fast=True: windowed kernel + certified bound, uncertified maps re-done by the full-map kernel;
    fast=False: full-map kernel for every map."""
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(3)
    n = 24
    maps = np.maximum(rs.standard_normal((n, geo.h, geo.w)).astype(np.float32) * 0.2, 0)
    for k in range(n):  # plant peaks (some at the borders / corners)
        r, c = rs.randint(0, geo.h), rs.randint(0, geo.w)
        if k % 6 == 0:
            r, c = (0, 0) if k % 12 == 0 else (geo.h - 1, geo.w - 1)
        maps[k, r, c] = 0.9 + 0.01 * k
    maps[1] = 0.0  # all-zero map: arg-max index 0
    maps[2, 3, 4] = maps[2, 5, 6] = 0.95  # exact tie: first index wins
    head = synth.head_weights(kind, seed=7)
    model = make_model(geo, torch.zeros(2, 8, geo.h, geo.w), head)
    stride = lib.dinotrk_map_stride(ctypes.byref(model._geom))
    buf = torch.zeros(n, stride, device=DEV)
    buf[:, : geo.P] = torch.from_numpy(maps.reshape(n, -1)).to(DEV)
    out = torch.empty(n, 2, device=DEV)
    aux = torch.empty(n, 2, device=DEV, dtype=torch.int32)
    scratch = torch.zeros(n + 1, device=DEV, dtype=torch.int32) if fast else None
    _lib.check(lib.dinotrk_head(_lib.ptr(buf), n, ctypes.byref(model._geom), ctypes.byref(model.head_weights()), None,
                                _lib.ptr(out), 2, 1, _lib.ptr(aux), _lib.ptr(scratch), _lib.stream_ptr()))
    if fast:
        n_slow = int(scratch[0])
        print(f"[{kind} {geo.h}x{geo.w}] maps sent to the full-map kernel: {n_slow}/{n}")
        if kind in ("well", "sharp"):
            assert n_slow <= 2  # (the all-zero map may not certify)
    ref, raux = ot.head_forward(torch.from_numpy(maps)[:, None], head, geo, return_aux=True)
    assert torch.equal(aux[:, 0].cpu().long(), raux["argmax"])
    assert torch.equal(aux[:, 1].cpu().bool(), raux["fallback"])
    if kind == "default" and geo.H == 476:
        assert raux["fallback"].any()
    scale = torch.tensor([geo.W - 1, geo.H - 1]) / 2  # normalised units -> px
    assert ((out.cpu() - ref).abs() * scale).max().item() <= XY_TOL


@pytest.mark.parametrize("name", ["track_small_well", "track_small_fallback", "track_full_fallback"])
def test_forward_matches_reference_vectors(name):
    from dino_tracker_b200 import generate_trajectory_input
    cfg, geo, feats, head, g = load_track_case(name)
    model = make_model(geo, feats, head)
    model.cache_refined_embeddings()
    q = torch.from_numpy(g["query_points"]).to(DEV)
    inp = generate_trajectory_input(q[0], model.video)
    with torch.no_grad():            # inference kernels (tests/test_train_gpu.py covers the graph path)
        out = model(inp)
    scale = np.array([geo.W - 1, geo.H - 1]) / 2
    assert (np.abs(out.cpu().numpy() - g["forward0"]) * scale).max() <= XY_TOL
    # anchor-style input: sources in their own frames, one target
    T = cfg["T"]
    preds = torch.from_numpy(g["trajectories"][1]).to(DEV)
    fs = torch.cat([torch.tensor([2]), torch.arange(T)]).int().to(DEV)
    inp2 = (preds, torch.arange(1, T + 1, device=DEV), torch.zeros(T, dtype=torch.long, device=DEV), fs)
    with torch.no_grad():
        out2 = model(inp2).cpu()
    ref2 = ot.tracker_forward(feats, (preds.cpu(), torch.arange(1, T + 1), torch.zeros(T, dtype=torch.long), fs.cpu()),
                              head, geo)
    assert ((out2 - ref2).abs() * torch.from_numpy(scale).float()).max().item() <= XY_TOL


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", sorted(TRACK_CASES))
def test_infer_matches_reference_vectors(name, precision):
    from dino_tracker_b200 import ModelInference
    cfg, geo, feats, head, g = load_track_case(name)
    model = make_model(geo, feats, head, precision)
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)
    assert torch.equal(model.refined_features.cpu(), feats)  # default delta-DINO: exactly zero residual
    q = torch.from_numpy(g["query_points"]).to(DEV)
    r = mi.infer_all(q, cfg["batch"])
    traj, occ = mi.infer(q, cfg["batch"])
    assert np.abs(r["traj"].cpu().numpy() - g["trajectories"]).max() <= XY_TOL
    assert np.abs(r["cos_sims"].cpu().numpy() - g["cos_sims"]).max() <= 2e-5
    assert np.array_equal(occ.cpu().numpy(), g["occlusion"])
    assert np.array_equal(traj.cpu().numpy(), r["traj"][..., :2].cpu().numpy())
    vis = g["cos_sims"] >= 0.7
    for n in range(q.shape[0]):
        m = int(g["n_anchors"][n])
        got = r["anchors"][n].cpu().numpy()[vis[n]]
        assert got.shape[0] == m
        assert np.abs(got - g["anchors"][n, :m]).max() <= XY_TOL
    # piecewise API
    t2 = mi.compute_trajectories(q, cfg["batch"])
    c2 = mi.compute_trajectory_cos_sims(t2, q)
    a2 = mi.compute_anchor_trajectories(t2, c2, cfg["batch"])
    o2 = mi.compute_occlusion(t2, c2, a2)
    assert torch.equal(t2, r["traj"]) and torch.equal(c2, r["cos_sims"])
    assert np.array_equal(o2.cpu().numpy(), g["occlusion"])
    assert all(a2[n].shape == (int(g["n_anchors"][n]), cfg["T"], 2) for n in range(q.shape[0]))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_infer_medium_against_oracle(precision):
    """Full token geometry, wider batch (GEMM path, several chunks) against the oracle run here."""
    from dino_tracker_b200 import ModelInference
    geo = Geometry()
    T, C = 6, 128
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=40, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=40)
    q = synth.lattice_query_points(5, 4, geo.H, geo.W, t_q=[i % T for i in range(20)], margin=30.0, jitter_seed=40)
    model = make_model(geo, feats, head, precision)
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)
    r = mi.infer_all(q.to(DEV))
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (r["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(r["occ"].bool().cpu(), o_ref)
    assert (r["cos_sims"].cpu() - aux["cos_sims"]).abs().max().item() <= 2e-5


def test_infer_overlap_modes_agree():
    """Phase-C pipelining (sampling side stream, double-buffered chunks, deferred full-map head) must not change a bit:
    modes 0 / 1 and several chunk sizes against each other, and against the oracle."""
    from dino_tracker_b200 import ModelInference, _lib, model_inference as mim
    geo = Geometry()
    T, C = 6, 128
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=41, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=41)
    q = synth.lattice_query_points(5, 4, geo.H, geo.W, t_q=[i % T for i in range(20)], margin=30.0, jitter_seed=41)
    model = make_model(geo, feats, head, "fp16x3")
    mi = ModelInference(model, model.range_normalizer, 0.7, 0.6)
    lib = _lib.load()
    assert lib.dinotrk_infer_set_overlap(2) == -22   # DINOTRK_EINVAL: the modes are -1, 0 and 1
    old = mim.DEFAULT_CHUNK_MAPS
    results = {}
    try:
        for chunk in (256, 300, 16384):
            for mode in (0, 1):
                assert lib.dinotrk_infer_set_overlap(mode) == 0
                mim.DEFAULT_CHUNK_MAPS = chunk
                r = mi.infer_all(q.to(DEV))
                torch.cuda.synchronize()
                results[(chunk, mode)] = {k: r[k].clone() for k in ("traj", "cos_sims", "anchors", "occ")}
    finally:
        mim.DEFAULT_CHUNK_MAPS = old
        lib.dinotrk_infer_set_overlap(-1)
    ref = results[(16384, 0)]
    vis = ref["cos_sims"] >= 0.7
    for key, r in results.items():
        assert torch.equal(r["traj"], ref["traj"]) and torch.equal(r["cos_sims"], ref["cos_sims"]), key
        assert torch.equal(r["occ"], ref["occ"]), key
        assert torch.equal(r["anchors"][vis], ref["anchors"][vis]), key
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (ref["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(ref["occ"].bool().cpu(), o_ref)


def test_full_size_properties():
    """BASELINE.json config 2 at full size (854x476, T=50, C=1024, 256 query points, 652 800 correlation maps), where the
    oracle would need a day: size-independent properties instead.
      * query-order equivariance: permuting the query points permutes the outputs, bit for bit (every map's arithmetic is
        independent of its row in the GEMM group);
      * chunking invariance: 4 096-map chunks (160 chunks, pipelined) == 32 768-map chunks, bit for bit;
      * precision: the split-fp16 tensor path against the exact-fp32 FFMA path: |dxy| <= 1e-3 px, identical occlusion;
      * semantics: the synthetic video is a translating field; every track follows the known shift of its frame."""
    import bench
    from bench_inputs import sharp_head
    from dino_tracker_b200 import ModelInference, Tracker, model_inference as mim
    T, C, nq = 50, 1024, 256
    feats = bench.synth_video_features(T, C, DEV, 1234, 0.25)
    video = torch.zeros(T, 3, bench.H, bench.W, device=DEV)
    q = bench.query_lattice(nq, 0).to(DEV)
    old = mim.DEFAULT_CHUNK_MAPS
    try:
        res = {}
        for prec in ("fp16x3", "fp32"):
            m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=[3, 4, 4, 4, C], corr_precision=prec)
            m.tracker_head.load_state_dict(sharp_head(0))
            mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
            mim.DEFAULT_CHUNK_MAPS = 32768
            res[prec] = mi.infer_all(q)
            if prec == "fp16x3":
                perm = torch.randperm(nq, generator=torch.Generator().manual_seed(0)).to(DEV)
                rp = mi.infer_all(q[perm])
                mim.DEFAULT_CHUNK_MAPS = 4096
                rc = mi.infer_all(q)
            del m, mi
        a = res["fp16x3"]
        assert torch.equal(rp["traj"], a["traj"][perm]) and torch.equal(rp["occ"], a["occ"][perm])
        assert torch.equal(rp["cos_sims"], a["cos_sims"][perm])
        assert torch.equal(rc["traj"], a["traj"]) and torch.equal(rc["occ"], a["occ"]) and torch.equal(rc["anchors"], a["anchors"])
        b = res["fp32"]
        assert (a["traj"] - b["traj"]).abs().max().item() <= XY_TOL
        assert torch.equal(a["occ"], b["occ"])
        # every frame is an anchor frame on this workload: 256 * 50 * 51 maps
        assert int((a["cos_sims"] >= 0.7).sum().item()) == nq * T
        # the field translates by whole tokens: frame t shows frame 0 shifted by (dy_t, dx_t) tokens (same recurrence as
        # bench.synth_video_features), so every track must follow -7 px * shift_t to within half a token
        cg = torch.Generator().manual_seed(1234)
        shifts = torch.zeros(T, 2, dtype=torch.long)
        for t in range(1, T):
            shifts[t] = (shifts[t - 1] + torch.randint(-1, 2, (2,), generator=cg)).clamp(-3, 3)
        expect = a["traj"][:, :1, :2].cpu() - 7.0 * shifts[:, [1, 0]].float()[None]       # (x, y) <- (dx, dy)
        assert (a["traj"][:, :, :2].cpu() - expect).abs().max().item() < 3.5
    finally:
        mim.DEFAULT_CHUNK_MAPS = old

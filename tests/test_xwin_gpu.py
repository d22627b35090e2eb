"""GPU: the anchor phase's coarse-pass + exact-window pipeline (csrc/xwin.cu) against the full-map pipeline and the oracle.

The exact-window pipeline never writes a correlation map: one single-pass fp16 GEMM keeps tile maxima, the split-precision
contraction is evaluated on a 21 x 21 token box per (query, anchor frame) cell, a warp-per-map head finishes.  Whatever the
coarse pass cannot decide rigorously (near-tied arg-max candidates, maps that leave their cell's box, uncertified softmax)
is re-done by the full-map pipeline, so the two pipelines must agree to the parity bar on every input -- including inputs
built to defeat the fast path."""
import numpy as np
import pytest
import torch

from oracle import inference as oi
from oracle import synth
from oracle.tracker import Geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XY_TOL = 1e-3


def _run(feats, head, q, geo, path, chunk=None):
    from dino_tracker_b200 import ModelInference, Tracker, _lib, model_inference as mim
    lib = _lib.load()
    T = feats.shape[0]
    m = Tracker(video=torch.zeros(T, 3, geo.H, geo.W, device=DEV), dino_embed_video=feats, device=DEV,
                delta_channels=[3, 4, 4, 4, feats.shape[1]])
    m.tracker_head.load_state_dict(head)
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    old = mim.DEFAULT_CHUNK_MAPS
    try:
        if chunk:
            mim.DEFAULT_CHUNK_MAPS = chunk
        assert lib.dinotrk_infer_set_path(path) == 0
        r = mi.infer_all(q.to(DEV))
        torch.cuda.synchronize()
        stats = _lib.infer_stats()
    finally:
        lib.dinotrk_infer_set_path(-1)
        mim.DEFAULT_CHUNK_MAPS = old
    return {k: v.clone() for k, v in r.items()}, stats


def _agree(a, b, tol=XY_TOL):
    vis = a["cos_sims"] >= 0.7
    assert torch.equal(a["traj"], b["traj"]) and torch.equal(a["cos_sims"], b["cos_sims"])   # phases A / B are shared
    d = (a["anchors"][vis] - b["anchors"][vis]).abs().max().item() if vis.any() else 0.0
    assert d <= tol, d
    assert torch.equal(a["occ"], b["occ"])
    return d


@pytest.mark.parametrize("kind", ["sharp", "well"])
@pytest.mark.parametrize("geo,T,C", [(Geometry(H=98, W=126), 5, 32), (Geometry(), 6, 128), (Geometry(), 9, 256)])
def test_exact_window_matches_full_map_and_oracle(geo, T, C, kind):
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=7 + T, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=T)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=14.0, jitter_seed=T)
    full, s0 = _run(feats, head, q, geo, 0)
    xw, s1 = _run(feats, head, q, geo, 1)
    assert s0["pipeline"] == "full-map" and s1["pipeline"] == "exact-window"
    d = _agree(xw, full)
    print(f"[{geo.h}x{geo.w} T={T} C={C} {kind}] exact-window vs full-map: anchors max |dxy| = {d:.2e} px; {s1}")
    assert s1["exact_window"] + s1["full_map"] == s1["anchor_maps"] == int((xw["cos_sims"] >= 0.7).sum().item()) * T
    assert s1["exact_window"] >= 0.9 * s1["anchor_maps"]          # a translating field: cells cluster, windows fit
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (xw["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(xw["occ"].bool().cpu(), o_ref)
    vis = aux["cos_sims"] >= 0.7
    for n in range(q.shape[0]):
        assert (xw["anchors"][n].cpu()[vis[n]] - aux["anchors"][n]).abs().max().item() <= XY_TOL


def test_chunking_and_stream_modes_do_not_change_a_bit():
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    geo = Geometry()
    T, C = 6, 128
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=43, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=43)
    q = synth.lattice_query_points(5, 4, geo.H, geo.W, t_q=[i % T for i in range(20)], margin=30.0, jitter_seed=43)
    ref, _ = _run(feats, head, q, geo, 1, chunk=16384)
    vis = ref["cos_sims"] >= 0.7
    try:
        for mode in (0, 1):
            assert lib.dinotrk_infer_set_overlap(mode) == 0
            for chunk in (60, 120, 300):     # (multiples of the 20 queries per frame: the trajectory phase keeps whole groups)
                r, st = _run(feats, head, q, geo, 1, chunk=chunk)
                assert torch.equal(r["traj"], ref["traj"]) and torch.equal(r["occ"], ref["occ"]), (mode, chunk)
                assert torch.equal(r["anchors"][vis], ref["anchors"][vis]), (mode, chunk)
    finally:
        lib.dinotrk_infer_set_overlap(-1)


def test_adversarial_inputs_fall_back_correctly():
    """(a) duplicated frames content inside a frame: exact ties between two far-apart tokens -> ambiguous maps;
    (b) pure-noise features: the arg-maxes of a cell scatter over the whole frame -> windows leave the box;
    (c) zero descriptors (a query on a frame whose features vanish in one corner region is not possible without (d));
    (d) an all-zero frame (token norms below XW_MIN_NORM void the coarse bound): the whole call must take the full-map
    pipeline even when the exact-window one is requested.  All must come out as the full-map pipeline computes them."""
    geo = Geometry(H=140, W=182)            # 19 x 25 tokens: smaller than the 21-row box in one direction
    T, C = 6, 64
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=90, noise=0.1, max_shift=1)
    feats[2, :, 3, 4] = feats[2, :, 12, 20]                    # (a) an exact duplicate token in frame 2
    feats[3] = synth.random_features(1, C, geo.h, geo.w, seed=91)[0]   # (b) frame 3 is noise
    head = synth.head_weights("sharp", seed=9)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[0, 1, 2, 4] * 3, margin=14.0, jitter_seed=9)
    q[0, :2] = torch.tensor([7.0 + 7 * 20, 7.0 + 7 * 12])      # sits on the duplicated token of frame 2
    q[0, 2] = 2
    full, _ = _run(feats, head, q, geo, 0)
    for chunk in (None, 12):
        xw, st = _run(feats, head, q, geo, 1, chunk=chunk)
        d = _agree(xw, full)
        print(f"adversarial: exact-window vs full-map max |dxy| = {d:.2e} px; {st}")
        assert st["full_map"] > 0                                # the fallbacks were exercised
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (xw["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(xw["occ"].bool().cpu(), o_ref)
    # (d) a frame of zeros: no coarse pass at all
    feats[5] = 0.0
    full, _ = _run(feats, head, q, geo, 0)
    xw, st = _run(feats, head, q, geo, 1)
    assert st["pipeline"] == "full-map" and st["exact_window"] == 0
    _agree(xw, full)
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (xw["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(xw["occ"].bool().cpu(), o_ref)


def test_uncertifiable_head_switches_pipeline():
    """'default'-like refiner weights (kernel sums ~ 0): every map needs the full-map refiner; the automatic choice must
    notice it in the trajectory phase and not waste the exact-window attempt; forcing it must still be correct."""
    geo = Geometry(H=98, W=126)
    T, C = 5, 32
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=77, noise=0.2, max_shift=2)
    head = synth.head_weights("default", seed=7)
    q = synth.lattice_query_points(3, 2, geo.H, geo.W, t_q=[0, 1, 2, 3, 4, 0], margin=14.0, jitter_seed=7)
    auto, s_auto = _run(feats, head, q, geo, -1)
    forced, s_forced = _run(feats, head, q, geo, 1)
    full, _ = _run(feats, head, q, geo, 0)
    print(f"uncertifiable head: auto -> {s_auto}; forced -> {s_forced}")
    assert s_auto["pipeline"] == "full-map"
    assert s_forced["pipeline"] == "exact-window" and s_forced["full_map"] >= 0.9 * s_forced["anchor_maps"]
    _agree(forced, full)
    _agree(auto, full)


def test_long_video_cells_split_into_blocks():
    """T > 128: the source frames of a (query, anchor frame) pair are split into cells of <= 128 rows (wgmma N <= 128)."""
    geo = Geometry(H=98, W=126)
    T, C = 150, 32
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=5, noise=0.15, max_shift=2)
    head = synth.head_weights("sharp", seed=5)
    q = synth.lattice_query_points(2, 2, geo.H, geo.W, t_q=[0, 40, 80, 149], margin=20.0, jitter_seed=5)
    full, _ = _run(feats, head, q, geo, 0)
    xw, st = _run(feats, head, q, geo, 1, chunk=4096)
    d = _agree(xw, full)
    print(f"T=150: exact-window vs full-map max |dxy| = {d:.2e} px; {st}")
    assert st["exact_window"] > 0

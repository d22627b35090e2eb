"""GPU: the exact-window pipeline reads anchor descriptors in place from the unique (query, source frame) table where the
anchor lists allow it and gathers the rest into the chunk's own rows (csrc/inference.cu: plan_chunks, anchor_scalars_kernel,
gather_anchor_kernel).  Where a row comes from must not change a bit of the result.

Videos here have frames with regions of noise: queries whose track crosses such a region fall below the anchor threshold
on that frame, so the per-frame anchor lists have long runs (read in place), short runs and isolated queries (gathered).
With T = 17 the slot index of the first source frame leaks weight onto slot 0 for every query (fp32 round trip of
1 / 17 * 2 - 1): every descriptor depends on its anchor frame and none may be read in place."""
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


def _video(T, C, geo, seed):
    """A translating field; frames 5 and 11 are noise on the left half (every other run of 4 lattice queries drops out),
    frame 8 on one small patch (an isolated query or two drop out), the others keep (nearly) every query."""
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.1, max_shift=1)
    noise = synth.random_features(T, C, geo.h, geo.w, seed=seed + 1)
    for t in (5, 11):
        feats[t, :, :, : geo.w // 2] = noise[t, :, :, : geo.w // 2]
    feats[8, :, 4:8, 9:13] = noise[8, :, 4:8, 9:13]
    head = synth.head_weights("sharp", seed=seed)
    clean = [t for t in range(T) if t not in (5, 8, 11)]           # query frames: every query has a clean descriptor
    q = synth.lattice_query_points(8, 6, geo.H, geo.W, t_q=[clean[i % len(clean)] for i in range(48)], margin=20.0,
                                   jitter_seed=seed)
    return feats, head, q


def _check_against_full_map_and_oracle(xw, feats, head, q, geo):
    full, s0 = _run(feats, head, q, geo, 0)
    assert s0["pipeline"] == "full-map" and s0["desc_in_place"] == 0 and s0["desc_gathered"] == 0
    vis = xw["cos_sims"] >= 0.7
    assert torch.equal(xw["traj"], full["traj"]) and torch.equal(xw["cos_sims"], full["cos_sims"])
    assert (xw["anchors"][vis] - full["anchors"][vis]).abs().max().item() <= XY_TOL
    assert torch.equal(xw["occ"], full["occ"])
    t_ref, o_ref, aux = oi.infer(feats, q, head, geo, 0.7, 0.6, return_all=True)
    assert (xw["traj"].cpu() - aux["trajs"]).abs().max().item() <= XY_TOL
    assert torch.equal(xw["occ"].bool().cpu(), o_ref)
    ovis = aux["cos_sims"] >= 0.7
    for n in range(q.shape[0]):
        if ovis[n].any():
            assert (xw["anchors"][n].cpu()[ovis[n]] - aux["anchors"][n]).abs().max().item() <= XY_TOL


def test_rows_in_place_and_gathered_give_the_same_bits():
    geo = Geometry(H=98, W=126)
    T, C = 16, 64
    feats, head, q = _video(T, C, geo, seed=31)
    ref, st = _run(feats, head, q, geo, 1, chunk=16384)
    print(f"T=16, 48 queries, one chunk: {st}")
    assert st["pipeline"] == "exact-window"
    vis = ref["cos_sims"] >= 0.7
    print("queries anchored per frame:", vis.sum(0).cpu().numpy())
    assert st["desc_in_place"] > 0 and st["desc_gathered"] > 0    # full frames and ragged ones
    assert st["desc_in_place"] + st["desc_gathered"] == st["anchor_maps"] == int(vis.sum().item()) * T
    # smaller chunks move the run cuts: rows change sides, no bit of the result may
    seen = {(st["desc_in_place"], st["desc_gathered"])}
    for chunk in (768, 1536, 3840):     # (multiples of the 48 queries per frame: the trajectory phase keeps whole groups)
        r, s = _run(feats, head, q, geo, 1, chunk=chunk)
        seen.add((s["desc_in_place"], s["desc_gathered"]))
        assert s["desc_in_place"] + s["desc_gathered"] == s["anchor_maps"], chunk
        assert torch.equal(r["traj"], ref["traj"]) and torch.equal(r["occ"], ref["occ"]), chunk
        assert torch.equal(r["anchors"][vis], ref["anchors"][vis]), chunk
    assert len(seen) > 1
    # every row gathered (chunks of three cells, 48 rows): the pipeline as it was before rows were read in place
    r, s = _run(feats, head, q, geo, 1, chunk=48)
    assert s["desc_in_place"] == 0
    assert torch.equal(r["anchors"][vis], ref["anchors"][vis]) and torch.equal(r["occ"], ref["occ"])
    _check_against_full_map_and_oracle(ref, feats, head, q, geo)


def test_leaking_slot_index_is_never_read_in_place():
    geo = Geometry(H=98, W=126)
    T, C = 17, 64
    feats, head, q = _video(T, C, geo, seed=37)
    xw, st = _run(feats, head, q, geo, 1, chunk=16384)
    print(f"T=17 (slot 1 leaks onto slot 0): {st}")
    assert st["pipeline"] == "exact-window" and st["anchor_maps"] > 0
    assert st["desc_in_place"] == 0 and st["desc_gathered"] == st["anchor_maps"]
    _check_against_full_map_and_oracle(xw, feats, head, q, geo)

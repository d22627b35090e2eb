"""GPU: the best-buddy preprocessing above 476 x 854 -- best buddies, their peak filter, trajectory chaining, the nearest
trajectory, the flow filter, the fg / bg split and the whole best-buddy preprocessing -- on the large-grid envelope
(tests/test_large_grid_gpu.py) against float64 and the oracle on the same GPU.

Frames: 1274 x 714 and 714 x 1274 (18,281 tokens: 72 column tiles of 256, the last holding 105 tokens), 1274 x 1274
(32,761 tokens: 128 tiles, the last holding 249) and 98 x 1799 (13 x 256 tokens, the widest grid; 3,328 = 13 x 256
tokens fill every tile).  The best-buddy resolve merges one top-2 record per column tile, tile t on lane t mod 32, so
beyond 8,192 tokens a lane merges two to four records before the butterfly.  Planted three-way near-tie ladders put the
tied tokens where that merge decides: in tiles t, t + 32 and t + 64 of one lane, in the last partial tile, on
neighbouring lanes, for source rows beyond 8,192 and 16,384.

Bars are those of DESIGN.md 5: every arg-max equals float64's where the float64 gap to the runner-up is >= DELTA_BB,
every exact-fp32 cosine is within 2e-6 of float64, the mutual set equals float64's outside rows with a near-tie in
either direction; peaks within 2e-6 and r within 4e-6 of a float64 restatement of the peak filter outside rows whose
arg-max or rank decision is a float64 near-tie.  Each test prints its worst error and the rows it excluded."""
import functools
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bb_nms as onms
from oracle import best_buddies as obb
from oracle import fg_masks as ofg
from oracle import of_filter as oof
from oracle import synth
from oracle import trajectories as otr
from oracle.tracker import Geometry

from test_fp16_range_gpu import DELTA_BB
from test_preprocess_gpu import _bb_equal, _by_start, _close, _same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
COS_TOL = 2e-6         # exact-fp32 cosines and peak values against float64
R_TOL = 4e-6           # r = second / first peak
TILE = 256             # column tile of the best-buddy GEMM epilogue (TC_BN): one top-2 record per tile and source row
IOU = 0.2              # preprocessing.yaml dino_bb_iou_threshold
TOPK = 400             # compute_dino_bb_nms.py's top-k
LADDER_GAP = 1e-4      # float64 cosine 1 - gap of the best rung of a ladder
RUNGS = (0.0, 1e-7, 1e-6, 1e-5, 1e-4)

# (H, W, T, C): T = 8 on the 98 x 1799 frames gives 56 ordered pairs, two launches of pairs_per_launch = 48
BB_SHAPES = [(1274, 714, 4, 1024), (714, 1274, 4, 1024), (1274, 1274, 4, 1024), (98, 1799, 8, 768)]


def _ids(shapes):
    return [f"{H}x{W}-T{T}-C{C}" for H, W, T, C in shapes]


def _sync_time():
    torch.cuda.synchronize()
    return time.perf_counter()


# ---- planted near-ties ------------------------------------------------------------------------------------------------
def _ladder_tiles(kind, nt, rs):
    """Column tiles of the three copies of one ladder on a grid of nt tiles (tile t -> resolve lane t mod 32)."""
    last = nt - 1
    rnd = lambda: int(rs.randint(0, nt))
    if kind == 0:      # one lane merges three records: tiles t, t + 32, t + 64
        if nt > 64:
            t = int(rs.randint(0, nt - 64))
            return (t, t + 32, t + 64)
        kind = 1
    if kind == 1:      # two records on one lane, the third on the neighbouring lane (the butterfly's first partner)
        if nt > 32:
            t = int(rs.randint(0, nt - 32))
            return (t, t + 32, t + 1)
        kind = 4
    if kind == 2:      # the last, partial tile and the tiles of its lane
        return (last, last - 32 if nt > 32 else rnd(), last - 64 if nt > 64 else rnd())
    if kind == 3:      # two copies inside the last tile (its epilogue record keeps both), one elsewhere
        return (last, last, rnd())
    t = int(rs.randint(0, nt - 2))
    return (t, t + 1, t + 2)   # three neighbouring lanes


def _plant_ladders(f, src, dst, rs, used, n_ladders=50):
    """In frame ``dst`` of f [T][C][P] (float64, in place), three far-apart near-copies of token n of frame ``src`` at
    float64 cosines 1 - g, 1 - g - s, 1 - g - 2 s (order shuffled over the tiles; rung s from RUNGS, 0 = three different
    vectors at the same float64 cosine).  Every (tile pattern, rung) combination appears; the source rows cycle through
    [0, 8192), [8192, 16384) and [16384, P).  Returns [(n, [copy tokens])]."""
    P, C = f.shape[2], f.shape[1]
    nt = -(-P // TILE)
    bands = [(lo, min(hi, P)) for lo, hi in ((0, 8192), (8192, 16384), (16384, P)) if lo < P]
    out = []

    def fresh(lo, hi):
        while True:
            m = int(rs.randint(lo, hi))
            if m not in used:
                used.add(m)
                return m
    for k in range(n_ladders):
        kind, rung, band = k % 5, RUNGS[(k // 5) % 5], bands[k % len(bands)]
        n = fresh(*band)
        o = f[src, :, n].clone()
        gaps = [LADDER_GAP, LADDER_GAP + rung, LADDER_GAP + 2 * rung]
        rs.shuffle(gaps)
        copies = []
        for t, g in zip(_ladder_tiles(kind, nt, rs), gaps):
            m = fresh(t * TILE, min((t + 1) * TILE, P))
            v = torch.from_numpy(rs.standard_normal(C)).to(f)
            v = v - o * (o @ v) / (o @ o)
            eta = 1.0 / (1.0 - g) ** 2 - 1.0
            f[dst, :, m] = o + v * (o.norm() * np.sqrt(eta) / v.norm())
            copies.append(m)
        out.append((n, copies))
    return out


@functools.lru_cache(maxsize=4)
def _bb_video(H, W, T, C):
    """(geometry, features T x C x h x w fp32 on the host, {(src, dst): ladders}): shifted-field features (many mutual
    pairs) with ladders for the rows of ordered pair (0, 1) and for those of (3, 2) (the column side of (2, 3))."""
    geo = Geometry(H=H, W=W)
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=H + W + C + T, noise=0.3, max_shift=2)
    f = feats.double().reshape(T, C, -1)
    rs = np.random.RandomState(H * 7 + W * 3 + T)
    used = set()
    ladders = {(0, 1): _plant_ladders(f, 0, 1, rs, used), (3, 2): _plant_ladders(f, 3, 2, rs, used)}
    return geo, f.reshape(T, C, geo.h, geo.w).float(), ladders


# ---- float64 references -----------------------------------------------------------------------------------------------
def _unit64(feats):
    """T x C x h x w -> T x P x C float64 unit rows on the GPU (the reference clamps |a| |b| at 1e-8; these norms are ~10)."""
    T, C = feats.shape[:2]
    f = feats.to(DEV).double().reshape(T, C, -1).transpose(1, 2).contiguous()
    return f / f.norm(dim=2, keepdim=True)


def _top2_64(a, b, block=2048):
    """One float64 GEMM a b^T in row blocks, a running top-2 per row and per column: (row arg-max, row gap, column
    arg-max, column gap), the gap being best minus second best.  Rows of a are s's tokens, rows of b t's."""
    P, Q = a.shape[0], b.shape[0]
    ri = torch.empty(P, dtype=torch.long, device=DEV)
    rg = torch.empty(P, dtype=torch.float64, device=DEV)
    cv = torch.full((2, Q), -float("inf"), dtype=torch.float64, device=DEV)
    ci = torch.zeros(2, Q, dtype=torch.long, device=DEV)
    for r0 in range(0, P, block):
        S = a[r0:r0 + block] @ b.t()
        t = S.topk(2, dim=1)
        ri[r0:r0 + S.shape[0]] = t.indices[:, 0]
        rg[r0:r0 + S.shape[0]] = t.values[:, 0] - t.values[:, 1]
        c = S.topk(min(2, S.shape[0]), dim=0)
        vals, idx = torch.cat([cv, c.values]), torch.cat([ci, c.indices + r0])
        m = vals.topk(2, dim=0)
        cv, ci = m.values, idx.gather(0, m.indices)
        del S
    return ri, rg, ci[0], cv[0] - cv[1]


def _check_rows(nn, cos, mutual, best, gap, back_best, back_gap, a, b, what):
    """Kernel answers for the rows of a against b (nn_idx, nn_cos, mutual mask) against float64: arg-max where the gap is
    >= DELTA_BB, the cosine at the kernel's own partner, the mutual set outside rows with a near-tie in either direction.
    Returns (worst cosine error, rows excluded from the mutual check, rows resolved to another near-tied token)."""
    nn = nn.long()
    wrong = (nn != best) & (gap >= DELTA_BB)
    assert not wrong.any(), (what, wrong.nonzero()[:5].flatten().tolist(), gap[wrong][:5].tolist())
    err = (cos.double() - (a * b[nn]).sum(1)).abs().max().item()
    assert err <= COS_TOL, (what, err)
    ref_mutual = back_best[best] == torch.arange(a.shape[0], device=DEV)
    excl = (gap < DELTA_BB) | (back_gap[best] < DELTA_BB)
    bad = (mutual != ref_mutual) & ~excl
    assert not bad.any(), (what, bad.nonzero()[:5].flatten().tolist())
    return err, int(excl.sum()), int((nn != best).sum())


def _tokens(coords, geo):
    """Token index of pixel coordinates on the token grid (x = 7 + 7 c, y = 7 + 7 r)."""
    c = coords.to(DEV).double()
    return (((c[:, 1] - geo.patch // 2) / geo.stride).round().long() * geo.w
            + ((c[:, 0] - geo.patch // 2) / geo.stride).round().long())


def _peaks64(a, b, toks, geo, box, block=1024):
    """The rule bb_nms_kernel documents, in float64 on the similarity rows a[toks] b^T: the arg-max (first index), the best
    value whose box has IoU <= IOU with the arg-max's box (0 if none), kept when fewer than TOPK values exceed it.
    Boxes and IoU in fp32 as torchvision forms them.  Returns (first, second, r, near-tie rows): a row is a near-tie when
    its two largest values, or its second peak and its TOPK-th value, are closer than DELTA_BB."""
    P = b.shape[0]
    idx = torch.arange(P, device=DEV)
    xs = (geo.patch // 2 + (idx % geo.w) * geo.stride).float()
    ys = (geo.patch // 2 + (idx // geo.w) * geo.stride).float()
    bx = float(box)
    out = []
    for i0 in range(0, toks.shape[0], block):
        v = a[toks[i0:i0 + block]] @ b.t()
        R = v.shape[0]
        top = v.topk(TOPK, dim=1).values
        am = v.argmax(dim=1)
        ax, ay = xs[am][:, None], ys[am][:, None]
        iw = (torch.minimum(ax + bx, xs + bx) - torch.maximum(ax - bx, xs - bx)).clamp(min=0)
        ih = (torch.minimum(ay + bx, ys + bx) - torch.maximum(ay - bx, ys - bx)).clamp(min=0)
        inter = iw * ih
        area = ((ax + bx) - (ax - bx)) * ((ay + bx) - (ay - bx))
        ok = ~(inter / (area + area - inter) > IOU)
        ok[torch.arange(R, device=DEV), am] = False
        v2 = torch.where(ok, v, torch.zeros_like(v)).amax(dim=1).clamp_min(0)
        above = (v > v2[:, None]).sum(dim=1)
        second = torch.where(above < TOPK, v2, torch.zeros_like(v2))
        tie = (top[:, 0] - top[:, 1] < DELTA_BB) | ((v2 - top[:, TOPK - 1]).abs() < DELTA_BB)
        out.append((top[:, 0], second, second / top[:, 0], tie))
        del v, iw, ih, inter, ok
    return tuple(torch.cat(x) for x in zip(*out))


def _check_peaks(d, d_rev, s, t, f64, geo, box, what):
    """peak_affs of the s_t dict and r (the larger of both directions, compute_max_r) after the peak filter, against
    _peaks64.  Returns (worst peak error, worst r error, rows excluded)."""
    src, tgt = _tokens(d["source_coords"], geo), _tokens(d["target_coords"], geo)
    first, second, r, tie = _peaks64(f64[s], f64[t], src, geo, box)
    _, _, r_rev, tie_rev = _peaks64(f64[t], f64[s], _tokens(d_rev["source_coords"], geo), geo, box)
    pos = torch.full((geo.P,), -1, dtype=torch.long, device=DEV)
    pos[_tokens(d_rev["source_coords"], geo)] = torch.arange(d_rev["source_coords"].shape[0], device=DEV)
    j = pos[tgt]                     # the reverse row of every pair: its source is this pair's target
    assert bool((j >= 0).all()), what
    ok = ~(tie | tie_rev[j])
    pk = d["peak_affs"].to(DEV).double()
    e_p = max((pk[ok, 0] - first[ok]).abs().max().item(), (pk[ok, 1] - second[ok]).abs().max().item())
    e_r = (d["r"].to(DEV).double()[ok] - torch.maximum(r, r_rev[j])[ok]).abs().max().item()
    assert e_p <= COS_TOL and e_r <= R_TOL, (what, e_p, e_r)
    return e_p, e_r, int((~ok).sum())


# ---- 1. best buddies --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,T,C", BB_SHAPES, ids=_ids(BB_SHAPES))
def test_best_buddies_against_float64(H, W, T, C):
    from dino_tracker_b200.best_buddies import PackedFeatures, best_buddies, nearest_neighbours
    t0 = time.perf_counter()
    geo, feats, ladders = _bb_video(H, W, T, C)
    P = geo.P
    t1 = _sync_time()
    pk = PackedFeatures(feats)
    pairs = [(s, t) for s in range(T) for t in range(s + 1, T)]
    ordered = [p for (s, t) in pairs for p in ((s, t), (t, s))]
    nn_idx, nn_cos = nearest_neighbours(pk.tpc, pk.norms, pk.geom, ordered)
    bb = best_buddies(feats, H, W)
    t2 = _sync_time()
    f64 = _unit64(feats)
    coords = obb.token_coords(H, W).to(DEV)
    ar = torch.arange(P, device=DEV)
    worst, n_excl, n_other, n_mutual, n_ladder_checked = 0.0, 0, 0, 0, 0
    for k, (s, t) in enumerate(pairs):
        ri, rg, ci, cg = _top2_64(f64[s], f64[t])
        st, ts = nn_idx[2 * k], nn_idx[2 * k + 1]
        m_st, m_ts = ts.long()[st.long()] == ar, st.long()[ts.long()] == ar
        for nn, cos, mk, best, gap, bb_, bg, a, b, x, y in (
                (st, nn_cos[2 * k], m_st, ri, rg, ci, cg, f64[s], f64[t], s, t),
                (ts, nn_cos[2 * k + 1], m_ts, ci, cg, ri, rg, f64[t], f64[s], t, s)):
            e, ne, no = _check_rows(nn, cos, mk, best, gap, bb_, bg, a, b, f"{H}x{W} {x}_{y}")
            worst, n_excl, n_other = max(worst, e), n_excl + ne, n_other + no
            n_mutual += int(mk.sum())
            # best_buddies' dict is the mutual rows of the same search
            d = bb[f"{x}_{y}"]
            assert torch.equal(d["source_coords"], coords[mk])
            assert torch.equal(d["target_coords"], coords[nn[mk].long()])
            assert torch.equal(d["cos_sims"], cos[mk])
            for n, copies in ladders.get((x, y), []):   # the ladders are what they claim: the row arg-max is a copy
                assert int(best[n]) in copies, (x, y, n)
                n_ladder_checked += int(gap[n] >= DELTA_BB)
    t3 = _sync_time()
    print(f"[best buddies {H}x{W} ({geo.h}x{geo.w} = {P} tokens, {-(-P // TILE)} column tiles) T={T} C={C}] "
          f"{len(ordered)} ordered pairs, {n_mutual} mutual rows; max |nn_cos - float64| {worst:.2e}; {n_excl} rows "
          f"excluded from the mutual check (float64 gap < {DELTA_BB:g}), {n_other} resolved to another near-tied token; "
          f"{n_ladder_checked} ladder rows above the gap bar.  Time: inputs {t1 - t0:.1f} s, kernels {t2 - t1:.2f} s, "
          f"float64 reference {t3 - t2:.1f} s")
    assert n_mutual > P * len(ordered) // 4
    assert n_excl < P * len(ordered) // 1000 + 200
    assert n_ladder_checked >= 20


def test_refined_best_buddies_at_1274x714_against_float64():
    """contrastive.refined_best_buddies (the in-training search: the same kernels, self pairs allowed) on 181 x 101 token
    frames with the planted ladders, a self pair and a pair whose column side carries ladders."""
    from dino_tracker_b200.contrastive import refined_best_buddies
    H, W, T, C = BB_SHAPES[0]
    geo, feats, _ = _bb_video(H, W, T, C)
    pairs = [(0, 1), (2, 2), (2, 3), (1, 3)]
    mutual, partner, cos_at = refined_best_buddies(feats.to(DEV), pairs, H, W)
    f64 = _unit64(feats)
    worst, n_excl, n_other = 0.0, 0, 0
    for k, (s, t) in enumerate(pairs):
        ri, rg, ci, cg = _top2_64(f64[s], f64[t])
        e, ne, no = _check_rows(partner[k], cos_at[k], mutual[k], ri, rg, ci, cg, f64[s], f64[t], f"refined {s}_{t}")
        worst, n_excl, n_other = max(worst, e), n_excl + ne, n_other + no
        if s == t:
            assert bool(mutual[k].all()) and torch.equal(partner[k], torch.arange(geo.P, device=DEV))
    print(f"[refined best buddies {H}x{W}] max |cos - float64| {worst:.2e}; {n_excl} rows excluded from the mutual check, "
          f"{n_other} resolved to another near-tied token")


# ---- 2. peak filter ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,T,C", BB_SHAPES, ids=_ids(BB_SHAPES))
def test_peak_filter_against_float64(H, W, T, C):
    """compute_bb_nms, compute_max_r and nms_dict on the best buddies of pair (0, 1) at box_size 30 (preprocessing.yaml)
    and 50 (the script's default).  The coordinate grid is the frame's own token grid: the reference script's run()
    builds create_meshgrid(h=476, w=854) whatever the frame size, which indexes past its end above 8,107 tokens;
    run_nms / compute_bb_nms take the grid from the features, and the oracle below is given token_coords(H, W)."""
    from dino_tracker_b200.best_buddies import PackedFeatures, best_buddies, compute_bb_nms, nms_dict
    geo, feats, _ = _bb_video(H, W, T, C)
    pk = PackedFeatures(feats)
    bb = best_buddies(feats, H, W, unordered_pairs=[(0, 1)])
    f64 = _unit64(feats)
    for box in (30, 50):
        t0 = _sync_time()
        sub = {k: dict(v) for k, v in bb.items()}
        nms_dict(sub, pk, 7, box, IOU)
        t1 = _sync_time()
        res = [_check_peaks(sub[f"{s}_{t}"], sub[f"{t}_{s}"], s, t, f64, geo, box, f"{H}x{W} box {box} {s}_{t}")
               for s, t in ((0, 1), (1, 0))]
        n = sum(sub[k]["r"].shape[0] for k in sub)
        print(f"[peak filter {H}x{W} box {box}] {n} maps; max |peak - float64| {max(r[0] for r in res):.2e}, max |r - "
              f"float64| {max(r[1] for r in res):.2e}; {sum(r[2] for r in res)} rows excluded (float64 near-tie at the "
              f"arg-max or the rank-{TOPK} test); kernels {t1 - t0:.2f} s")
        assert sum(r[2] for r in res) <= n // 100 + 5
    # the greedy-NMS restatement (torchvision.ops.batched_nms) on 200 source points
    got = compute_bb_nms(bb["0_1"], 0, 1, pk, box_size=30, iou_thresh=IOU)
    sub = {k: v.cpu()[:200] for k, v in bb["0_1"].items()}
    ref = onms.compute_bb_nms(sub, 0, 1, feats, obb.token_coords(H, W), box_size=30, iou_thresh=IOU)
    _, _, _, tie = _peaks64(f64[0], f64[1], _tokens(sub["source_coords"], geo), geo, 30)
    ok = ~tie.cpu()
    e_p = (got["peak_affs"].cpu()[:200][ok] - ref["peak_affs"][ok]).abs().max().item()
    e_r = (got["r"].cpu()[:200][ok] - ref["r"][ok]).abs().max().item()
    print(f"[peak filter {H}x{W} vs greedy NMS, 200 maps] max |peak| {e_p:.2e}, max |r| {e_r:.2e}; {int(tie.sum())} excluded")
    assert e_p <= COS_TOL and e_r <= R_TOL


def test_peak_values_at_shipped_width_476x854():
    """The reduced case of test_peak_filter_against_float64: at C = 1024 the peak values of maps from the split-fp16
    tensor-core GEMM were up to 9e-6 off float64 (its accumulation error grows with C; the tests at C <= 256 stayed
    within the bar), so the peak filter's maps come from the exact-fp32 correlation GEMM."""
    from dino_tracker_b200.best_buddies import PackedFeatures, compute_bb_nms
    geo = Geometry()
    T, C = 2, 1024
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=79, noise=0.3, max_shift=2)
    toks = torch.arange(0, geo.P, 27, device=DEV)
    d = {"source_coords": obb.token_coords(geo.H, geo.W).to(DEV)[toks]}
    got = compute_bb_nms(d, 0, 1, PackedFeatures(feats), box_size=30, iou_thresh=IOU)
    first, second, r, tie = _peaks64(*_unit64(feats), toks, geo, 30)
    ok = ~tie
    pk = got["peak_affs"].double()
    e_p = max((pk[ok, 0] - first[ok]).abs().max().item(), (pk[ok, 1] - second[ok]).abs().max().item())
    e_r = (got["r"].double()[ok] - r[ok]).abs().max().item()
    print(f"[peak values 476x854 C=1024, {toks.shape[0]} maps] max |peak - float64| {e_p:.2e}, max |r - float64| "
          f"{e_r:.2e}; {int(tie.sum())} rows excluded")
    assert e_p <= COS_TOL and e_r <= R_TOL


# ---- 3. trajectories and the flow filter ------------------------------------------------------------------------------
EXACT_CASES = [(1025, 1025, False), (1025, 1025, True), (513, 1025, False), (513, 1025, True)]


@pytest.mark.parametrize("H,W,direct", EXACT_CASES)
def test_chaining_exact_on_integer_flows_large(H, W, direct):
    """Whole-pixel flows on (2^a + 1) x (2^b + 1) frames above 476 x 854 (oracle.make_golden_preprocess.TRAJ_CASES'
    construction): every operation is exact, so masks, trajectories and their count equal the oracle's bit for bit."""
    from dino_tracker_b200.trajectories import chain_trajectories, flow_masks
    T = 5
    thr, min_len, dthr = (1.5, 3, 2.5) if direct else (1.0, 2, None)
    flow = otr.smooth_flows(T, H, W, seed=H + W + int(direct), amplitude=6.0, integer=True, device=DEV)
    fwd, bwd, dfn = otr.stack_flows(flow, T)
    assert torch.equal(flow_masks(fwd, bwd, thr), otr.flow_masks(fwd, bwd, thr)[..., 0])
    d = dfn if direct else None
    got = chain_trajectories(fwd, bwd, d, thr, min_len, dthr)
    ora = otr.extract_trajectories(fwd, bwd, d, thr, min_len, dthr)
    valid = ~got.isnan().any(dim=-1)
    print(f"[exact chaining {H}x{W} direct={direct}] {got.shape[0]} trajectories (oracle {ora.shape[0]}), mean length "
          f"{valid.sum(1).float().mean().item():.2f}")
    assert got.shape[0] > 10_000
    assert _same(got, ora), (got.shape, ora.shape)


def _smooth_traj(H, W, T, seed, direct=False, **kw):
    fwd, bwd, dfn = otr.stack_flows(otr.smooth_flows(T, H, W, seed=seed, device=DEV, **kw), T)
    return fwd, bwd, (dfn if direct else None)


@pytest.mark.parametrize("direct", [False, True])
@pytest.mark.parametrize("H,W", [(1274, 714), (714, 1274)])
def test_chaining_smooth_flows_large(H, W, direct):
    """Smooth fractional flows: survivor sets within 0.01 %, positions within max(1e-4 px, 2 ulp) -- 2.4e-4 px above
    x = 1024 (test_preprocess_gpu.test_chaining_smooth_flows_full_size's rules)."""
    from dino_tracker_b200.trajectories import chain_trajectories
    T = 6
    fwd, bwd, d = _smooth_traj(H, W, T, 87 + H, direct, amplitude=3.0, noise=False)
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
    print(f"[smooth chaining {H}x{W} direct={direct}] {len(ko)} trajectories, {diff} differ, max |dxy| {err:.3g} px")
    assert _close(a[both], b[both])
    assert (a.isnan() != b.isnan()).any(dim=-1).any(dim=-1).sum().item() <= 1e-4 * len(ko)


def test_nearest_trajectory_at_1274x1274():
    """32,761 token centres (181 x 181), 60,000 trajectories on a quarter-pixel lattice (exact equidistant ties), a third
    of the positions NaN, duplicated rows, frame 3 all NaN."""
    from dino_tracker_b200.best_buddies import nearest_trajectories
    g = torch.Generator().manual_seed(97)
    M, T, H, W = 60_000, 4, 1274, 1274
    traj = (torch.rand(M, T, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0]) * 4).round() / 4
    traj[torch.rand(M, T, generator=g) < 0.33] = float("nan")
    traj[:, 3] = float("nan")
    traj[40_000:40_100] = traj[100:200]
    got = nearest_trajectories(traj.to(DEV), H, W, 7)
    ref = oof.nearest_grid(traj.to(DEV), H, W, 7)
    assert got.shape == (T, 181, 181)
    assert torch.equal(got, ref)
    assert (got[3] == 0).all()


def test_nearest_trajectory_past_2_31_floats():
    """M = 11 M trajectories of T = 100 frames: M T 2 = 2.2e9 floats (8.8 GB, and as much again for the transposed copy
    in the workspace).  Every row is NaN except 5 at the start and 3,000 at the end of the array, so the oracle scans
    only those; the last 5 rows repeat the first 5 (equidistant ties across the whole array go to the first)."""
    from dino_tracker_b200.best_buddies import nearest_trajectories
    M, T, H, W = 11_000_000, 100, 714, 1274
    assert M * T * 2 > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(98)
    rows = torch.cat([torch.arange(0, 5), torch.arange(M - 3000, M)]).to(DEV)
    pos = (torch.rand(rows.shape[0], T, 2, generator=g, device=DEV) * torch.tensor([W - 1.0, H - 1.0], device=DEV) * 4
           ).round() / 4
    pos[torch.rand(rows.shape[0], T, generator=g, device=DEV) < 0.3] = float("nan")
    pos[:, 7] = float("nan")
    pos[-5:] = pos[:5]
    traj = torch.full((M, T, 2), float("nan"), device=DEV)
    traj[rows] = pos
    t0 = _sync_time()
    got = nearest_trajectories(traj, H, W, 7)
    t1 = _sync_time()
    ref = rows[oof.nearest_grid(pos, H, W, 7)]
    print(f"[nearest trajectory, M = {M}, T = {T}] kernel {t1 - t0:.2f} s; "
          f"{int((got >= M - 3000).sum())} of {got.numel()} answers in the last 3,000 rows")
    assert torch.equal(got, ref)
    assert (got[7] == 0).all() and bool((got >= M - 3000).any())
    del traj


def _large_traj(H, W, T, seed):
    """Trajectories of whole-pixel flows large enough to break many walks (test_preprocess_best_buddies_end_to_end's)."""
    from dino_tracker_b200.trajectories import chain_trajectories
    fwd, bwd, _ = _smooth_traj(H, W, T, seed, amplitude=6.0, integer=True)
    return chain_trajectories(fwd, bwd, None, 1.5, 2)


def test_of_filter_at_1274x714_matches_oracle():
    """The flow filter of the best buddies of test_best_buddies_against_float64's 1274 x 714 video by trajectories chained
    at that frame size: field for field the oracle's."""
    from dino_tracker_b200.best_buddies import best_buddies, of_filter
    H, W, T, C = BB_SHAPES[0]
    _, feats, _ = _bb_video(H, W, T, C)
    bb = best_buddies(feats, H, W)
    traj = _large_traj(H, W, T, 99)
    got = of_filter(bb, traj, H, W, 7)
    ref = oof.of_filter(bb, traj, H, W, 7)
    _bb_equal(got, ref)
    kept = sum(0 if v["source_coords"] is None else v["source_coords"].shape[0] for v in got.values())
    total = sum(v["source_coords"].shape[0] for v in bb.values())
    print(f"[flow filter {H}x{W}] {traj.shape[0]} trajectories; {kept} of {total} best buddies kept")
    assert 0 < kept < total


def test_preprocess_best_buddies_end_to_end_1274x714(tmp_path):
    """best buddies -> trajectories (synthetic flow_fn) -> flow filter -> peak filter in one process at 1274 x 714:
    best buddies against float64, trajectories against the oracle (test_chaining_smooth_flows_large's rules), the flow
    filter against the oracle's on them, peaks and r against float64."""
    from dino_tracker_b200.pipeline import preprocess_best_buddies
    H, W, T, C = 1274, 714, 3, 64
    geo = Geometry(H=H, W=W)
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=36, noise=0.5, max_shift=2)
    flow = otr.smooth_flows(T, H, W, seed=89, amplitude=6.0, integer=True, device=DEV)
    video = torch.arange(T, dtype=torch.float32).view(T, 1, 1, 1).expand(T, 3, H, W).contiguous() / 8

    def flow_fn(a, b):   # the frames carry their index in their (constant) value
        ia, ib = (x[:, 0, 0, 0].mul(8).round().long().tolist() for x in (a, b))
        return torch.stack([flow(i, j) for i, j in zip(ia, ib)])

    bb, traj, filt = preprocess_best_buddies(feats, video, str(tmp_path / "bb"), str(tmp_path / "traj" / "trajectories.pt"),
                                             H, W, flow_fn=flow_fn, threshold=1.5, box_size=30, iou_thresh=IOU)
    # step 1: best buddies against float64
    f64 = _unit64(feats)
    worst, n_excl = 0.0, 0
    for s in range(T):
        for t in range(s + 1, T):
            ri, rg, ci, cg = _top2_64(f64[s], f64[t])
            for x, y, best, gap, back, bgap in ((s, t, ri, rg, ci, cg), (t, s, ci, cg, ri, rg)):
                d = bb[f"{x}_{y}"]
                src, tgt = _tokens(d["source_coords"], geo), _tokens(d["target_coords"], geo)
                mk = torch.zeros(geo.P, dtype=torch.bool, device=DEV)
                mk[src] = True
                excl = (gap < DELTA_BB) | (bgap[best] < DELTA_BB)
                ref_m = back[best] == torch.arange(geo.P, device=DEV)
                assert not ((mk != ref_m) & ~excl).any(), (x, y)
                sure = ~excl[src]
                assert torch.equal(tgt[sure], best[src][sure]), (x, y)
                e = (d["cos_sims"].double() - (f64[x][src] * f64[y][tgt]).sum(1)).abs().max().item()
                assert e <= COS_TOL, (x, y, e)
                worst, n_excl = max(worst, e), n_excl + int(excl.sum())
    # step 2: trajectories against the oracle
    fwd, bwd, _ = otr.stack_flows(flow, T)
    ora = otr.extract_trajectories(fwd, bwd, None, 1.5, 2)
    kg, ko = _by_start(traj, W), _by_start(ora, W)
    common = sorted(set(kg) & set(ko))
    diff = len(set(kg) ^ set(ko))
    assert diff <= 1e-4 * len(ko), (diff, len(ko))
    a, b = traj[[kg[k] for k in common]], ora[[ko[k] for k in common]]
    assert (a.isnan() != b.isnan()).any(dim=-1).any(dim=-1).sum().item() <= 1e-4 * len(ko)
    both = ~(a.isnan() | b.isnan())
    assert _close(a[both], b[both])
    # step 3: the oracle's flow filter on the same best buddies and trajectories
    ref = oof.of_filter(bb, traj, H, W, 7)
    assert list(filt) == list(ref)
    n_kept, e_p, e_r, n_tie = 0, 0.0, 0.0, 0
    for k, v in ref.items():
        if v["source_coords"] is None:
            assert filt[k]["source_coords"] is None and filt[k]["r"] is None, k
            continue
        for f in ("source_coords", "target_coords", "cos_sims"):
            assert torch.equal(filt[k][f], v[f]), (k, f)
        n_kept += v["source_coords"].shape[0]
        # step 4: peaks and r against float64
        s, t = (int(x) for x in k.split("_"))
        p, r, nt = _check_peaks(filt[k], filt[f"{t}_{s}"], s, t, f64, geo, 30, f"end to end {k}")
        e_p, e_r, n_tie = max(e_p, p), max(e_r, r), n_tie + nt
    print(f"[end to end {H}x{W}] best buddies: max |cos - float64| {worst:.2e}, {n_excl} rows excluded; trajectories "
          f"{traj.shape[0]} ({diff} differ from the oracle); {n_kept} pairs kept by the flow filter; peaks max error "
          f"{e_p:.2e}, r {e_r:.2e}, {n_tie} rows excluded")
    assert n_kept > 0


# ---- 4. masks and the fg / bg split -----------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(181, 101, 1274, 714), (13, 256, 98, 1799)])
def test_mask_upsample_large(hw):
    from dino_tracker_b200 import fg_masks as fgm
    h, w, H, W = hw
    tm = torch.rand(3, h, w, generator=torch.Generator().manual_seed(h * w)) < 0.5
    ref = F.interpolate(tm.to(DEV)[None].float(), size=(H, W), mode="nearest")[0]
    got = fgm.upsample_mask(tm.to(DEV), (H, W))
    assert torch.equal(got, (ref * 255).to(torch.uint8))


@pytest.mark.parametrize("H,W", [(1274, 714), (714, 1274)])
def test_fg_bg_split_large(H, W):
    """Trajectories chained at the frame size, split by disc masks: fg and bg equal the oracle's bit for bit."""
    from dino_tracker_b200.fg_masks import split_trajectories
    T = 4
    traj = _large_traj(H, W, T, 101 + H)
    _, masks = ofg.split_case_inputs(1, T, H, W, seed=102)
    masks = masks.to(DEV)
    fg, bg = split_trajectories(traj, masks)
    print(f"[split {H}x{W}] {traj.shape[0]} trajectories, {fg.shape[0]} fg")
    assert fg.shape[0] > 1000 and bg.shape[0] > 1000
    assert _same(fg, ofg.mask_filter(traj, masks))
    assert _same(bg, ofg.mask_filter(traj, masks, filter_bg=True))

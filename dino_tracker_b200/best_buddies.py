"""Host mirror of ``preprocessing_dino_bb/extract_dino_best_buddies.py`` over libdinotrk.

``run(args)`` keeps the reference script's contract (``--dino-emb-path --h --w --stride --out-path``;
output ``dict['s_t'] -> {source_coords, target_coords, cos_sims}``, rows in ascending source-token
order).  The affinity matrices never reach HBM: every ordered pair runs through the wgmma split-fp16
GEMM with a fused top-2 epilogue, candidates are re-evaluated in exact fp32, and the mutual check
works on index vectors (``dinotrk_best_buddies_pairs`` / ``dinotrk_bb_mutual``).

Pairs shard trivially over ranks (``rank`` / ``world`` arguments): SURVEY.md 8e config 5.
"""
import ctypes
import math
import os
import warnings

import torch

from . import _lib


def token_coords(H, W, step=7, patch=14, device="cpu"):
    """``create_meshgrid`` of preprocessing_dino_bb/dino_bb_utils.py:5-15: pixel (x, y) of every token."""
    s = patch // 2
    x = torch.arange(s, W, step, device=device).float()
    y = torch.arange(s, H, step, device=device).float()
    yy, xx = torch.meshgrid(y, x, indexing="ij")
    return torch.stack([xx.reshape(-1), yy.reshape(-1)], dim=-1)


@torch.no_grad()
def nearest_neighbours(tpc, norms, geom, pairs, hi=None, lo=None, pairs_per_launch=48):
    """pairs: list of ordered (s, t).  Returns nn_idx [n_pairs][P] int32, nn_cos [n_pairs][P] fp32 (device)."""
    with torch.cuda.device(tpc.device):   # the library launches on the current device
        return _nearest_neighbours(tpc, norms, geom, pairs, hi, lo, pairs_per_launch)


def _nearest_neighbours(tpc, norms, geom, pairs, hi, lo, pairs_per_launch):
    lib = _lib.load()
    dev = tpc.device
    T, P, C = tpc.shape
    if hi is None:
        max_abs, min_norm, ok = _lib.split_range(tpc, norms, _lib.stream_ptr())
        if not ok and 0.0 < max_abs < math.inf:
            # Outside the split's faithful range the GEMM's ranking error can exceed the resolve margin.  Best buddies are
            # cosines only, so run on a copy scaled by 2^e (max |x| in (2^13, 2^14]): an exact scaling of every product,
            # sum and norm, so the exact-fp32 cosines of the copy are bit-identical to the video's own (wherever the video's
            # own products do not underflow and |d| |F| stays above the 1e-8 clamp).
            s = 2.0 ** (14 - math.ceil(math.log2(max_abs)))
            tpc, norms = tpc * s, norms * s
            max_abs, min_norm, ok = _lib.split_range(tpc, norms, _lib.stream_ptr())
        if not ok:   # a spread of token norms wider than the range (or non-finite features): no scale brings it inside
            warnings.warn(f"best buddies: feature video outside the fp16 split's faithful range even after rescaling (max |x| = "
                          f"{max_abs:.3g}, smallest token norm = {min_norm:.3g}, C = {C}): the affinity GEMM's ranking is not "
                          f"bounded by the exact-fp32 resolve margin", RuntimeWarning, stacklevel=3)
        hi, lo = _lib.split_fp16(tpc, _lib.stream_ptr())
    feat = _lib.make_features(tpc, norms, hi, lo)
    n = len(pairs)
    nn_idx = torch.empty(n, P, device=dev, dtype=torch.int32)
    nn_cos = torch.empty(n, P, device=dev, dtype=torch.float32)
    ws_bytes = lib.dinotrk_best_buddies_workspace_bytes(min(n, pairs_per_launch), P)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    pt = torch.tensor(pairs, dtype=torch.int32, device=dev).reshape(-1, 2)
    for i in range(0, n, pairs_per_launch):
        e = min(i + pairs_per_launch, n)
        src = pt[i:e, 0].contiguous()
        tgt = pt[i:e, 1].contiguous()
        _lib.check(lib.dinotrk_best_buddies_pairs(ctypes.byref(feat), ctypes.byref(geom), _lib.ptr(src), _lib.ptr(tgt),
                                                  e - i, _lib.ptr(nn_idx[i:e]), _lib.ptr(nn_cos[i:e]), _lib.ptr(ws),
                                                  ws_bytes, _lib.stream_ptr()), "best_buddies_pairs")
    return nn_idx, nn_cos


@torch.no_grad()
def best_buddies(features_chw, H, W, stride=7, patch=14, device="cuda:0", rank=0, world=1, unordered_pairs=None):
    """features_chw: T x C x h x w.  Returns the reference's dict for the unordered pairs owned by this rank
    (both orientations of each): {'s_t': {...}, 't_s': {...}}."""
    dev = _lib.require_cuda(device)
    with torch.cuda.device(dev):
        return _best_buddies(features_chw, H, W, stride, patch, dev, rank, world, unordered_pairs)


def _best_buddies(features_chw, H, W, stride, patch, dev, rank, world, unordered_pairs):
    lib = _lib.load()
    T, C, h, w = features_chw.shape
    geom = _lib.make_geom((h - 1) * stride + patch, (w - 1) * stride + patch, patch, stride, 35)
    assert (geom.h, geom.w) == (h, w)
    chw = features_chw.to(dev, torch.float32).contiguous()
    tpc = torch.empty(T, h * w, C, device=dev)
    norms = torch.empty(T, h * w, device=dev)
    _lib.check(lib.dinotrk_pack_features(_lib.ptr(chw), _lib.ptr(tpc), _lib.ptr(norms), T, C, h * w, _lib.stream_ptr()))
    del chw
    if unordered_pairs is None:
        unordered_pairs = [(s, t) for s in range(T) for t in range(s + 1, T)]
    mine = unordered_pairs[rank::world]
    ordered = [p for (s, t) in mine for p in ((s, t), (t, s))]
    nn_idx, nn_cos = nearest_neighbours(tpc, norms, geom, ordered)
    n = len(ordered)
    P = h * w
    mutual = torch.empty(n, P, device=dev, dtype=torch.uint8)
    # the partner of ordered pair 2k is 2k+1 and vice versa
    partner = nn_idx.view(-1, 2, P).flip(1).reshape(n, P).contiguous()
    _lib.check(lib.dinotrk_bb_mutual(_lib.ptr(nn_idx), _lib.ptr(partner), n, P, _lib.ptr(mutual), _lib.stream_ptr()))
    coords = token_coords(H, W, stride, patch, device=dev)
    out = {}
    mutual = mutual.bool()
    for k, (s, t) in enumerate(ordered):
        mk = mutual[k]
        out[f"{s}_{t}"] = {"source_coords": coords[mk], "target_coords": coords[nn_idx[k][mk].long()],
                          "cos_sims": nn_cos[k][mk]}
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Peak filter of the best-buddy pairs: preprocessing_dino_bb/compute_dino_bb_nms.py (SURVEY.md 8f-3)
class PackedFeatures:
    """Token-major copy of a T x C x h x w feature video on the GPU (+ norms): what ``compute_bb_nms`` needs of
    ``dino_emb``; pack once per video.  No fp16 hi / lo halves: the peak filter reports map values, so its maps come
    from the exact-fp32 correlation GEMM.  The split-fp16 tensor-core GEMM accumulates with an error that grows with C
    (about 9e-6 of a cosine at C = 1024, against 3e-7 in exact fp32)."""

    def __init__(self, features_chw, stride=7, patch=14, device="cuda:0"):
        lib = _lib.load()
        self.dev = _lib.require_cuda(device)
        T, C, h, w = features_chw.shape
        self.geom = _lib.make_geom((h - 1) * stride + patch, (w - 1) * stride + patch, patch, stride, 35)
        with torch.cuda.device(self.dev):
            chw = features_chw.to(self.dev, torch.float32).contiguous()
            self.tpc = torch.empty(T, h * w, C, device=self.dev)
            self.norms = torch.empty(T, h * w, device=self.dev)
            _lib.check(lib.dinotrk_pack_features(_lib.ptr(chw), _lib.ptr(self.tpc), _lib.ptr(self.norms), T, C, h * w, _lib.stream_ptr()))
        self.feat = _lib.make_features(self.tpc, self.norms)


@torch.no_grad()
def compute_bb_nms(dino_bb_sf_tf, sf, tf, dino_emb, coords=None, stride=7, box_size=50, iou_thresh=0.2, topk=400):
    """compute_dino_bb_nms.py:50-70.  ``dino_emb``: T x C x h x w features or a ``PackedFeatures``.  For every source point
    of the pair: its similarity map against frame ``tf`` (the tracker's exact-fp32 correlation kernels), then per map the two largest
    values surviving box NMS among the ``topk`` largest and their ratio r (``dinotrk_bb_nms``).  ``coords`` is accepted for
    signature parity (the token grid is implied by the features)."""
    lib = _lib.load()
    pk = dino_emb if isinstance(dino_emb, PackedFeatures) else PackedFeatures(dino_emb, stride=stride)
    g = pk.geom
    src = dino_bb_sf_tf["source_coords"].to(pk.dev, torch.float32)
    n = int(src.shape[0])
    out = dict(dino_bb_sf_tf)
    out["peak_coords"] = None
    if n == 0:
        out["peak_affs"] = torch.zeros(0, 2, device=pk.dev)
        out["r"] = torch.zeros(0, device=pk.dev)
        return out
    half = g.patch // 2
    tok = ((src[:, 1] - half) / stride).int().long() * g.w + ((src[:, 0] - half) / stride).int().long()   # xy_to_fxy + .int()
    with torch.cuda.device(pk.dev):
        desc = pk.tpc[sf][tok].contiguous()
        dn = pk.norms[sf][tok].contiguous()
        grp = torch.tensor([[tf], [0], [n], [0]], dtype=torch.int32, device=pk.dev)
        ms = lib.dinotrk_map_stride(ctypes.byref(g))
        maps = torch.empty(n, ms, device=pk.dev)
        nb = lib.dinotrk_corr_maps_workspace_bytes(n, 1, pk.tpc.shape[2])
        ws = torch.empty(nb, device=pk.dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_corr_maps(ctypes.byref(pk.feat), ctypes.byref(g), _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(grp[0]),
                                         _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), 1, n, n, _lib.ptr(maps), _lib.ptr(ws),
                                         nb, _lib.stream_ptr()), "corr_maps")
        peak = torch.empty(n, 2, device=pk.dev)
        r = torch.empty(n, device=pk.dev)
        _lib.check(lib.dinotrk_bb_nms(_lib.ptr(maps), n, ctypes.byref(g), float(box_size), float(iou_thresh), int(topk),
                                      _lib.ptr(peak), _lib.ptr(r), _lib.stream_ptr()), "bb_nms")
    out["peak_affs"] = peak
    out["r"] = r
    return out


@torch.no_grad()
def compute_max_r(bb, bb_rev):
    """compute_dino_bb_nms.py:72-82, vectorised: a mutual pair's r is the larger of its two directions' values.  The
    reverse partner of pair i of ``bb`` is the pair of ``bb_rev`` whose source point is i's target point."""
    if bb["target_coords"].shape[0] == 0:
        return bb, bb_rev
    d = torch.cdist(bb["target_coords"].float(), bb_rev["source_coords"].float())
    rev = d.argmin(dim=1)
    assert torch.equal(bb_rev["target_coords"][rev].float(), bb["source_coords"].float()), "best buddies are not mutual"
    m = torch.maximum(bb["r"], bb_rev["r"][rev])
    bb["r"] = m
    bb_rev["r"][rev] = m
    return bb, bb_rev


def nms_dict(dino_bb, pk, stride=7, box_size=50, iou_thresh=0.2):
    """The loop of ``compute_dino_bb_nms.run`` over a best-buddy dict (in place; returns it).  ``pk``: PackedFeatures."""
    for key in list(dino_bb.keys()):
        if dino_bb[key]["source_coords"] is None:
            dino_bb[key]["peak_coords"] = dino_bb[key]["peak_affs"] = dino_bb[key]["r"] = None
            continue
        if dino_bb[key].get("r", None) is not None:
            continue
        sf, tf = int(key.split("_")[0]), int(key.split("_")[1])
        bb = compute_bb_nms(dino_bb[f"{sf}_{tf}"], sf, tf, pk, None, stride, box_size, iou_thresh)
        bb_rev = compute_bb_nms(dino_bb[f"{tf}_{sf}"], tf, sf, pk, None, stride, box_size, iou_thresh)
        bb, bb_rev = compute_max_r(bb, bb_rev)
        dino_bb[key], dino_bb[f"{tf}_{sf}"] = bb, bb_rev
    return dino_bb


def run_nms(args):
    """Drop-in for ``compute_dino_bb_nms.run`` (same argparse namespace: dino_bb_path, dino_emb_path, out_path, stride,
    box_size, iou_thresh)."""
    dino_bb = torch.load(args.dino_bb_path)
    pk = PackedFeatures(torch.load(args.dino_emb_path, map_location="cpu"), stride=args.stride)
    nms_dict(dino_bb, pk, args.stride, args.box_size, args.iou_thresh)
    os.makedirs(os.path.dirname(args.out_path), exist_ok=True)
    torch.save(dino_bb, args.out_path)


# ---------------------------------------------------------------------------------------------------------------------
# Optical-flow filter of the best-buddy pairs: preprocessing_dino_bb/of_filter_dino_best_buddies.py (SURVEY.md 8f-3)
_BB_FIELDS = ("source_coords", "target_coords", "cos_sims", "peak_coords", "peak_affs", "r")


@torch.no_grad()
def nearest_trajectories(traj, h, w, stride=7):
    """of_filter_dino_best_buddies.py:51-56: [T][rows][columns] int64 index of the trajectory nearest to every token
    centre of create_meshgrid(h, w, stride) at every frame (``dinotrk_traj_nearest``)."""
    lib = _lib.load()
    dev = _lib.require_cuda(traj.device)
    traj = traj.to(dev, torch.float32).contiguous()
    M, T = traj.shape[:2]
    if M == 0:
        raise ValueError("no trajectories: the nearest trajectory is undefined (torch.argmin over an empty dimension)")
    gh, gw = len(range(7, h, stride)), len(range(7, w, stride))
    with torch.cuda.device(dev):
        out = torch.empty(T, gh, gw, device=dev, dtype=torch.int32)
        nb = lib.dinotrk_traj_nearest_workspace_bytes(M, T, gh, gw)
        ws = torch.empty(nb, device=dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_traj_nearest(_lib.ptr(traj), M, T, gh, gw, 7.0, float(stride), _lib.ptr(out), _lib.ptr(ws), nb,
                                            _lib.stream_ptr()), "traj_nearest")
    return out.long()


@torch.no_grad()
def of_filter(bb_dict, traj, h, w, stride=7):
    """of_filter_dino_best_buddies.run (:45-108) on in-memory inputs.  ``bb_dict``: 's_t' -> {source_coords,
    target_coords, cos_sims[, peak_coords, peak_affs, r]} for every ordered pair of the T = traj.shape[1] frames;
    ``traj`` [M][T][2].  Keeps the pairs whose points' nearest trajectories do not reach the other frame.  Returns the
    reference's dict: every field None for a pair with nothing kept, the optional fields None when absent."""
    lib = _lib.load()
    dev = _lib.require_cuda(traj.device if traj.is_cuda else "cuda:0")
    traj = traj.to(dev, torch.float32).contiguous()
    M, T = traj.shape[:2]
    keys = [f"{s}_{t}" for s in range(T) for t in range(T) if s != t]
    counts = [int(bb_dict[k]["source_coords"].shape[0]) for k in keys]
    with torch.cuda.device(dev):
        nearest = nearest_trajectories(traj, h, w, stride).int()
        src = torch.cat([bb_dict[k]["source_coords"].to(dev, torch.float32) for k in keys]).reshape(-1, 2).contiguous()
        tgt = torch.cat([bb_dict[k]["target_coords"].to(dev, torch.float32) for k in keys]).reshape(-1, 2).contiguous()
        pairs = torch.tensor([[int(x) for x in k.split("_")] for k in keys], dtype=torch.int32).reshape(-1, 2)
        pair_src, pair_tgt = pairs[:, 0].contiguous().to(dev), pairs[:, 1].contiguous().to(dev)
        offsets = torch.tensor([0] + counts, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)
        n = int(src.shape[0])
        keep = torch.zeros(n, device=dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_of_filter(_lib.ptr(traj), M, T, _lib.ptr(nearest), nearest.shape[1], nearest.shape[2], int(stride),
                                         _lib.ptr(src), _lib.ptr(tgt), _lib.ptr(pair_src), _lib.ptr(pair_tgt), _lib.ptr(offsets),
                                         len(keys), n, _lib.ptr(keep), _lib.stream_ptr()), "of_filter")
        keep = keep.bool().cpu()                                   # one read-back for all pairs
    out, i0 = {}, 0
    for k, c in zip(keys, counts):
        kp = keep[i0:i0 + c]
        i0 += c
        f = dict.fromkeys(_BB_FIELDS)
        if bool(kp.any()):
            bb = bb_dict[k]
            for name in _BB_FIELDS:
                v = bb.get(name, None)
                if v is not None:
                    f[name] = v[kp.to(v.device)]
        out[k] = f
    return out


def run_of_filter(args):
    """Drop-in for ``of_filter_dino_best_buddies.run`` (same argparse namespace: dino_bb_path, traj_path, out_path,
    dino_bb_stride, h, w)."""
    bb = torch.load(args.dino_bb_path)
    traj = torch.load(args.traj_path, map_location="cpu")
    out = of_filter(bb, traj, args.h, args.w, args.dino_bb_stride)
    os.makedirs(os.path.dirname(args.out_path), exist_ok=True)
    torch.save(out, args.out_path)
    print(f"Saved filtered best buddies to {args.out_path}")


def run(args):
    """Drop-in for ``extract_dino_best_buddies.run`` (same argparse namespace)."""
    feats = torch.load(args.dino_emb_path, map_location="cpu")
    bb = best_buddies(feats, args.h, args.w, stride=args.stride)
    os.makedirs(os.path.dirname(args.out_path), exist_ok=True)
    torch.save(bb, args.out_path)
    print(f"Saved best buddies to {args.out_path}")

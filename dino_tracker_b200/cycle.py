"""Cycle-consistency term of the training step (models/tracker.py:182-301, dino_tracker.py:346-353) on the CUDA path.

The reference loops over ``cyc_n_frames`` random (source, target) slot pairs: per pair a host ``randperm`` over the
source frame's foreground and one over its background pixels, two no-grad ``get_point_predictions`` calls (there and
back), the keep test, and then two more graph calls that repeat the survivors' predictions.  Here the same random draws
are made in the same order, but

* the randperms are exact prefixes (``dinotrk_randperm_prefix``): the first 179 / 77 entries in O(k), with the host
  generator left exactly where ``torch.randperm(n)`` leaves it;
* the drawn ranks are mapped to pixels on the device against a per-frame foreground scan cached per mask set;
* each leg is ONE batch over all pairs (sample, correlation maps grouped by target slot, head), the keep test and the
  survivors' compaction are kernels, and the host reads back one count;
* the graph predictions are the survivors' rows of those legs: one autograd node whose backward is one
  ``dinotrk_track_backward`` over both legs' survivor rows.

A map's arithmetic is that of ``TrackFunction``; only its grouping differs (all pairs with the same target slot form
one group).  A frame's group with at most 8 maps goes to the exact-fp32 streaming kernel, a wider one to the fp16x3
tensor-core GEMM (``csrc/corr.cu``), so a map whose group width crosses 8 between the reference's per-pair calls and
this batch moves within the fp16x3 path's 1e-3 px bar.
"""
import ctypes

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib
from . import train as _train

_RANDPERM_MAX = 2 ** 32 // 20      # torch's randperm_cpu draws 64-bit numbers from here on
_prefix_checked = None


def _prefix_raw(gen, n, k):
    """The first min(k, n) entries of ``torch.randperm(n, generator=gen)``; ``gen`` advanced as randperm advances it."""
    state = gen.get_state().contiguous()
    out = torch.empty(min(k, n), dtype=torch.int64)
    _lib.check(_lib.load().dinotrk_randperm_prefix(ctypes.c_void_p(state.data_ptr()), state.numel(), n, k,
                                                   ctypes.c_void_p(out.data_ptr())), "randperm_prefix")
    gen.set_state(state)
    return out


def _self_check():
    """The helper against torch.randperm on a private generator: prefix, whole permutation and the state afterwards."""
    try:
        for seed, n, k in ((7, 1000, 13), (8, 625, 625), (9, 5000, 5000)):
            a, b = torch.Generator().manual_seed(seed), torch.Generator().manual_seed(seed)
            torch.rand(401, generator=a)
            torch.rand(401, generator=b)
            want = torch.randperm(n, generator=a)[:k]
            if not torch.equal(_prefix_raw(b, n, k), want) or not torch.equal(a.get_state(), b.get_state()):
                return False
        return True
    except _lib.DinotrkError:
        return False


def randperm_prefix(n, k):
    """``torch.randperm(n)[:k]`` on the default CPU generator, with the same later draws.  O(k) through
    ``dinotrk_randperm_prefix`` once a self-check against torch.randperm has passed; torch.randperm otherwise."""
    global _prefix_checked
    if _prefix_checked is None:
        _prefix_checked = _self_check()
    if _prefix_checked and n < _RANDPERM_MAX:
        return _prefix_raw(torch.default_generator, n, k)
    return torch.randperm(n)[:k]


def _mask_table(tracker, fg_masks):
    """(fg [T][P] uint8, off [T][blocks], host list of per-frame foreground counts) of a mask set, cached on the tracker
    for the same tensor at the same version."""
    cached = getattr(tracker, "_cyc_masks", None)
    if cached is not None and cached[0] is fg_masks and cached[1] == fg_masks._version:
        return cached[2]
    dev = tracker._dev
    T, H, W = fg_masks.shape[-3:]
    P = H * W
    fg = (fg_masks > 0).to(device=dev, dtype=torch.uint8).reshape(T, P).contiguous()
    lib = tracker._lib
    off = torch.empty(T, -(-P // 256), device=dev, dtype=torch.int32)
    n_fg = torch.empty(T, device=dev, dtype=torch.int32)
    ws_bytes = lib.dinotrk_cycle_mask_workspace_bytes(T, P)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    _lib.check(lib.dinotrk_cycle_mask_scan(_lib.ptr(fg), T, P, _lib.ptr(off), _lib.ptr(n_fg), _lib.ptr(ws), ws_bytes,
                                           _lib.stream_ptr(dev)), "cycle_mask_scan")
    table = (fg, off, n_fg.tolist())
    tracker._cyc_masks = (fg_masks, fg_masks._version, table)
    return table


def _groups(slots, lengths):
    """Pairs ordered by slot (stable): (pair order, [4][groups] = slot, first row, rows, first map, widest group)."""
    order = sorted(range(len(slots)), key=lambda p: slots[p])
    grp, row = [], 0
    for p in order:
        if lengths[p] == 0:
            continue
        if grp and grp[-1][0] == slots[p]:
            grp[-1][2] += lengths[p]
        else:
            grp.append([slots[p], row, lengths[p], row])
        row += lengths[p]
    return order, np.array(grp, dtype=np.int32).T.reshape(4, -1), max(g[2] for g in grp)


def _leg(tracker, e, feat, hw, pts, grp, widest, out_index):
    """One batch of maps: descriptors at pts [R][3] = (x_px, y_px, slot), maps grouped as grp, head with aux; the
    normalised (x, y) of row j lands in row out_index[j] of the output."""
    lib, dev, geom = tracker._lib, tracker._dev, tracker._geom
    N, P, C = e.shape
    R = pts.shape[0]
    st = _lib.stream_ptr(dev)
    slots = torch.arange(N, device=dev, dtype=torch.int32)
    desc = torch.empty(R, C, device=dev, dtype=torch.float32)
    dn = torch.empty(R, device=dev, dtype=torch.float32)
    _lib.check(lib.dinotrk_sample_descriptors(_lib.ptr(e), N, C, ctypes.byref(geom), _lib.ptr(pts), R, _lib.ptr(slots), N, 0,
                                              _lib.ptr(desc), _lib.ptr(dn), st), "sample_descriptors")
    n_groups = grp.shape[1]
    maps = torch.empty(R, lib.dinotrk_map_stride(ctypes.byref(geom)), device=dev, dtype=torch.float32)
    ws_bytes = lib.dinotrk_corr_maps_workspace_bytes(R, n_groups, C)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    _lib.check(lib.dinotrk_corr_maps(ctypes.byref(feat), ctypes.byref(geom), _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(grp[0]),
                                     _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), n_groups, R, widest, _lib.ptr(maps),
                                     _lib.ptr(ws), ws_bytes, st), "corr_maps")
    out = torch.empty(R, 2, device=dev, dtype=torch.float32)
    aux = torch.empty(R, 2, device=dev, dtype=torch.int32)
    _lib.check(lib.dinotrk_head(_lib.ptr(maps), R, ctypes.byref(geom), ctypes.byref(hw), _lib.ptr(out_index), _lib.ptr(out),
                                2, 1, _lib.ptr(aux), None, st), "head")
    return out, desc, dn, maps, aux


@torch.no_grad()
def draw(tracker, frames_set_t, fg_masks, emb_chw):
    """One draw of models/tracker.py:183-267 for all pairs.  Returns (the reference's no-grad dict, the survivors' rows
    of both legs for ``predictions``)."""
    lib, dev = tracker._lib, tracker._dev
    n_pairs, n_set = tracker.cyc_n_frames, frames_set_t.shape[0]
    sel_dev = frames_set_t.device                  # randint on the frame set's device, as the reference draws
    src_sel = torch.randint(n_set, (n_pairs,), device=sel_dev)
    tgt_sel = torch.randint(n_set, (n_pairs,), device=sel_dev)
    T, H, W = fg_masks.shape[-3:]
    P = H * W
    fg, off, counts = _mask_table(tracker, fg_masks)
    sel = torch.cat([src_sel, tgt_sel, frames_set_t.to(sel_dev).long()]).tolist()       # the one read-back of the draws
    src, tgt, fs = sel[:n_pairs], sel[n_pairs:2 * n_pairs], sel[2 * n_pairs:]
    if fs and (min(fs) < 0 or max(fs) >= T):
        raise IndexError(f"frames_set_t must index the {T} foreground masks, got {fs}")
    n_fg = int(tracker.cyc_batch_size_per_frame * tracker.cyc_fg_points_ratio)
    n_bg = tracker.cyc_batch_size_per_frame - n_fg
    blocks, lengths = [], []
    for s, t in zip(src, tgt):                     # per pair: foreground then background randperm, in pair order
        ts, tt = fs[s], fs[t]
        for is_fg, ranks in ((1, randperm_prefix(counts[ts], n_fg)), (0, randperm_prefix(P - counts[ts], n_bg))):
            b = np.empty((ranks.shape[0], 8), dtype=np.int32)
            b[:] = (ts, is_fg, 0, s, t, tt, 0, 0)
            b[:, 2] = ranks.numpy()
            blocks.append(b)
        lengths.append(blocks[-1].shape[0] + blocks[-2].shape[0])
    rows = np.concatenate(blocks)
    R = rows.shape[0]
    if R == 0:
        raise ValueError("cyc_batch_size_per_frame must be positive: a draw without points never yields a survivor")
    first = np.cumsum([0] + lengths[:-1])
    there_pairs, grp_there, wide_there = _groups(tgt, lengths)
    back_pairs, grp_back, wide_back = _groups(src, lengths)
    there_order = np.concatenate([np.arange(first[p], first[p] + lengths[p]) for p in there_pairs]).astype(np.int32)
    back_order = np.concatenate([np.arange(first[p], first[p] + lengths[p]) for p in back_pairs]).astype(np.int32)
    rows[there_order, 6] = np.arange(R)
    rows[back_order, 7] = np.arange(R)
    flat = torch.from_numpy(np.concatenate([rows.reshape(-1), there_order, back_order, grp_there.reshape(-1),
                                            grp_back.reshape(-1)])).to(dev)                   # one upload
    rows_d = flat[:8 * R].view(R, 8)
    there_order_d, back_order_d = flat[8 * R:9 * R], flat[9 * R:10 * R]
    g0 = 10 * R
    grp_there_d = flat[g0:g0 + grp_there.size].view(4, -1)
    grp_back_d = flat[g0 + grp_there.size:].view(4, -1)

    st = _lib.stream_ptr(dev)
    start = torch.empty(R, 3, device=dev, dtype=torch.float32)
    there_pts = torch.empty(R, 3, device=dev, dtype=torch.float32)
    _lib.check(lib.dinotrk_cycle_select(_lib.ptr(fg), T, H, W, _lib.ptr(off), _lib.ptr(rows_d), R, _lib.ptr(start),
                                        _lib.ptr(there_pts), st), "cycle_select")
    N, C, h, w = emb_chw.shape
    e = emb_chw.detach().permute(0, 2, 3, 1).reshape(N, h * w, C).contiguous()
    norms = torch.empty(N, h * w, device=dev, dtype=torch.float32)
    _lib.check(lib.dinotrk_token_norms(_lib.ptr(e), _lib.ptr(norms), N, C, h * w, st), "token_norms")
    feat = tracker.features_struct(e, norms)
    head = tracker.tracker_head.cnn_refiner
    hw = _train._head_struct(head[0].normalized_weight_graph(), head[0].bias, head[2].normalized_weight_graph(), head[2].bias)
    there_out, desc_t, dn_t, maps_t, aux_t = _leg(tracker, e, feat, hw, there_pts, grp_there_d, wide_there, there_order_d)
    there_px = torch.empty(R, 3, device=dev, dtype=torch.float32)
    back_pts = torch.empty(R, 3, device=dev, dtype=torch.float32)
    _lib.check(lib.dinotrk_cycle_unnorm(_lib.ptr(there_out), _lib.ptr(rows_d), R, H, W, _lib.ptr(there_px), _lib.ptr(back_pts),
                                        st), "cycle_unnorm")
    back_out, desc_b, dn_b, maps_b, aux_b = _leg(tracker, e, feat, hw, back_pts, grp_back_d, wide_back, back_order_d)
    keep_rows = torch.empty(R, device=dev, dtype=torch.int32)
    cycle_px = torch.empty(R, 2, device=dev, dtype=torch.float32)
    n_keep = torch.empty(1, device=dev, dtype=torch.int32)
    _lib.check(lib.dinotrk_cycle_keep(_lib.ptr(start), _lib.ptr(back_out), R, H, W, float(tracker.cyc_thresh),
                                      _lib.ptr(keep_rows), _lib.ptr(cycle_px), _lib.ptr(n_keep), st), "cycle_keep")
    m = int(n_keep.item())                         # the one read-back for the output shapes
    kr = keep_rows[:m].long()
    rk = rows_d[kr].long()
    out = {"source_points": start[kr], "target_points": there_px[kr], "cycle_points": cycle_px[:m],
           "source_frame_indices": rk[:, 3], "target_frame_indices": rk[:, 4]}
    for name, col in (("source", 0), ("target", 5)):
        t3 = rk[:, col].unsqueeze(1).repeat(1, 3).float()
        out[f"{name}_times_normalized"] = tracker.range_normalizer(t3, dst=(-1, 1), dims=[2])[:, 2]
    jt, jb = rk[:, 6], rk[:, 7]
    tgt_t, tgt_b = rows_d[there_order_d.long(), 4], rows_d[back_order_d.long(), 3]
    legs = {"e": e, "norms": norms, "hw": hw, "fwd": there_out[kr], "bwd": back_out[kr],
            "pts": torch.cat([there_pts[jt], back_pts[jb]]), "desc": torch.cat([desc_t[jt], desc_b[jb]]),
            "dn": torch.cat([dn_t[jt], dn_b[jb]]), "tgt": torch.cat([tgt_t[jt], tgt_b[jb]]).contiguous(),
            "maps": torch.cat([maps_t[jt], maps_b[jb]]), "aux": torch.cat([aux_t[jt], aux_b[jb]])}
    return out, legs


class CycleFunction(torch.autograd.Function):
    """(source -> target, target -> source) coords [m][2] of the survivors (normalised) = f(emb_tpc [N][P][C], w1n, b1, w2n,
    b2): the rows ``draw`` already computed, kept with their maps for one ``dinotrk_track_backward`` over both legs."""

    @staticmethod
    def forward(ctx, emb_tpc, w1n, b1, w2n, b2, tracker, legs):
        ctx.tracker, ctx.hw = tracker, legs["hw"]
        ctx.save_for_backward(legs["e"], legs["norms"], legs["pts"], legs["desc"], legs["dn"], legs["tgt"], legs["maps"],
                              legs["aux"])
        return legs["fwd"], legs["bwd"]

    @staticmethod
    @once_differentiable
    def backward(ctx, g_fwd, g_bwd):
        tracker = ctx.tracker
        lib, dev, geom = tracker._lib, tracker._dev, tracker._geom
        e, norms, pts, desc, dn, tgt, maps, aux = ctx.saved_tensors
        N, P, C = e.shape
        B = pts.shape[0]
        with torch.cuda.device(dev):
            g = torch.cat([g_fwd, g_bwd]).to(device=dev, dtype=torch.float32).contiguous()
            grad_w = torch.zeros(305, device=dev, dtype=torch.float32)
            grad_emb = torch.zeros_like(e) if ctx.needs_input_grad[0] else None
            slots = torch.arange(N, device=dev, dtype=torch.int32)
            ws_bytes = lib.dinotrk_track_backward_workspace_bytes(B, C, ctypes.byref(geom))
            ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            feat = _lib.make_features(e, norms)
            _lib.check(lib.dinotrk_track_backward(
                ctypes.byref(feat), ctypes.byref(geom), ctypes.byref(ctx.hw), _lib.ptr(pts), _lib.ptr(slots), N,
                _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(tgt), _lib.ptr(maps), _lib.ptr(aux), _lib.ptr(g), B,
                _lib.ptr(grad_w), _lib.ptr(grad_emb) if grad_emb is not None else None, _lib.ptr(ws), ws_bytes,
                _lib.stream_ptr(dev)), "track_backward")
        return (grad_emb, grad_w[:144].view(16, 1, 3, 3), grad_w[144:160], grad_w[160:304].view(1, 16, 3, 3), grad_w[304:305],
                None, None)


def predictions(tracker, emb_chw, legs):
    """(source_target_coords, target_source_coords) [m][2] with the graph to emb_chw and the refiner."""
    N, C, h, w = emb_chw.shape
    head = tracker.tracker_head.cnn_refiner
    return CycleFunction.apply(emb_chw.permute(0, 2, 3, 1).reshape(N, h * w, C), head[0].normalized_weight_graph(), head[0].bias,
                               head[2].normalized_weight_graph(), head[2].bias, tracker, legs)

"""Differentiable tracker forward for the training step (SURVEY.md 8f-4).

``dino_tracker.py:405-429`` calls ``model(inputs)`` with gradients enabled; the graph runs
``delta_dino -> refined embeddings -> sample -> correlation -> refiner -> soft-argmax`` (``models/tracker.py:113-129,
170-180, 303-325``).  Here the tracker part is ONE autograd node: its forward is the inference kernels with the maps kept
(``dinotrk_sample_descriptors`` + ``dinotrk_corr_maps`` + ``dinotrk_head``), its backward is ``dinotrk_track_backward``
(``csrc/train.cu``).  Inputs with gradient: the frame set's embeddings (token-major ``[N][P][C]``; the permutation from
the reference's ``N x C x h x w`` and everything upstream -- delta-DINO, the residual add -- stay torch graphs) and the
refiner's NORMALISED weights (the spatial-sum normalisation of ``conv_norm.py:34-46`` is a small torch graph on top).
"""
import ctypes

import torch

from . import _lib


def _head_struct(w1n, b1, w2n, b2):
    hw = _lib.HeadWeights()
    flat = torch.cat([w1n.detach().reshape(-1), b1.detach().reshape(-1), w2n.detach().reshape(-1),
                      b2.detach().reshape(-1)]).to("cpu", torch.float32)
    assert flat.numel() == 305, "the refiner is NormalizedConv2d(1, 16, 3) -> ReLU -> NormalizedConv2d(16, 1, 3)"
    ctypes.memmove(ctypes.addressof(hw), flat.numpy().ctypes.data, 305 * 4)
    return hw


def track_forward(tracker, emb_tpc, w1n, b1, w2n, b2, pts, tgt_slot):
    """The tracker node's forward: the inference kernels with the maps kept.  Returns (out [B][2] in the caller's row
    order, the head weights as passed to the kernels, saved) with saved = (emb, norms, pts_sorted, desc, dn, tgt_sorted,
    maps, aux, order, slots): the per-map rows of pts_sorted / desc / dn / tgt_sorted / maps / aux are sorted by target
    slot, row j being the caller's row order[j] -- the arguments ``dinotrk_track_backward`` takes."""
    lib, dev, geom = tracker._lib, tracker._dev, tracker._geom
    with torch.cuda.device(dev):
        emb = emb_tpc.detach().contiguous()
        N, P, C = emb.shape
        B = pts.shape[0]
        st = _lib.stream_ptr(dev)
        norms = torch.empty(N, P, device=dev, dtype=torch.float32)
        _lib.check(lib.dinotrk_token_norms(_lib.ptr(emb), _lib.ptr(norms), N, C, P, st), "token_norms")
        feat = tracker.features_struct(emb, norms)
        # maps grouped by target frame (the grouped GEMM's contract); results scattered back through `order`
        tgt = tgt_slot.to(dev).long()
        order = torch.argsort(tgt, stable=True)
        tgt_sorted = tgt[order].to(torch.int32).contiguous()
        uniq, counts = torch.unique_consecutive(tgt_sorted, return_counts=True)
        pts_sorted = pts.to(device=dev, dtype=torch.float32)[order].contiguous()
        slots = torch.arange(N, device=dev, dtype=torch.int32)
        desc = torch.empty(B, C, device=dev, dtype=torch.float32)
        dn = torch.empty(B, device=dev, dtype=torch.float32)
        _lib.check(lib.dinotrk_sample_descriptors(_lib.ptr(emb), N, C, ctypes.byref(geom), _lib.ptr(pts_sorted), B,
                                                  _lib.ptr(slots), N, 0, _lib.ptr(desc), _lib.ptr(dn), st), "sample_descriptors")
        row0 = (torch.cumsum(counts, 0) - counts).to(torch.int32)
        grp = torch.stack([uniq.to(torch.int32), row0, counts.to(torch.int32), row0]).contiguous()
        n_groups = int(uniq.shape[0])
        stride = lib.dinotrk_map_stride(ctypes.byref(geom))
        maps = torch.empty(B, stride, device=dev, dtype=torch.float32)
        ws_bytes = lib.dinotrk_corr_maps_workspace_bytes(B, n_groups, C)
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_corr_maps(ctypes.byref(feat), ctypes.byref(geom), _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(grp[0]),
                                         _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), n_groups, B, int(counts.max()),
                                         _lib.ptr(maps), _lib.ptr(ws), ws_bytes, st), "corr_maps")
        hw = _head_struct(w1n, b1, w2n, b2)
        out = torch.empty(B, 2, device=dev, dtype=torch.float32)
        aux = torch.empty(B, 2, device=dev, dtype=torch.int32)
        out_index = order.to(torch.int32).contiguous()
        # full-map head kernel for every map: exact on both branches of tracker_head.py:84-98
        _lib.check(lib.dinotrk_head(_lib.ptr(maps), B, ctypes.byref(geom), ctypes.byref(hw), _lib.ptr(out_index), _lib.ptr(out),
                                    2, 1, _lib.ptr(aux), None, st), "head")
    return out, hw, (emb, norms, pts_sorted, desc, dn, tgt_sorted, maps, aux, order, slots)


class TrackFunction(torch.autograd.Function):
    """coords[B, 2] (normalised, the output of ``Tracker.forward``) = f(emb_tpc [N][P][C], w1n, b1, w2n, b2).

    ``pts`` [B][3] = (x_px, y_px, source slot), ``tgt_slot`` [B] index the frame set (= the N rows of ``emb_tpc``)."""

    @staticmethod
    def forward(ctx, emb_tpc, w1n, b1, w2n, b2, pts, tgt_slot, tracker):
        out, hw, saved = track_forward(tracker, emb_tpc, w1n, b1, w2n, b2, pts, tgt_slot)
        ctx.tracker, ctx.hw = tracker, hw
        ctx.save_for_backward(*saved)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        tracker = ctx.tracker
        lib, dev, geom = tracker._lib, tracker._dev, tracker._geom
        emb, norms, pts_sorted, desc, dn, tgt_sorted, maps, aux, order, slots = ctx.saved_tensors
        N, P, C = emb.shape
        B = pts_sorted.shape[0]
        with torch.cuda.device(dev):
            g = grad_out.to(device=dev, dtype=torch.float32)[order].contiguous()
            grad_w = torch.zeros(305, device=dev, dtype=torch.float32)
            grad_emb = torch.zeros_like(emb) if ctx.needs_input_grad[0] else None
            ws_bytes = lib.dinotrk_track_backward_workspace_bytes(B, C, ctypes.byref(geom))
            ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            feat = _lib.make_features(emb, norms)
            _lib.check(lib.dinotrk_track_backward(
                ctypes.byref(feat), ctypes.byref(geom), ctypes.byref(ctx.hw), _lib.ptr(pts_sorted), _lib.ptr(slots), N,
                _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(tgt_sorted), _lib.ptr(maps), _lib.ptr(aux), _lib.ptr(g), B,
                _lib.ptr(grad_w), _lib.ptr(grad_emb) if grad_emb is not None else None, _lib.ptr(ws), ws_bytes,
                _lib.stream_ptr(dev)), "track_backward")
        return (grad_emb, grad_w[:144].view(16, 1, 3, 3), grad_w[144:160], grad_w[160:304].view(1, 16, 3, 3), grad_w[304:305],
                None, None, None)


class SampleFunction(torch.autograd.Function):
    """``Tracker.sample_embeddings`` with a graph: desc [B][C] = trilinear samples of emb_tpc [T][P][C] at pts [B][3] =
    (x_n, y_n, frame index), both in [-1, 1] x index space (models/tracker.py:96-111)."""

    @staticmethod
    def forward(ctx, emb_tpc, pts, tracker):
        emb = emb_tpc.detach().contiguous()
        slots = torch.arange(emb.shape[0], device=tracker._dev, dtype=torch.int32)
        desc, _ = tracker._sample(emb, pts, slots, normalized=True)
        ctx.tracker, ctx.shape = tracker, emb.shape
        ctx.save_for_backward(pts.to(device=tracker._dev, dtype=torch.float32).contiguous(), slots)
        return desc

    @staticmethod
    def backward(ctx, grad_desc):
        tracker = ctx.tracker
        pts, slots = ctx.saved_tensors
        T, P, C = ctx.shape
        with torch.cuda.device(tracker._dev):
            grad = torch.zeros(T, P, C, device=tracker._dev, dtype=torch.float32)
            g = grad_desc.to(torch.float32).contiguous()
            _lib.check(tracker._lib.dinotrk_sample_backward(T, C, ctypes.byref(tracker._geom), _lib.ptr(pts), pts.shape[0],
                                                            _lib.ptr(slots), T, 1, _lib.ptr(g), _lib.ptr(grad),
                                                            _lib.stream_ptr(tracker._dev)), "sample_backward")
        return grad, None, None


def sample_points(tracker, emb_chw, pts):
    T, C, h, w = emb_chw.shape
    if pts.shape[0] == 0:
        return emb_chw.new_zeros(0, C)
    return SampleFunction.apply(emb_chw.permute(0, 2, 3, 1).reshape(T, h * w, C), pts, tracker)


def track_points(tracker, emb_chw, inp):
    """``Tracker.get_point_predictions`` (models/tracker.py:175-180) with a graph: emb_chw N x C x h x w (the frame set's
    embeddings, may require grad), inp as in ``Tracker.forward``.  Returns B x 2 in [-1, 1]."""
    src_pts, src_idx, tgt_idx, _ = inp
    N, C, h, w = emb_chw.shape
    if src_pts.shape[0] == 0:                      # nothing to track (e.g. an empty cycle-consistency draw)
        return emb_chw.new_zeros(0, 2)
    emb_tpc = emb_chw.permute(0, 2, 3, 1).reshape(N, h * w, C)
    head = tracker.tracker_head.cnn_refiner
    pts = torch.cat([src_pts.to(tracker._dev, torch.float32)[:, :2], src_idx.to(tracker._dev).to(torch.float32)[:, None]], dim=1)
    return TrackFunction.apply(emb_tpc, head[0].normalized_weight_graph(), head[0].bias, head[2].normalized_weight_graph(),
                               head[2].bias, pts, tgt_idx, tracker)

"""Differentiable tracker forward for the training step (SURVEY.md 8f-4).

``dino_tracker.py:405-429`` calls ``model(inputs)`` with gradients enabled; the graph runs
``delta_dino -> refined embeddings -> sample -> correlation -> refiner -> soft-argmax`` (``models/tracker.py:113-129,
170-180, 303-325``).  Here the tracker part is ONE autograd node: its forward is the inference kernels with the maps kept
(``dinotrk_sample_descriptors`` + ``dinotrk_corr_maps`` + ``dinotrk_head``), its backward is ``dinotrk_track_backward``
(``csrc/train.cu``).  Inputs with gradient: the frame set's embeddings (token-major ``[N][P][C]``; the permutation from
the reference's ``N x C x h x w`` and the residual add stay torch graphs) and the refiner's NORMALISED weights (the
spatial-sum normalisation of ``conv_norm.py:34-46`` is a small torch graph on top).

Delta-DINO upstream of it is a second node, ``DeltaTrainFunction`` (``csrc/delta_train.cu``): per chunk of frames the
convolutions as split-precision wgmma GEMMs, BatchNorm on the batch statistics, BlurPool and the alignment, and the
reverse pass of all of it down to the 16 parameter gradients.
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

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


_CONV, _BN = (0, 4, 8, 12), (1, 5, 9, 13)


def _kmajor(w):
    """Conv weights [O][I][5][5] -> K-major [O][Kp] ([O][5][5][I_pad], I padded to 4, K to a multiple of 8): the layout
    of the forward's weight operand and of the weight gradient ``dinotrk_delta_train_backward`` writes."""
    w = w.detach().float().permute(0, 2, 3, 1)
    if w.shape[-1] % 4:
        w = torch.nn.functional.pad(w, (0, 4 - w.shape[-1] % 4))
    w = w.reshape(w.shape[0], -1)
    if w.shape[1] % 8:
        w = torch.nn.functional.pad(w, (0, 8 - w.shape[1] % 8))
    return w.contiguous()


def _from_kmajor(g, shape):
    O, I = shape[:2]
    ip = I + (-I) % 4
    return g[:, :25 * ip].reshape(O, 5, 5, ip)[..., :I].permute(0, 3, 1, 2).contiguous()


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])


class DeltaTrainFunction(torch.autograd.Function):
    """residual B x C x h x w = delta-DINO of one chunk of frames (one BatchNorm batch), aligned to the h x w token grid
    (``DeltaDINO.forward`` with a graph, widths multiples of 8).  Forward ``dinotrk_delta_train_forward`` (BatchNorm in the
    module's mode; train mode updates the running statistics), backward ``dinotrk_delta_train_backward``.  Inputs with
    gradient: the 16 parameters (conv weights, conv biases, BN weights, BN biases, layer order); frames get none."""

    @staticmethod
    def forward(ctx, frames, module, vit_hw, *params):
        lib = _lib.load()
        dev = frames.device
        bns = [module.layers[i] for i in _BN]
        training = bns[0].training
        assert all(bn.momentum is not None and bn.track_running_stats for bn in bns), "BatchNorm2d with momentum and running stats"
        # the C entry takes one mode, momentum and eps for the four BatchNorms
        assert all((bn.training, bn.momentum, bn.eps) == (training, bns[0].momentum, bns[0].eps) for bn in bns), \
            "delta-DINO's four BatchNorms must share their mode, momentum and eps"
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            fr = frames.detach().float().contiguous()
            B, _, H, W = fr.shape
            h, w = vit_hw
            C = module.channels[-1]
            ch, cw = H, W
            for _ in range(3):
                ch, cw = (ch - 1) // 2 + 1, (cw - 1) // 2 + 1
            ixs, iys = module.align_tables((ch, cw), (h, w), dev, vit_stride=module.vit_stride)
            chan = (ctypes.c_int * 5)(*module.channels)
            splits = [_lib.split_fp16(_kmajor(p), st) for p in params[0:4]]
            vecs = [p.detach().float().contiguous() for p in params[4:16]]
            for bn in bns:
                assert bn.running_mean.dtype == torch.float32 and bn.running_mean.is_contiguous() and bn.running_var.is_contiguous()
            saved_bytes = lib.dinotrk_delta_train_saved_bytes(B, H, W, chan)
            saved = torch.empty(saved_bytes, device=dev, dtype=torch.uint8)
            ws_bytes = lib.dinotrk_delta_train_forward_workspace_bytes(B, H, W, chan)
            work = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            res = torch.empty(B, h * w, C, device=dev, dtype=torch.float32)
            _lib.check(lib.dinotrk_delta_train_forward(
                _lib.ptr(fr), B, H, W, chan, _ptrs([s[0] for s in splits]), _ptrs([s[1] for s in splits]), _ptrs(vecs[0:4]),
                _ptrs(vecs[4:8]), _ptrs(vecs[8:12]), _ptrs([bn.running_mean for bn in bns]), _ptrs([bn.running_var for bn in bns]),
                int(training), float(bns[0].momentum), float(bns[0].eps), _lib.ptr(ixs), _lib.ptr(iys), h, w, _lib.ptr(res),
                _lib.ptr(saved), saved_bytes, _lib.ptr(work), ws_bytes, st), "delta_train_forward")
            if training:
                for bn in bns:
                    bn.num_batches_tracked.add_(1)
        ctx.module, ctx.training, ctx.hw = module, training, (h, w)
        # through save_for_backward, so that autograd frees the saved activations (~1.7 GB per 8 frames) after backward
        ctx.save_for_backward(fr, saved, ixs, iys, *params)
        return res.view(B, h, w, C).permute(0, 3, 1, 2)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        lib = _lib.load()
        fr, saved, ixs, iys, *params = ctx.saved_tensors
        dev = fr.device
        B, _, H, W = fr.shape
        h, w = ctx.hw
        module = ctx.module
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            chan = (ctypes.c_int * 5)(*module.channels)
            g = grad.to(torch.float32).permute(0, 2, 3, 1).contiguous()          # [B][h][w][C] = token-major
            wt = [None] + [_lib.split_fp16(p.detach().float().permute(1, 2, 3, 0).reshape(p.shape[1], -1).contiguous(), st)
                           for p in params[1:4]]
            vecs = [p.detach().float().contiguous() for p in params[8:16]]
            gw = [torch.empty(p.shape[0], _kmajor(p).shape[1], device=dev, dtype=torch.float32) for p in params[0:4]]
            gv = [torch.empty(p.shape[0], device=dev, dtype=torch.float32) for p in params[4:16]]
            ws_bytes = lib.dinotrk_delta_train_backward_workspace_bytes(B, H, W, chan)
            work = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            _lib.check(lib.dinotrk_delta_train_backward(
                _lib.ptr(fr), B, H, W, chan, _ptrs([t[0] if t else None for t in wt]), _ptrs([t[1] if t else None for t in wt]),
                _ptrs(vecs[0:4]), _ptrs(vecs[4:8]), int(ctx.training), _lib.ptr(ixs), _lib.ptr(iys), h, w, _lib.ptr(g),
                _lib.ptr(saved), saved.numel(), _ptrs(gw), _ptrs(gv[0:4]), _ptrs(gv[4:8]), _ptrs(gv[8:12]), _lib.ptr(work),
                ws_bytes, st), "delta_train_backward")
        grads = [_from_kmajor(gw[i], params[i].shape) for i in range(4)] + gv
        return (None, None, None, *[gr.to(p.dtype) for gr, p in zip(grads, params)])


def delta_train(module, frames, vit_hw):
    """``DeltaDINO.forward`` with a graph on the CUDA path: the aligned residual B x C x h x w of one chunk."""
    L = module.layers
    params = [L[i].weight for i in _CONV] + [L[i].bias for i in _CONV] + [L[i].weight for i in _BN] + [L[i].bias for i in _BN]
    return DeltaTrainFunction.apply(frames, module, tuple(int(v) for v in vit_hw), *params)


def sample_points(tracker, emb_chw, pts):
    T, C, h, w = emb_chw.shape
    if pts.shape[0] == 0:
        return emb_chw.new_zeros(0, C)
    return SampleFunction.apply(emb_chw.permute(0, 2, 3, 1).reshape(T, h * w, C), pts, tracker)


def token_rows(emb_chw):
    """N x C x h x w -> [N][P][C], as ``track_points`` reads the frame set.  A view (no copy) where the embeddings are
    token-major in memory, as the training forward's are."""
    N, C, h, w = emb_chw.shape
    return emb_chw.permute(0, 2, 3, 1).reshape(N, h * w, C)


class RegularisersFunction(torch.autograd.Function):
    """(norm_reg, angle_reg) = (mean_p |a/b - 1|, mean_p |d/(a b) - 1|) of the refined embeddings E and the raw DINO
    embeddings R, both token-major [n][P][C] (``get_emb_norm_regularization_loss`` / ``get_emb_angle_regularization_loss``
    of dino_tracker.py:136-146).  Forward ``dinotrk_emb_reg_forward``, backward ``dinotrk_emb_reg_backward``: the upstream
    gradients stay on the device, so the backward never waits for the host.  R is a constant (the raw features)."""

    @staticmethod
    def forward(ctx, E, R):
        if R.requires_grad:
            raise ValueError("RegularisersFunction: the raw embeddings R are constants and must not require grad")
        lib = _lib.load()
        dev = E.device
        E_, R_ = E.detach().contiguous(), R.detach().contiguous()
        n, P, C = E_.shape
        assert R_.shape == E_.shape and E_.dtype == R_.dtype == torch.float32
        with torch.cuda.device(dev):
            out = torch.empty(2, device=dev, dtype=torch.float32)
            aux = torch.empty(n * P, 3, device=dev, dtype=torch.float32)
            ws_bytes = lib.dinotrk_emb_reg_workspace_bytes(n, P)
            ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
            _lib.check(lib.dinotrk_emb_reg_forward(_lib.ptr(E_), _lib.ptr(R_), n, P, C, _lib.ptr(out), _lib.ptr(aux),
                                                   _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "emb_reg_forward")
        ctx.save_for_backward(E_, R_, aux)
        return out[0], out[1]

    @staticmethod
    @once_differentiable
    def backward(ctx, g_norm, g_angle):
        lib = _lib.load()
        E, R, aux = ctx.saved_tensors
        n, P, C = E.shape
        dev = E.device
        with torch.cuda.device(dev):
            zero = torch.zeros((), device=dev, dtype=torch.float32)
            g_n = zero if g_norm is None else g_norm.detach().float().contiguous()
            g_a = zero if g_angle is None else g_angle.detach().float().contiguous()
            dE = torch.empty_like(E)
            _lib.check(lib.dinotrk_emb_reg_backward(_lib.ptr(E), _lib.ptr(R), n, P, C, _lib.ptr(aux), _lib.ptr(g_n), _lib.ptr(g_a),
                                                    _lib.ptr(dE), _lib.stream_ptr()), "emb_reg_backward")
        return dE, None


def emb_regularisers(model):
    """(norm_reg, angle_reg) of the last training forward's ``model.frame_embeddings`` / ``model.raw_embeddings`` as one
    node: the two regularisers of dino_tracker.py:136-146 with a graph to the refined embeddings."""
    return RegularisersFunction.apply(token_rows(model.frame_embeddings), token_rows(model.raw_embeddings))


def track_points(tracker, emb_chw, inp):
    """``Tracker.get_point_predictions`` (models/tracker.py:175-180) with a graph: emb_chw N x C x h x w (the frame set's
    embeddings, may require grad), inp as in ``Tracker.forward``.  Returns B x 2 in [-1, 1]."""
    src_pts, src_idx, tgt_idx, _ = inp
    N, C, h, w = emb_chw.shape
    if src_pts.shape[0] == 0:                      # nothing to track (e.g. an empty cycle-consistency draw)
        return emb_chw.new_zeros(0, 2)
    emb_tpc = token_rows(emb_chw)
    head = tracker.tracker_head.cnn_refiner
    pts = torch.cat([src_pts.to(tracker._dev, torch.float32)[:, :2], src_idx.to(tracker._dev).to(torch.float32)[:, None]], dim=1)
    return TrackFunction.apply(emb_tpc, head[0].normalized_weight_graph(), head[0].bias, head[2].normalized_weight_graph(),
                               head[2].bias, pts, tgt_idx, tracker)

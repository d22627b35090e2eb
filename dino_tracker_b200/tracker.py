"""Host mirror of the reference ``models/tracker.py::Tracker`` (SURVEY.md 8b) over libdinotrk.

Same constructor kwargs, attributes, ``forward`` / ``load_weights`` / ``cache_refined_embeddings`` /
``sample_embeddings`` signatures and state-dict keys as the reference (``models/tracker.py:17-180,
303-325``), so ``dino_tracker.py::get_model`` and ``ModelInference`` use it unchanged.  All arithmetic is
in the CUDA kernels; this file only owns tensors and forwards calls.  With gradients enabled (the training step of
``dino_tracker.py:405-429``) ``forward`` builds a graph: delta-DINO as torch ops, the tracker as one autograd node
with hand-written forward and backward kernels (``train.py``, ``csrc/train.cu``); the cycle-consistency methods
(``models/tracker.py:182-301``) run all pairs as one batch (``cycle.py``).  The losses / optimiser loop of
``dino_tracker.py`` are ``trainer.py``'s.

Internal layout: features are kept token-major ``[T][P][C]`` (see include/dinotrk.h);
``refined_features`` / ``dino_embed_video`` expose zero-copy ``T x C x h x w`` views of them.
"""
import ctypes
import gc
import os
from pathlib import Path

import torch
import torch.nn as nn

from . import _lib
from . import cycle as _cycle
from . import train as _train
from .networks import DeltaDINO, TrackerHead
from .range_normalizer import RangeNormalizer

EPS = 1e-08


def _as_f32(t, device):
    return t.to(device=device, dtype=torch.float32).contiguous()


class Tracker(nn.Module):
    def __init__(self, video=None, ckpt_path="", dino_embed_path="", dino_patch_size=14, stride=7,
                 device="cuda:0", cyc_n_frames=4, cyc_batch_size_per_frame=256, cyc_fg_points_ratio=0.7,
                 cyc_thresh=4, dino_embed_video=None, delta_channels=None, corr_precision="fp16x3", _adopt_tpc=None):
        super().__init__()
        self.device = device
        self._dev = _lib.require_cuda(device)
        self._lib = _lib.load()
        self.stride = stride
        self.dino_patch_size = dino_patch_size
        self.dino_embed_path = dino_embed_path
        self.ckpt_path = ckpt_path
        self.cyc_n_frames = cyc_n_frames
        self.cyc_batch_size_per_frame = cyc_batch_size_per_frame
        self.cyc_fg_points_ratio = cyc_fg_points_ratio
        self.cyc_thresh = cyc_thresh
        self.video = video
        t, c, h, w = video.shape
        self._geom = _lib.make_geom(h, w, dino_patch_size, stride, 35)
        assert corr_precision in ("fp16x3", "fp32")
        # "fp16x3": wide correlation groups on wgmma tensor cores (fp16 hi/lo split, 3 passes, fp32-faithful);
        # "fp32"  : exact-fp32 FFMA GEMM on the CUDA cores (validation path)
        self.corr_precision = corr_precision
        self._refined_tpc = None
        self._refined_norms = None
        self._head_cache = (None, None)
        self._local = None   # (refined tpc, norms) of the last uncached forward without a graph
        self._graph = None   # (embeddings, raw, residual) of the last forward WITH a graph (training step)

        with torch.cuda.device(self._dev):
            if _adopt_tpc is not None:            # token-major features straight from the in-process ViT stage (no copy)
                self._dino_tpc = _adopt_tpc
                self._dino_norms = torch.empty(_adopt_tpc.shape[:2], device=self._dev, dtype=torch.float32)
                _lib.check(self._lib.dinotrk_token_norms(_lib.ptr(_adopt_tpc), _lib.ptr(self._dino_norms), _adopt_tpc.shape[0],
                                                          _adopt_tpc.shape[2], _adopt_tpc.shape[1], _lib.stream_ptr(self._dev)), "token_norms")
            elif dino_embed_video is not None:    # in-process features given as T x C x h x w
                self._set_dino(dino_embed_video)
            else:
                self.load_dino_embed_video()
        C = self._dino_tpc.shape[-1]
        channels = list(delta_channels) if delta_channels is not None else [3, 64, 128, 256, C]
        self.delta_dino = DeltaDINO(channels=channels, vit_stride=stride).to(self._dev)
        self.cmap_relu = nn.ReLU(inplace=True)
        self.tracker_head = TrackerHead(patch_size=dino_patch_size, step_h=stride, step_w=stride,
                                        video_h=h, video_w=w).to(self._dev)
        self.range_normalizer = RangeNormalizer(shapes=(w, h, t), device=self._dev)

    # ------------------------------------------------------------------ feature cache
    def _chw_view(self, tpc):
        T, P, C = tpc.shape
        return tpc.view(T, self._geom.h, self._geom.w, C).permute(0, 3, 1, 2)

    @_lib.on_device
    def _pack(self, chw):
        """T x C x h x w (any device) -> token-major [T][P][C] + per-token norms on the GPU."""
        chw = _as_f32(chw, self._dev)
        T, C, h, w = chw.shape
        assert (h, w) == (self._geom.h, self._geom.w), \
            f"feature grid {h}x{w} does not match the video ({self._geom.h}x{self._geom.w} tokens)"
        assert C % 4 == 0, "feature dimension must be a multiple of 4"
        tpc = torch.empty(T, h * w, C, device=self._dev, dtype=torch.float32)
        norms = torch.empty(T, h * w, device=self._dev, dtype=torch.float32)
        _lib.check(self._lib.dinotrk_pack_features(_lib.ptr(chw), _lib.ptr(tpc), _lib.ptr(norms), T, C, h * w,
                                                    _lib.stream_ptr(self._dev)), "pack_features")
        return tpc, norms

    @_lib.on_device
    def features_struct(self, tpc, norms, quant=False):
        """C struct for a [T][P][C] feature video (+ its cached fp16 hi/lo split in fp16x3 mode).  A video outside the
        split's faithful range gets no split: its contractions run on the exact-fp32 path (with a RuntimeWarning).
        quant: also the anchor phase's own operands, the int8 rows of the coarse pass and the interleaved split of the exact
        box GEMM (dinotrk_infer only; computed on first request and cached with the split)."""
        if self.corr_precision != "fp16x3" or tpc.shape[-1] % 8:
            return _lib.make_features(tpc, norms)
        # The split lives ON the tensor object it was computed from: a fresh feature tensor (uncached forward,
        # re-cached embeddings) never inherits the split of a dead tensor that happened to own the same address.
        # Feature tensors are written once by the kernel that creates them; _version guards torch-level in-place edits.
        split = getattr(tpc, "_dtk_split", None)
        if split is None or split[0] != tpc._version:
            hi, lo = _lib.split_features(tpc, norms, _lib.stream_ptr(self._dev))
            split = [tpc._version, hi, lo, None, None]
            tpc._dtk_split = split
        if quant and split[3] is None and split[1] is not None:
            split[3] = _lib.quantise_features(tpc, norms, _lib.stream_ptr(self._dev))
        if quant and split[4] is None and split[1] is not None:
            split[4] = _lib.split_hilo(tpc, _lib.stream_ptr(self._dev))
        return _lib.make_features(tpc, norms, split[1], split[2], split[3] if quant else None, split[4] if quant else None)

    def _set_dino(self, chw):
        self._dino_tpc, self._dino_norms = self._pack(chw)

    def _refined_norms_or_dino(self):
        return self._refined_norms if self._refined_norms is not None else self._dino_norms

    @torch.no_grad()
    def load_dino_embed_video(self):
        """models/tracker.py:64-71: ``dino_embed_video.pt`` holds T x C x h x w fp32."""
        assert os.path.exists(self.dino_embed_path)
        self._set_dino(torch.load(self.dino_embed_path, map_location="cpu"))

    @property
    def dino_embed_video(self):
        return self._chw_view(self._dino_tpc)

    @dino_embed_video.setter
    def dino_embed_video(self, chw):
        self._set_dino(chw)

    @property
    def refined_features(self):
        return None if self._refined_tpc is None else self._chw_view(self._refined_tpc)

    @refined_features.setter
    def refined_features(self, chw):
        if chw is None:
            self._refined_tpc = self._refined_norms = None
        else:
            self._refined_tpc, self._refined_norms = self._pack(chw)

    def get_dino_embed_video(self, frames_set_t):
        return self.dino_embed_video[frames_set_t.to(self._dev).long()]

    def get_refined_embeddings(self, frames_set_t, return_raw_embeddings=False):
        """models/tracker.py:113-129: refined = dino + align(delta_cnn(frames)) for the given frames."""
        idx = frames_set_t.to(self._dev).long()
        raw = self.dino_embed_video[idx]
        if self.delta_dino.wants_graph():     # training: residual with delta-DINO's graph, batches of 8 frames (:118-123)
            frames = _as_f32(self.video[idx.to(self.video.device)], self._dev)
            residual = torch.cat([self.delta_dino(frames[i:i + 8], raw[i:i + 8]) for i in range(0, idx.shape[0], 8)], dim=0)
            refined = raw + residual
        else:
            tpc, _ = self._refined_for(idx)
            refined = self._chw_view(tpc)
            residual = refined - raw
        if return_raw_embeddings:
            return refined, residual, raw
        return refined, residual

    @_lib.on_device
    def _refined_for(self, idx):
        dino = self._dino_tpc[idx].contiguous()
        frames = _as_f32(self.video[idx.to(self.video.device)], self._dev)
        return self.delta_dino.refine_tpc(frames, dino, self._geom)

    @torch.no_grad()
    def cache_refined_embeddings(self, move_dino_to_cpu=False):
        T = self.video.shape[0]
        self._refined_tpc, self._refined_norms = self._refined_for(torch.arange(T, device=self._dev))
        # (move_dino_to_cpu is accepted for API parity; 180 GB of HBM make the paging unnecessary)

    def uncache_refined_embeddings(self, move_dino_to_gpu=False):
        self._refined_tpc = self._refined_norms = None
        torch.cuda.empty_cache()
        gc.collect()

    # ------------------------------------------------------------------ weights
    def save_weights(self, iter):
        torch.save(self.tracker_head.state_dict(), Path(self.ckpt_path) / f"tracker_head_{iter}.pt")
        torch.save(self.delta_dino.state_dict(), Path(self.ckpt_path) / f"delta_dino_{iter}.pt")

    def load_weights(self, iter):
        self.tracker_head.load_state_dict(
            torch.load(os.path.join(self.ckpt_path, f"tracker_head_{iter}.pt"), map_location=self._dev))
        self.delta_dino.load_state_dict(
            torch.load(os.path.join(self.ckpt_path, f"delta_dino_{iter}.pt"), map_location=self._dev))

    def head_weights(self):
        """Normalised refiner weights as the C struct (cached per parameter version)."""
        params = [self.tracker_head.cnn_refiner[0].weight, self.tracker_head.cnn_refiner[0].bias,
                  self.tracker_head.cnn_refiner[2].weight, self.tracker_head.cnn_refiner[2].bias]
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._head_cache[0] != key:
            self._head_cache = (key, self.tracker_head.packed_weights())
        return self._head_cache[1]

    # ------------------------------------------------------------------ sampling
    def normalize_points_for_sampling(self, points):
        """models/tracker.py:77-94 (tensor plumbing kept for API parity; the kernels apply the same affine)."""
        t, c, h, w = self.video.shape
        p, s = self.dino_patch_size, self.stride
        last_h = ((h - p) // s) * s + (p / 2)
        last_w = ((w - p) // s) * s + (p / 2)
        a = torch.tensor([[2 / (last_w - (p / 2)), 2 / (last_h - (p / 2)), 1]]).to(points.device)
        b = torch.tensor([[1 - last_w * 2 / (last_w - (p / 2)), 1 - last_h * 2 / (last_h - (p / 2)), 0]]).to(points.device)
        return a * points + b

    def sample_embeddings(self, embeddings, source_points):
        """models/tracker.py:96-111: embeddings T x C x h x w, source_points B x 3 = (x_n, y_n, t_index)
        with x_n, y_n in [-1, 1].  Returns B x C."""
        if embeddings is not None and torch.is_grad_enabled() and embeddings.requires_grad:
            return _train.sample_points(self, embeddings, source_points)      # contrastive losses, dino_tracker.py:215-220
        if embeddings is not None and self._refined_tpc is not None and \
                embeddings.data_ptr() == self._refined_tpc.data_ptr():
            tpc = self._refined_tpc
        else:
            tpc, _ = self._pack(embeddings)
        T = tpc.shape[0]
        frames_set = torch.arange(T, device=self._dev, dtype=torch.int32)
        desc, _ = self._sample(tpc, source_points, frames_set, normalized=True)
        return desc

    @_lib.on_device
    def _sample(self, tpc, points, frames_set, normalized):
        pts = _as_f32(points, self._dev)
        B = pts.shape[0]
        C = tpc.shape[-1]
        desc = torch.empty(B, C, device=self._dev, dtype=torch.float32)
        dn = torch.empty(B, device=self._dev, dtype=torch.float32)
        fs = frames_set.to(device=self._dev, dtype=torch.int32).contiguous()
        _lib.check(self._lib.dinotrk_sample_descriptors(
            _lib.ptr(tpc), tpc.shape[0], C, ctypes.byref(self._geom), _lib.ptr(pts), B, _lib.ptr(fs), fs.shape[0],
            1 if normalized else 0, _lib.ptr(desc), _lib.ptr(dn), _lib.stream_ptr(self._dev)), "sample_descriptors")
        return desc, dn

    # ------------------------------------------------------------------ forward
    def _features_for_forward(self, frames_set_t, use_raw_features):
        if use_raw_features:
            return self._dino_tpc, self._dino_norms, None
        if self._refined_tpc is not None:
            return self._refined_tpc, self._refined_norms, None
        # no cache (training-style call): refine just the requested frames; indices become set slots
        tpc, norms = self._refined_for(frames_set_t.to(self._dev).long())
        self._local = (tpc, norms)
        return tpc, norms, "local"

    @_lib.on_device
    def forward(self, inp, use_raw_features=False):
        """models/tracker.py:303-325.  inp = (source_points B x 3 px, source_frame_indices B,
        target_frame_indices B, frames_set_t N).  Returns B x 2 in [-1, 1]."""
        src_pts, src_idx, tgt_idx, frames_set_t = inp
        # the reference indexes tensors with these (IndexError when out of range); the kernels would read out of bounds
        fs_host = frames_set_t.detach().to("cpu").long()
        n_set, n_frames = int(fs_host.numel()), int(self._dino_tpc.shape[0])
        if n_set == 0 or int(fs_host.min()) < 0 or int(fs_host.max()) >= n_frames:
            raise IndexError(f"frames_set_t must hold frame indices in [0, {n_frames}), got {fs_host.tolist()}")
        for name, idx in (("source_frame_indices", src_idx), ("target_frame_indices", tgt_idx)):
            ih = idx.detach().to("cpu").long()
            if ih.numel() and (int(ih.min()) < 0 or int(ih.max()) >= n_set):
                raise IndexError(f"{name} must index the frame set (size {n_set})")
        self._local = None
        self._graph = None
        if self._wants_graph(use_raw_features):
            return self._forward_graph(inp, use_raw_features)
        tpc, norms, mode = self._features_for_forward(frames_set_t, use_raw_features)
        self._last_frames = (frames_set_t, use_raw_features)
        B = src_pts.shape[0]
        fs = frames_set_t.to(self._dev).to(torch.int32)
        if mode == "local":
            fs = torch.arange(fs.shape[0], device=self._dev, dtype=torch.int32)
        T, P, C = tpc.shape
        # group the maps by target frame (host side: tiny index vectors)
        tgt_frames = fs[tgt_idx.to(self._dev).long()].cpu()
        order = torch.argsort(tgt_frames, stable=True)
        uniq, counts = torch.unique_consecutive(tgt_frames[order], return_counts=True)
        pts = torch.cat([_as_f32(src_pts, self._dev)[:, :2],
                         src_idx.to(self._dev).to(torch.float32)[:, None]], dim=1)[order.to(self._dev)].contiguous()
        desc, dn = self._sample(tpc, pts, fs, normalized=False)
        row0 = torch.cumsum(counts, 0) - counts
        grp = torch.stack([uniq.to(torch.int32), row0.to(torch.int32), counts.to(torch.int32),
                           row0.to(torch.int32)]).to(self._dev).contiguous()
        out_index = order.to(device=self._dev, dtype=torch.int32).contiguous()
        out = torch.empty(B, 2, device=self._dev, dtype=torch.float32)
        n_groups = int(uniq.shape[0])
        ws_bytes = self._lib.dinotrk_corr_track_workspace_bytes(B, n_groups, C, ctypes.byref(self._geom))
        ws = torch.empty(ws_bytes, device=self._dev, dtype=torch.uint8)
        feat = self.features_struct(tpc, norms)
        _lib.check(self._lib.dinotrk_corr_track(
            ctypes.byref(feat), ctypes.byref(self._geom), ctypes.byref(self.head_weights()),
            _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(grp[0]), _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]),
            n_groups, B, int(counts.max()), _lib.ptr(out_index), _lib.ptr(out), 2, 1,
            _lib.ptr(ws), ws_bytes, _lib.stream_ptr(self._dev)), "corr_track")
        return out

    # ------------------------------------------------------------------ training-step forward (graph)
    def _wants_graph(self, use_raw_features):
        if not torch.is_grad_enabled():
            return False
        if any(p.requires_grad for p in self.tracker_head.parameters()):
            return True
        return not use_raw_features and self._refined_tpc is None and self.delta_dino.wants_graph()

    def _forward_graph(self, inp, use_raw_features):
        """models/tracker.py:303-325 with autograd: same three sources of embeddings, kept (with their graph) as
        ``frame_embeddings`` / ``raw_embeddings`` / ``residual_embeddings`` for the regularisation losses
        (dino_tracker.py:136-146)."""
        frames_set_t = inp[-1]
        idx = frames_set_t.to(self._dev).long()
        residual = None
        if use_raw_features:
            emb = raw = self.dino_embed_video[idx]
        elif self._refined_tpc is not None:
            emb, raw = self.refined_features[idx], self.dino_embed_video[idx]
        else:
            emb, residual, raw = self.get_refined_embeddings(frames_set_t, return_raw_embeddings=True)
        self._graph = (emb, raw, residual)
        self._last_frames = (frames_set_t, use_raw_features)
        return self.get_point_predictions(inp, emb)

    def get_point_predictions(self, inp, frame_embeddings):
        """models/tracker.py:175-180: B x 2 in [-1, 1] from the frame set's embeddings N x C x h x w."""
        return _train.track_points(self, frame_embeddings, inp)

    # ------------------------------------------------------------------ cycle consistency (models/tracker.py:182-301)
    @_lib.on_device
    def _cycle_draw(self, frames_set_t, fg_masks):
        return _cycle.draw(self, frames_set_t, fg_masks, self.frame_embeddings)

    @torch.no_grad()
    def get_cycle_consistent_coords(self, frames_set_t, fg_masks):
        """models/tracker.py:182-262.  ``cyc_n_frames`` random (source, target) slots of the frame set; per pair
        ``cyc_batch_size_per_frame`` pixel positions of the source frame (share ``cyc_fg_points_ratio`` inside
        ``fg_masks``), tracked source -> target -> source with the embeddings of the last forward; kept when they
        return within ``cyc_thresh`` px.  Random draws in the reference's order (two ``randint`` on the frame set's
        device, then per pair a foreground and a background ``randperm``); all pairs tracked as one batch (cycle.py)."""
        out, _ = self._cycle_draw(frames_set_t, fg_masks)
        return out

    def get_cycle_consistent_preds(self, frames_set_t, fg_masks):
        """models/tracker.py:264-301: redraw until at least one point survives the filter, then predict source -> target
        and target -> source WITH the graph (the cycle-consistency loss of dino_tracker.py:346-353 trains on them): the
        survivors' rows of the draw's two legs, as one autograd node."""
        while True:
            cyc, legs = self._cycle_draw(frames_set_t, fg_masks)
            if cyc["source_points"].shape[0] > 0:
                break
        fwd, bwd = _cycle.predictions(self, self.frame_embeddings, legs)
        return {
            "source_coords": self.range_normalizer(cyc["source_points"], dst=[-1, 1]),
            "target_coords": self.range_normalizer(cyc["target_points"], dst=[-1, 1]),
            "source_target_coords": fwd[:, :2],
            "target_source_coords": bwd[:, :2],
            "cycle_consistency_dists": torch.norm(cyc["cycle_points"][:, :2] - cyc["source_points"][:, :2], dim=1),
            "cycle_points": cyc["cycle_points"],
        }

    # the reference stores gathered copies of the frame set on every call (models/tracker.py:322-323);
    # they are materialised lazily here (only training code reads them)
    @property
    def frame_embeddings(self):
        fs, raw = self._last_frames
        if getattr(self, "_graph", None) is not None:
            return self._graph[0]
        if not raw and self._local is not None:   # uncached forward: the refined embeddings of that frame set
            return self._chw_view(self._local[0])
        src = self.dino_embed_video if raw else self.refined_features
        return src[fs.to(self._dev).long()]

    @property
    def residual_embeddings(self):
        """models/tracker.py:319-321: refined - raw of the last forward's frame set."""
        fs, raw = self._last_frames
        if raw:
            return None
        if getattr(self, "_graph", None) is not None and self._graph[2] is not None:
            return self._graph[2]
        return self.frame_embeddings - self.raw_embeddings

    @property
    def raw_embeddings(self):
        fs, _ = self._last_frames
        if getattr(self, "_graph", None) is not None:
            return self._graph[1]
        return self.dino_embed_video[fs.to(self._dev).long()]

"""Host mirror of the reference ``models/model_inference.py`` (SURVEY.md 8b) over libdinotrk.

``ModelInference.infer`` is ONE C call (``dinotrk_infer``): trajectories, cosine similarities, anchor
re-tracking and occlusion all run as grouped device work lists; the reference's two Python hot loops
(``model_inference.py:59-74``, ``:156-165``) and their per-call gathers disappear.  The piecewise
``compute_*`` methods and the module-level ``generate_*`` helpers keep the reference's signatures and
return types.
"""
import ctypes
from typing import Dict

import torch

from . import _lib
from .range_normalizer import RangeNormalizer
from .tracker import Tracker

# maps per correlation/head chunk, clamped to the work of the call.  A map is 4 bytes per token (32 KB at 854x476, 73 KB at
# 1274x714, 128 KB at 32,768 tokens) and two chunks are in flight, so the workspace grows with the grid: about 2 GiB at
# 854x476, 4.8 GiB at 1274x714 and 8 GiB at 1274x1274 for the maps alone.
DEFAULT_CHUNK_MAPS = 32768


# ---- module-level helpers (models/model_inference.py:8-74) -------------------------------------
def generate_trajectory_input(query_point, video, start_t=None, end_t=None):
    """models/model_inference.py:8-34: the (source_points, source_frame_indices, target_frame_indices,
    frames_set_t) tuple that tracks one query point through frames [start_t, end_t)."""
    start_t = 0 if start_t is None else start_t
    end_t = video.shape[0] if end_t is None else end_t
    rest = end_t - start_t
    device = query_point.device
    source_points = query_point[None].repeat(rest, 1)
    frames = torch.arange(start_t, end_t, dtype=torch.long, device=device)
    frames_set_t = torch.cat([query_point[2:3].to(torch.float32), frames.to(torch.float32)]).int()
    source_frame_indices = torch.zeros(rest, dtype=torch.long, device=device)
    target_frame_indices = torch.arange(rest, dtype=torch.long, device=device) + 1
    return source_points, source_frame_indices, target_frame_indices, frames_set_t


@torch.no_grad()
def generate_trajectory(query_point, video, model, range_normalizer, dst_range=(-1, 1), use_raw_features=False,
                        batch_size=None):
    """models/model_inference.py:37-57 -> rest x 3 (x, y, t)."""
    return generate_trajectories(query_point[None], video, model, range_normalizer, dst_range, use_raw_features,
                                 batch_size)[0]


@torch.no_grad()
def generate_trajectories(query_points, video, model, range_normalizer, dst_range=(-1, 1), use_raw_features=False,
                          batch_size=None):
    """models/model_inference.py:59-74 -> N x T x 3.  All query points and frames go through one grouped
    device pass (the frame chunking of ``batch_size`` does not change phase-A results: the query
    descriptor always sits in slot 0 of the frame set)."""
    assert tuple(dst_range) == (-1, 1)
    return _run_phases(model, query_points, 0, 0, batch_size, use_raw_features=use_raw_features)["traj"]


def _run_phases(model: Tracker, query_points, start, stop, batch_size, anchor_th=0.5, cos_th=0.5, traj=None,
                cos_sims=None, anchors=None, use_raw_features=False, chunk_maps=None):
    with torch.cuda.device(model._dev):   # the library launches on the current device
        return _run_phases_on_device(model, query_points, start, stop, batch_size, anchor_th, cos_th, traj, cos_sims,
                                     anchors, use_raw_features, chunk_maps)


def _traj3(traj, T, dev):
    """Trajectories as N x T x 3 (x, y, t).  The reference's occlusion / anchor code only reads [..., :2]
    (models/model_inference.py:137,191), so N x T x 2 -- what ``infer`` returns -- is accepted and completed with t."""
    traj = traj.to(device=dev, dtype=torch.float32)
    if traj.dim() != 3 or traj.shape[1] != T or traj.shape[2] not in (2, 3):
        raise ValueError(f"trajectories must be N x {T} x 2 or N x {T} x 3, got {tuple(traj.shape)}")
    if traj.shape[2] == 2:
        t = torch.arange(T, device=dev, dtype=torch.float32)[None, :, None].expand(traj.shape[0], T, 1)
        traj = torch.cat([traj, t], dim=2)
    return traj.contiguous()


def _run_phases_on_device(model: Tracker, query_points, start, stop, batch_size, anchor_th, cos_th, traj,
                          cos_sims, anchors, use_raw_features, chunk_maps):
    if chunk_maps is None:
        chunk_maps = DEFAULT_CHUNK_MAPS   # module attribute: read at call time (bench.py --chunk-maps sets it)
    chunk_maps = int(min(chunk_maps, max(256, query_points.shape[0] * model.video.shape[0] ** 2)))
    lib = _lib.load()
    dev = model._dev
    if use_raw_features:
        tpc, norms, _ = model._features_for_forward(None, True)
    else:
        assert model._refined_tpc is not None, "call cache_refined_embeddings() first"
        tpc, norms = model._refined_tpc, model._refined_norms
    T, P, C = tpc.shape
    q = query_points.to(device=dev, dtype=torch.float32).contiguous()
    N = q.shape[0]
    geom = model._geom
    if traj is None:
        traj = torch.zeros(N, T, 3, device=dev, dtype=torch.float32)
    else:
        traj = _traj3(traj, T, dev)
    if stop >= 1:
        cos_sims = torch.zeros(N, T, device=dev, dtype=torch.float32) if cos_sims is None else \
            cos_sims.to(device=dev, dtype=torch.float32).contiguous()
    if stop >= 2:
        anchors = torch.zeros(N, T, T, 2, device=dev, dtype=torch.float32) if anchors is None else \
            anchors.to(device=dev, dtype=torch.float32).contiguous()
    occ = torch.zeros(N, T, device=dev, dtype=torch.uint8) if stop >= 3 else None
    ws_bytes = lib.dinotrk_infer_workspace_bytes(T, C, ctypes.byref(geom), N, chunk_maps)
    ws = model.__dict__.get("_infer_ws")
    if ws is None or ws.numel() < ws_bytes:
        ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        model.__dict__["_infer_ws"] = ws
    fb = 0 if batch_size is None else int(batch_size)
    feat = model.features_struct(tpc, norms, quant=True)
    _lib.check(lib.dinotrk_infer(
        ctypes.byref(feat), ctypes.byref(geom), ctypes.byref(model.head_weights()), _lib.ptr(q), N,
        float(anchor_th), float(cos_th), fb, start, stop, chunk_maps, _lib.ptr(traj), _lib.ptr(cos_sims),
        _lib.ptr(anchors), _lib.ptr(occ), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev)), "infer")
    return {"traj": traj, "cos_sims": cos_sims, "anchors": anchors, "occ": occ}


class ModelInference(torch.nn.Module):
    def __init__(self, model: Tracker, range_normalizer: RangeNormalizer,
                 anchor_cosine_similarity_threshold: float = 0.5, cosine_similarity_threshold: float = 0.5) -> None:
        super().__init__()
        self.model = model
        self.model.eval()
        self.model.cache_refined_embeddings()
        self.range_normalizer = range_normalizer
        self.anchor_cosine_similarity_threshold = anchor_cosine_similarity_threshold
        self.cosine_similarity_threshold = cosine_similarity_threshold

    def compute_trajectories(self, query_points: torch.Tensor, batch_size=None) -> torch.Tensor:
        """models/model_inference.py:97-107 -> N x T x 3."""
        return _run_phases(self.model, query_points, 0, 0, batch_size)["traj"]

    def compute_trajectory_cos_sims(self, trajectories, query_points) -> torch.Tensor:
        """models/model_inference.py:110-126 -> N x T."""
        return _run_phases(self.model, query_points, 1, 1, None, traj=trajectories)["cos_sims"]

    def _get_model_preds_at_anchors(self, model, range_normalizer, preds, anchor_indices, batch_size=None):
        """models/model_inference.py:130-154 for ONE query point: ``preds`` T x 3 (its trajectory), ``anchor_indices`` the
        anchor frames -> M x T x 2, the track of every ``preds[i]`` (living in frame i) into every anchor frame.  Same work
        list as the anchor phase of ``infer`` (one device call instead of the reference's M x ceil(T / batch) model() calls)."""
        T = preds.shape[0]
        dev = model._dev
        cos = torch.zeros(1, T, device=dev, dtype=torch.float32)
        idx = torch.as_tensor(anchor_indices, device=dev).long().reshape(-1)
        cos[0, idx] = 1.0
        r = _run_phases(model, torch.zeros(1, 3, device=dev), 2, 2, batch_size, anchor_th=0.5, traj=preds[None], cos_sims=cos)
        return r["anchors"][0][idx]

    def compute_anchor_trajectories(self, trajectories: torch.Tensor, cos_sims: torch.Tensor,
                                    batch_size=None) -> Dict[int, torch.Tensor]:
        """models/model_inference.py:156-165 -> {n: M_n x T x 2} (rows = anchor frames, ascending)."""
        N = trajectories.shape[0]
        q = torch.zeros(N, 3, device=self.model._dev)
        r = _run_phases(self.model, q, 2, 2, batch_size, anchor_th=self.anchor_cosine_similarity_threshold,
                        traj=trajectories, cos_sims=cos_sims)
        vis = r["cos_sims"] >= self.anchor_cosine_similarity_threshold
        return {n: r["anchors"][n][vis[n]] for n in range(N)}

    def compute_occ_pred_for_qp(self, green_trajectories_qp, source_trajectories_qp, traj_cos_sim_qp, anch_sim_th,
                                cos_sim_th):
        """models/model_inference.py:169-177 for one query point (goes through the same device kernel)."""
        T = traj_cos_sim_qp.shape[0]
        dev = self.model._dev
        vis = traj_cos_sim_qp >= anch_sim_th
        anchors = torch.zeros(1, T, T, 2, device=dev)
        anchors[0][vis.to(dev)] = green_trajectories_qp.to(dev)
        traj = torch.zeros(1, T, 3, device=dev)
        traj[0, :, :2] = source_trajectories_qp.to(dev)
        return self._occlusion(traj, traj_cos_sim_qp[None], anchors, anch_sim_th, cos_sim_th)[0]

    def _occlusion(self, traj, cos_sims, anchors, anch_th, cos_th):
        lib = _lib.load()
        dev = self.model._dev
        cos_sims = cos_sims.to(device=dev, dtype=torch.float32).contiguous()
        N, T = cos_sims.shape
        traj = _traj3(traj, T, dev)                     # the kernel reads (x, y, t) triples
        anchors = anchors.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(anchors.shape) != (N, T, T, 2) or traj.shape[0] != N:
            raise ValueError(f"occlusion: anchors must be {N} x {T} x {T} x 2 and trajectories {N} x {T} x 2|3")
        # the reference takes a median over an empty anchor set and raises; say so instead of calling everything visible
        n_anchor = (cos_sims >= anch_th).sum(dim=1)
        if N and int(n_anchor.min()) == 0:
            raise ValueError("occlusion: query point %d has no anchor frame (cos-sim >= %.3f); the reference fails here too"
                             % (int(n_anchor.argmin()), anch_th))
        occ = torch.zeros(N, T, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            _lib.check(lib.dinotrk_occlusion(_lib.ptr(traj), _lib.ptr(cos_sims), _lib.ptr(anchors), N, T, float(anch_th),
                                             float(cos_th), _lib.ptr(occ), _lib.stream_ptr(dev)), "occlusion")
        return occ.bool()

    def compute_occlusion(self, trajectories, trajs_cos_sims, anchor_trajectories: Dict[int, torch.Tensor]):
        """models/model_inference.py:179-200 -> N x T bool."""
        N, T = trajs_cos_sims.shape
        dev = self.model._dev
        vis = (trajs_cos_sims >= self.anchor_cosine_similarity_threshold).to(dev)
        anchors = torch.zeros(N, T, T, 2, device=dev)
        for n in range(N):
            anchors[n][vis[n]] = anchor_trajectories[n].to(dev)
        return self._occlusion(trajectories, trajs_cos_sims, anchors, self.anchor_cosine_similarity_threshold,
                               self.cosine_similarity_threshold)

    @torch.no_grad()
    def infer(self, query_points: torch.Tensor, batch_size=None):
        """models/model_inference.py:203-216 -> (N x T x 2 px, N x T bool)."""
        r = _run_phases(self.model, query_points, 0, 3, batch_size,
                        anchor_th=self.anchor_cosine_similarity_threshold, cos_th=self.cosine_similarity_threshold)
        return r["traj"][..., :2], r["occ"].bool()

    @torch.no_grad()
    def infer_all(self, query_points: torch.Tensor, batch_size=None):
        """Like ``infer`` but also returns the intermediates (trajectories with t, cos-sims, dense anchors)."""
        return _run_phases(self.model, query_points, 0, 3, batch_size,
                           anchor_th=self.anchor_cosine_similarity_threshold,
                           cos_th=self.cosine_similarity_threshold)

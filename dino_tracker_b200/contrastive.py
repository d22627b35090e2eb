"""Best-buddy contrastive losses of the training step (dino_tracker.py:159-344) on libdinotrk.

``BBContrastiveFunction`` is ``get_bb_pairs_contrastive_loss`` for all pairs of one loss in one call
(``dinotrk_bb_contrastive_forward`` / ``_backward``).  The three functions below carry the reference's method signatures
and take the trainer as first argument, so they bind as ``DINOTracker`` methods (``dropin/dino_tracker.py``).  They make
the reference's random draws in the reference's order on the same generators (two ``randint`` on the frame set's device,
the dino-BB loss's redraw loop, per pair a foreground then a background ``randperm`` on the host), so a seeded run picks
the same points.  The GPU work of all pairs is launched before the one host read-back the draws need.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import _lib
from .best_buddies import nearest_neighbours


def _host_ptr(t):
    return ctypes.c_void_p(t.data_ptr())


class BBContrastiveFunction(torch.autograd.Function):
    """(E, S [B][C], U [B][C], groups, tau) -> (cl1 [B], cl2 [B], bb_mean [G], c_mean [G]).  E is the frame set, either
    as the ``frame_embeddings`` tensor N x C x h x w (made token-major inside, its gradient returned in the same layout) or
    token-major N x P x C.

    ``groups``: host int32 [4][G] = (source slot, target slot, first row, rows) per pair.  cl1 / cl2 and the means are the
    four return values of ``get_bb_pairs_contrastive_loss`` per pair (rows of no group give 0).  Gradients reach E, S, U."""

    @staticmethod
    def forward(ctx, E, S, U, groups, tau):
        lib = _lib.load()
        ctx.chw = tuple(E.shape) if E.dim() == 4 else None
        if ctx.chw:
            E = E.detach().reshape(E.shape[0], E.shape[1], -1).transpose(1, 2)
        N, P, C = E.shape
        B = S.shape[0]
        G = groups.shape[1]
        dev = E.device
        E_, S_, U_ = (t.detach().float().contiguous() for t in (E, S, U))
        with torch.cuda.device(dev):
            ld = lib.dinotrk_bb_contrastive_cos_stride(P)
            cosm = torch.empty(2 * B, ld, device=dev)
            out = torch.zeros(7, B, device=dev)
            nb = lib.dinotrk_bb_contrastive_forward_workspace_bytes(N, P, C, B, G)
            ws = torch.empty(nb, device=dev, dtype=torch.uint8)
            _lib.check(lib.dinotrk_bb_contrastive_forward(
                _lib.ptr(E_), N, P, C, _lib.ptr(S_), _lib.ptr(U_), B, *(_host_ptr(groups[i]) for i in range(4)), G,
                float(tau), _lib.ptr(cosm), _lib.ptr(out), _lib.ptr(ws), nb, _lib.stream_ptr()), "bb_contrastive_forward")
        bb_mean = torch.stack([out[0, r0:r0 + n].mean() for r0, n in groups[2:].t().tolist()]) if G else out.new_zeros(0)
        c_mean = torch.stack([(out[5, r0:r0 + n].sum() + out[6, r0:r0 + n].sum()) / (2 * n * P)
                              for r0, n in groups[2:].t().tolist()]) if G else out.new_zeros(0)
        ctx.save_for_backward(E_, S_, U_, cosm, out)
        ctx.groups, ctx.tau = groups, float(tau)
        return out[3].clone(), out[4].clone(), bb_mean, c_mean

    @staticmethod
    def backward(ctx, g1, g2, gbb, gcm):
        lib = _lib.load()
        E, S, U, cosm, out = ctx.saved_tensors
        groups = ctx.groups
        N, P, C = E.shape
        B = S.shape[0]
        G = groups.shape[1]
        dev = E.device

        def grad_or_zero(g, n):
            return torch.zeros(n, device=dev) if g is None else g.detach().float().contiguous()
        g1, g2, gbb, gcm = grad_or_zero(g1, B), grad_or_zero(g2, B), grad_or_zero(gbb, G), grad_or_zero(gcm, G)
        with torch.cuda.device(dev):
            dS = torch.empty(B, C, device=dev)
            dU = torch.empty(B, C, device=dev)
            dE = torch.zeros(N, P, C, device=dev)
            gp = [_host_ptr(groups[i]) for i in range(4)]
            nb = lib.dinotrk_bb_contrastive_backward_workspace_bytes(N, P, C, B, *gp, G)
            ws = torch.empty(nb, device=dev, dtype=torch.uint8)
            _lib.check(lib.dinotrk_bb_contrastive_backward(
                _lib.ptr(E), N, P, C, _lib.ptr(S), _lib.ptr(U), B, *gp, G, ctx.tau, _lib.ptr(cosm), _lib.ptr(out),
                _lib.ptr(g1), _lib.ptr(g2), _lib.ptr(gbb), _lib.ptr(gcm), _lib.ptr(dS), _lib.ptr(dU), _lib.ptr(dE),
                _lib.ptr(ws), nb, _lib.stream_ptr()), "bb_contrastive_backward")
        if ctx.chw:
            dE = dE.transpose(1, 2).reshape(ctx.chw)
        return dE, dS, dU, None, None


def bb_contrastive(E, S, U, groups, tau):
    """BBContrastiveFunction.apply with ``groups`` as a list of (source slot, target slot, first row, rows)."""
    g = torch.tensor(groups, dtype=torch.int32).reshape(-1, 4).t().contiguous()
    return BBContrastiveFunction.apply(E, S, U, g, tau)


def _token_rows(frame_embeddings):
    """N x C x h x w -> a token-major VIEW N x P x C (rows are gathered from it without a copy of the frame set)."""
    N, C = frame_embeddings.shape[:2]
    return frame_embeddings.reshape(N, C, -1).transpose(1, 2)


def vit_feature_coords(h, w, step=7, patch_size=14, device="cpu"):
    """models/utils.py:87-95 (get_vit_feature_coords_from_mask): pixel (x, y) of every token, row-major."""
    half = patch_size // 2
    x = torch.arange(half, w - half + 1, step=step, device=device).float()
    y = torch.arange(half, h - half + 1, step=step, device=device).float()
    yy, xx = torch.meshgrid(y, x, indexing="ij")
    return torch.stack([xx.reshape(-1), yy.reshape(-1)], dim=-1)


def foreground(coords, fg_mask, resw, resh):
    """models/utils.py:53-58 (filter_bb_foreground_pairs): bilinear grid_sample of the mask at the points, > 0."""
    scale = torch.tensor([resw, resh], device=coords.device, dtype=coords.dtype)
    v = F.grid_sample(fg_mask[None, None].float(), 2 * (coords[None, None] / scale) - 1)
    return v.reshape(-1) > 0


def _sampled(n_fg_all, n_bg_all, n_fg, n_bg):
    """The reference's per-pair draws: a foreground then a background randperm on the host."""
    return torch.randperm(n_fg_all)[:n_fg], torch.randperm(n_bg_all)[:n_bg]


def get_bb_pairs_contrastive_loss(self, source_bb_f, target_bb_f, source_f, target_f, temp=0.5):
    """dino_tracker.py:332-344 for one pair (source_f / target_f: n x c token rows)."""
    E = torch.stack([source_f, target_f])
    b = source_bb_f.shape[0]
    cl1, cl2, bbm, cm = bb_contrastive(E, source_bb_f, target_bb_f, [(0, 1, 0, b)], temp)
    return cl1, cl2, bbm[0], cm[0]


def draw_dino_bb_pairs(self, model, frames_set_t):
    """The draws of dino_tracker.py:160-207: [(source slot, target slot, selected best-buddy indices (host), pair dict)]
    for the pairs that contribute, or [] (no pair contributes)."""
    cfg = self.config
    batch_size = cfg["cl_n_frames"]
    n_set = frames_set_t.shape[0]
    source_selector = torch.randint(n_set, (batch_size,), device=frames_set_t.device)
    target_selector = torch.randint(n_set, (batch_size,), device=frames_set_t.device)
    while (source_selector == target_selector).any():
        target_selector = torch.randint(n_set, (batch_size,), device=frames_set_t.device)
    n_fg = int(cfg["cl_points_per_pair"] * cfg["cl_fg_points_ratio"])
    n_bg = cfg["cl_points_per_pair"] - n_fg
    dev = model.frame_embeddings.device
    H, W = model.video.shape[-2], model.video.shape[-1]
    frames = frames_set_t.tolist()
    pairs, flags = [], []
    for s, t in zip(source_selector.tolist(), target_selector.tolist()):
        if s == t:
            continue
        bb = self.dino_bb_pairs[f"{frames[s]}_{frames[t]}"]
        if bb["source_coords"] is None or bb["source_coords"].shape[0] == 0:
            continue
        pairs.append((s, t, bb))
        flags.append(foreground(bb["source_coords"].to(dev).float(), self.fg_masks[frames[s]].to(dev), W, H))
    if not pairs:
        return []
    flags = torch.cat(flags).cpu()                                     # the one read-back for the draws
    out, i0 = [], 0
    for s, t, bb in pairs:
        n = bb["source_coords"].shape[0]
        fg = flags[i0:i0 + n]
        i0 += n
        idx = torch.arange(n)
        fg_idx, bg_idx = idx[fg], idx[~fg]
        fg_sel, bg_sel = _sampled(fg_idx.shape[0], bg_idx.shape[0], n_fg, n_bg)
        sel = torch.cat([fg_idx[fg_sel], bg_idx[bg_sel]])
        if sel.shape[0]:
            out.append((s, t, sel, bb))
    return out


def get_dino_bb_contrastive_loss(self, model, frames_set_t):
    """dino_tracker.py:159-243."""
    cfg = self.config
    drawn = draw_dino_bb_pairs(self, model, frames_set_t)
    if not drawn:
        return torch.tensor(0.).to(frames_set_t.device)
    emb = model.frame_embeddings
    dev = emb.device
    src_pts, tgt_pts, groups, ws = [], [], [], []
    row = 0
    for s, t, sel, bb in drawn:
        sel_d = sel.to(bb["source_coords"].device)
        for pts, key, slot in ((src_pts, "source_coords", s), (tgt_pts, "target_coords", t)):
            c = bb[key][sel_d].to(dev).float()
            pts.append(torch.cat([c, torch.full((c.shape[0], 1), float(slot), device=dev)], dim=1))
        groups.append((s, t, row, sel.shape[0]))
        row += sel.shape[0]
        w = torch.sigmoid(cfg["bb_amb_sig_a"] * (1 - bb["r"][sel_d]) + cfg["bb_amb_sig_b"])
        ws.append((w * torch.clamp(2 * (bb["cos_sims"][sel_d] ** 3), 0)).to(dev))
    S = model.sample_embeddings(emb, model.normalize_points_for_sampling(torch.cat(src_pts)))
    U = model.sample_embeddings(emb, model.normalize_points_for_sampling(torch.cat(tgt_pts)))
    cl1, cl2, _, _ = bb_contrastive(emb, S, U, groups, cfg["cl_temp"])
    w = torch.cat(ws)
    cl_div = cfg["cl_div_dino_bb"]
    return ((cl1 * w / cl_div).sum() + (cl2 * w / cl_div).sum()) / 2


@torch.no_grad()
def refined_best_buddies(frame_embeddings, pairs, H, W, patch_size=14, stride=7):
    """In-training best-buddy search (dino_tracker.py:263-284) for the slot pairs ``pairs`` of a frame set N x C x h x w
    (self-pairs allowed): per pair the mutual mask [P], the partner token [P] and the exact-fp32 cosine at the pair [P]."""
    lib = _lib.load()
    N, C, h, w = frame_embeddings.shape
    P = h * w
    dev = frame_embeddings.device
    geom = _lib.make_geom((h - 1) * stride + patch_size, (w - 1) * stride + patch_size, patch_size, stride, 35)
    with torch.cuda.device(dev):
        chw = frame_embeddings.detach().float().contiguous()
        tpc = torch.empty(N, P, C, device=dev)
        norms = torch.empty(N, P, device=dev)
        _lib.check(lib.dinotrk_pack_features(_lib.ptr(chw), _lib.ptr(tpc), _lib.ptr(norms), N, C, P, _lib.stream_ptr()))
        ordered = [p for (s, t) in pairs for p in ((s, t), (t, s))]
        nn_idx, nn_cos = nearest_neighbours(tpc, norms, geom, ordered)
        n = len(pairs)
        st = nn_idx.view(n, 2, P)[:, 0].contiguous()
        ts = nn_idx.view(n, 2, P)[:, 1].contiguous()
        mutual = torch.empty(n, P, device=dev, dtype=torch.uint8)
        _lib.check(lib.dinotrk_bb_mutual(_lib.ptr(st), _lib.ptr(ts), n, P, _lib.ptr(mutual), _lib.stream_ptr()))
    return mutual.bool(), st.long(), nn_cos.view(n, 2, P)[:, 0]


def draw_refined_pairs(self, model, frames_set_t, frame_embeddings, batch_size, points_per_pair, fg_points_ratio=0.5):
    """The search and draws of dino_tracker.py:246-310: [(source slot, target slot, source tokens, target tokens, cosine at
    the pairs)] (device tensors) for the pairs with a non-empty selection."""
    n_set = frames_set_t.shape[0]
    source_selector = torch.randint(n_set, (batch_size,), device=frames_set_t.device)
    target_selector = torch.randint(n_set, (batch_size,), device=frames_set_t.device)
    H, W = model.video.shape[-2], model.video.shape[-1]
    patch = self.config["dino_patch_size"]
    dev = frame_embeddings.device
    coords = vit_feature_coords(H, W, step=model.stride, patch_size=patch, device=dev)
    n_fg = int(points_per_pair * fg_points_ratio)
    n_bg = points_per_pair - n_fg
    pairs = list(zip(source_selector.tolist(), target_selector.tolist()))
    frames = frames_set_t.tolist()
    mutual, partner, cos_at = refined_best_buddies(frame_embeddings, pairs, H, W, patch, model.stride)
    fg_tok = torch.stack([foreground(coords, self.fg_masks[frames[s]].to(dev), W, H) for s, _ in pairs])
    host = torch.stack([mutual, fg_tok]).cpu()                          # the one read-back for the draws
    out = []
    for k, (s, t) in enumerate(pairs):
        m = host[0, k]
        if not bool(m.any()):
            continue
        toks = torch.nonzero(m).reshape(-1)
        fg = host[1, k][toks]
        fg_sel, bg_sel = _sampled(int(fg.sum()), int((~fg).sum()), n_fg, n_bg)
        sel = torch.cat([toks[fg][fg_sel], toks[~fg][bg_sel]]).to(dev)
        if sel.shape[0]:
            out.append((s, t, sel, partner[k][sel], cos_at[k][sel]))
    return out


def get_refined_bb_contrastive_loss(self, model, frames_set_t, frame_embeddings, batch_size, points_per_pair,
                                    fg_points_ratio=0.5, temp=0.5, cl_div=800):
    """dino_tracker.py:245-330."""
    drawn = draw_refined_pairs(self, model, frames_set_t, frame_embeddings, batch_size, points_per_pair, fg_points_ratio)
    if not drawn:
        return torch.tensor(0.).to(frame_embeddings.device)
    rows = _token_rows(frame_embeddings)
    groups, src, tgt, row = [], [], [], 0
    for s, t, ss, ts, _ in drawn:
        groups.append((s, t, row, ss.shape[0]))
        row += ss.shape[0]
        src.append((torch.full_like(ss, s), ss))
        tgt.append((torch.full_like(ts, t), ts))
    S = rows[torch.cat([a for a, _ in src]), torch.cat([b for _, b in src])]
    U = rows[torch.cat([a for a, _ in tgt]), torch.cat([b for _, b in tgt])]
    cl1, cl2, _, _ = bb_contrastive(frame_embeddings, S, U, groups, temp)
    w = torch.clamp(2 * (torch.cat([c for *_, c in drawn]) ** 3), 0)
    return ((cl1 * w).sum() + (cl2 * w).sum()) / (2 * cl_div)

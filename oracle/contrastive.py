"""Plain-torch restatement of the best-buddy contrastive losses of the training step.

``dino_tracker.py:159-243`` (get_dino_bb_contrastive_loss), ``:245-330`` (get_refined_bb_contrastive_loss) and
``:332-344`` (get_bb_pairs_contrastive_loss), with the helpers ``models/utils.py:53-58`` (filter_bb_foreground_pairs) and
``:87-95`` (get_vit_feature_coords_from_mask).  Device-agnostic (no ``.cuda()``), and the arithmetic runs in the dtype
of the embeddings, so float64 runs on the GPU.  The random draws are the reference's, in its order, on the same
generators.  ``record`` (a list, optional) receives per contributing pair (source slot, target slot, selected source
index, selected target index): best-buddy indices for the dino-BB loss, token indices for the refined loss.

``ModelStandIn`` is the part of the tracker these losses touch (``video``, ``stride``, ``frame_embeddings``,
``normalize_points_for_sampling`` = models/tracker.py:77-94, ``sample_embeddings`` = :96-111).
"""
import torch
import torch.nn.functional as F

from .tracker import sample_descriptors


class ModelStandIn:
    def __init__(self, video, frame_embeddings, stride=7, dino_patch_size=14):
        self.video = video
        self.frame_embeddings = frame_embeddings
        self.stride = stride
        self.dino_patch_size = dino_patch_size

    def normalize_points_for_sampling(self, points):
        h, w = self.video.shape[-2], self.video.shape[-1]
        p, s = self.dino_patch_size, self.stride
        last_h = ((h - p) // s) * s + (p / 2)
        last_w = ((w - p) // s) * s + (p / 2)
        a = torch.tensor([[2 / (last_w - (p / 2)), 2 / (last_h - (p / 2)), 1]]).to(points.device)
        b = torch.tensor([[1 - last_w * 2 / (last_w - (p / 2)), 1 - last_h * 2 / (last_h - (p / 2)), 0]]).to(points.device)
        return a * points + b

    def sample_embeddings(self, embeddings, source_points):
        return sample_descriptors(embeddings, source_points)


def get_vit_feature_coords_from_mask(h, w, step=7, patch_size=14, device="cpu"):
    half_ps = patch_size // 2
    x = torch.arange(half_ps, w - half_ps + 1, step=step, device=device).float()
    y = torch.arange(half_ps, h - half_ps + 1, step=step, device=device).float()
    yy, xx = torch.meshgrid(y, x, indexing="ij")
    return torch.stack([xx.reshape(-1), yy.reshape(-1)], dim=-1)


def filter_bb_foreground_pairs(source_coords, target_coords, fg_mask, resw=854, resh=476):
    scale = torch.tensor([resw, resh], device=source_coords.device)
    fg = F.grid_sample(fg_mask[None, None, ...].float(), 2 * (source_coords[None, None, ...].float() / scale) - 1).squeeze()
    fg = fg > 0
    if len(fg.shape) < 1:
        fg = fg.unsqueeze(0)
    return source_coords[fg], target_coords[fg], fg


def get_bb_pairs_contrastive_loss(self, source_bb_f, target_bb_f, source_f, target_f, temp=0.5):
    bb_corrs = torch.einsum("bc,bc->b", source_bb_f, target_bb_f)
    st = torch.einsum("bc,nc->bn", source_bb_f, target_f)
    ts = torch.einsum("bc,nc->bn", target_bb_f, source_f)
    st = st / torch.clamp(source_bb_f.norm(dim=1)[:, None] * target_f.norm(dim=1)[None, ...], min=1e-08)
    ts = ts / torch.clamp(target_bb_f.norm(dim=1)[:, None] * source_f.norm(dim=1)[None, ...], min=1e-08)
    bb_corrs = bb_corrs / torch.clamp(source_bb_f.norm(dim=1) * target_bb_f.norm(dim=1), min=1e-08)
    loss_st = -torch.log(torch.exp(bb_corrs / temp) / torch.exp(st / temp).sum(dim=1))
    loss_ts = -torch.log(torch.exp(bb_corrs / temp) / torch.exp(ts / temp).sum(dim=1))
    return loss_st, loss_ts, bb_corrs.mean(), (st.mean() + ts.mean()) / 2


def _tokens(x):
    return x.reshape(x.shape[0], -1).t()   # c h w -> (h w) c


def get_dino_bb_contrastive_loss(self, model, frames_set_t, record=None):
    cfg = self.config
    batch_size = cfg["cl_n_frames"]
    dev = frames_set_t.device
    source_selector = torch.randint(frames_set_t.shape[0], (batch_size,), device=dev)
    target_selector = torch.randint(frames_set_t.shape[0], (batch_size,), device=dev)
    while (source_selector == target_selector).any():
        target_selector = torch.randint(frames_set_t.shape[0], (batch_size,), device=dev)
    n_fg = int(cfg["cl_points_per_pair"] * cfg["cl_fg_points_ratio"])
    n_bg = cfg["cl_points_per_pair"] - n_fg
    emb = model.frame_embeddings
    n_total_bb = 0
    loss_cl1, loss_cl2, l_ws, l_cos_ws = [], [], [], []
    for s, t in zip(source_selector, target_selector):
        if s == t:
            continue
        source_frame, target_frame = frames_set_t[s], frames_set_t[t]
        bb = self.dino_bb_pairs[f"{int(source_frame)}_{int(target_frame)}"]
        if bb["source_coords"] is None or bb["source_coords"].shape[0] == 0:
            continue
        bdev = bb["source_coords"].device
        _, _, fg = filter_bb_foreground_pairs(bb["source_coords"], bb["target_coords"], self.fg_masks[int(source_frame)].to(bdev),
                                              resw=model.video.shape[-1], resh=model.video.shape[-2])
        n = bb["source_coords"].shape[0]
        fg_indices = torch.arange(n, device=bdev)[fg]
        bg_indices = torch.arange(n, device=bdev)[~fg]
        fg_selector = torch.randperm(fg_indices.shape[0])[:n_fg]
        bg_selector = torch.randperm(bg_indices.shape[0])[:n_bg]
        selector = torch.cat([fg_indices[fg_selector.to(bdev)], bg_indices[bg_selector.to(bdev)]])
        if selector.shape[0] == 0:
            continue
        ed = emb.device

        def with_slot(c, slot):
            c = c.to(ed).float()
            return torch.cat([c, torch.full((c.shape[0], 1), float(slot), device=ed)], dim=1)
        src = with_slot(bb["source_coords"][selector], s)
        tgt = with_slot(bb["target_coords"][selector], t)
        sf = model.sample_embeddings(emb, model.normalize_points_for_sampling(src))
        tf = model.sample_embeddings(emb, model.normalize_points_for_sampling(tgt))
        cl1, cl2, _, _ = get_bb_pairs_contrastive_loss(self, sf, tf, _tokens(emb[s]), _tokens(emb[t]), temp=cfg["cl_temp"])
        n_total_bb += 2 * cl1.shape[0]
        loss_cl1.append(cl1)
        loss_cl2.append(cl2)
        ws = torch.sigmoid(cfg["bb_amb_sig_a"] * (1 - bb["r"][selector]) + cfg["bb_amb_sig_b"])
        l_ws.append(ws.to(ed, emb.dtype))
        l_cos_ws.append(torch.clamp(2 * (bb["cos_sims"][selector] ** 3), 0).to(ed, emb.dtype))
        if record is not None:
            record.append((int(s), int(t), selector.cpu(), selector.cpu()))
    if n_total_bb == 0:
        return torch.tensor(0.).to(dev)
    w = torch.cat(l_ws) * torch.cat(l_cos_ws)
    cl_div = cfg["cl_div_dino_bb"]
    return ((torch.cat(loss_cl1) * w / cl_div).sum() + (torch.cat(loss_cl2) * w / cl_div).sum()) / 2


def refined_best_buddies(source_f, target_f):
    """dino_tracker.py:263-284 on token rows: (source mask of mutual nearest neighbours [n], partner [n], affinity [n][m])."""
    affinity = torch.einsum("nc,mc->nm", source_f, target_f)
    affinity = affinity / torch.clamp(source_f.norm(dim=1)[:, None] * target_f.norm(dim=1)[None, ...], min=1e-08)
    amax_s = torch.argmax(affinity, dim=1)
    amax_t = torch.argmax(affinity, dim=0)
    mutual = torch.arange(source_f.shape[0], device=source_f.device) == amax_t[amax_s]
    return mutual, amax_s, affinity


def get_refined_bb_contrastive_loss(self, model, frames_set_t, frame_embeddings, batch_size, points_per_pair,
                                    fg_points_ratio=0.5, temp=0.5, cl_div=800, record=None, search=None):
    """``search`` (optional): (source slot, target slot) -> (mutual [P] bool, partner [P]) replacing the search's own
    arg-max, for comparisons at near-ties; the loss weights still read this dtype's affinity."""
    source_selector = torch.randint(frames_set_t.shape[0], (batch_size,), device=frames_set_t.device)
    target_selector = torch.randint(frames_set_t.shape[0], (batch_size,), device=frames_set_t.device)
    coords = get_vit_feature_coords_from_mask(h=model.video.shape[-2], w=model.video.shape[-1], step=model.stride,
                                              patch_size=self.config["dino_patch_size"]).to(frame_embeddings.device)
    n_fg = int(points_per_pair * fg_points_ratio)
    n_bg = points_per_pair - n_fg
    n_total_bb = 0
    loss = 0
    for s, t in zip(source_selector, target_selector):
        source_f, target_f = _tokens(frame_embeddings[s]), _tokens(frame_embeddings[t])
        with torch.no_grad():
            mutual, partner, affinity = refined_best_buddies(source_f, target_f)
            if search is not None:
                mutual, partner = search(int(s), int(t))
            target_idx = partner[mutual]
            if mutual.sum() == 0:
                continue
        _, _, fg = filter_bb_foreground_pairs(coords[mutual], coords[target_idx], self.fg_masks[int(frames_set_t[s])].to(coords.device),
                                              resw=model.video.shape[-1], resh=model.video.shape[-2])
        src_num = torch.arange(mutual.shape[0], device=mutual.device)[mutual]
        fg_selector = torch.randperm(int(fg.sum()))[:n_fg]
        bg_selector = torch.randperm(int((~fg).sum()))[:n_bg]
        src_sel = torch.cat([src_num[fg][fg_selector.to(mutual.device)], src_num[~fg][bg_selector.to(mutual.device)]])
        tgt_sel = torch.cat([target_idx[fg][fg_selector.to(mutual.device)], target_idx[~fg][bg_selector.to(mutual.device)]])
        cl1, cl2, _, _ = get_bb_pairs_contrastive_loss(self, source_f[src_sel], target_f[tgt_sel], source_f, target_f, temp=temp)
        with torch.no_grad():
            w = torch.clamp(2 * (affinity[src_sel, tgt_sel] ** 3), 0)
        n_total_bb += 2 * cl1.shape[0]
        loss = loss + (cl1 * w).sum() + (cl2 * w).sum()
        if record is not None:
            record.append((int(s), int(t), src_sel.cpu(), tgt_sel.cpu()))
    if n_total_bb == 0:
        return torch.tensor(0.).to(frame_embeddings.device)
    return loss / (2 * cl_div)

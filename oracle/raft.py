"""Device-agnostic plain-torch restatement of torchvision's ``raft_large`` forward pass (eval mode) with the library's
structure (dino_tracker_b200/csrc/raft.cu): each frame encoded once, the update loop on a batch of pairs (i, j), the
mask predictor and the convex upsampling after the last update only.  Runs in the dtype of the given state_dict's
tensors (float64 for the CPU check against torchvision)."""
import torch
import torch.nn.functional as F


def _conv(sd, key, x, stride=1, padding=None):
    w, b = sd[key + ".weight"], sd[key + ".bias"]
    kh, kw = w.shape[-2:]
    pad = (kh // 2, kw // 2) if padding is None else padding
    return F.conv2d(x, w, b, stride=stride, padding=pad)


def _norm(sd, key, x, inorm):
    if inorm:
        return F.instance_norm(x, eps=1e-5)
    return F.batch_norm(x, sd[key + ".running_mean"], sd[key + ".running_var"], sd[key + ".weight"], sd[key + ".bias"],
                        False, 0.0, 1e-5)


def _cnr(sd, key, x, inorm, stride=1, relu=True):
    y = _norm(sd, key + ".1", _conv(sd, key + ".0", x, stride), inorm)
    return F.relu(y) if relu else y


def encoder(sd, prefix, x, inorm):
    """FeatureEncoder (layers 64, 64, 96, 128, 256; strides 2, 1, 2, 2) of frames x [N][3][H][W] in [-1, 1]."""
    x = _cnr(sd, prefix + "convnormrelu", x, inorm, stride=2)
    for layer, stride in (("layer1", 1), ("layer2", 2), ("layer3", 2)):
        for blk in range(2):
            k = f"{prefix}{layer}.{blk}"
            s = stride if blk == 0 else 1
            y = _cnr(sd, k + ".convnormrelu1", x, inorm, stride=s)
            y = _cnr(sd, k + ".convnormrelu2", y, inorm)
            if s != 1:
                x = _cnr(sd, k + ".downsample", x, inorm, stride=s, relu=False)
            x = F.relu(x + y)
    return _conv(sd, prefix + "conv", x)


def encode(sd, frames01):
    """frames [T][3][H][W] in [0, 1], H and W multiples of 8 -> (fmap [T][256][h][w], hidden [T][128][h][w],
    context [T][128][h][w])."""
    x = (frames01 - 0.5) / 0.5
    fmap = encoder(sd, "feature_encoder.", x, True)
    c = encoder(sd, "context_encoder.", x, False)
    return fmap, torch.tanh(c[:, :128]), F.relu(c[:, 128:])


def pyramid(fmap, pairs):
    """Correlation pyramid of each pair: 4 levels [P * h * w][1][h_l][w_l]."""
    i = torch.tensor([p[0] for p in pairs], device=fmap.device)
    j = torch.tensor([p[1] for p in pairs], device=fmap.device)
    P, C, h, w = len(pairs), fmap.shape[1], fmap.shape[2], fmap.shape[3]
    a, b = fmap[i].reshape(P, C, h * w), fmap[j].reshape(P, C, h * w)
    corr = (a.transpose(1, 2) @ b / 16.0).reshape(P * h * w, 1, h, w)
    levels = [corr]
    for _ in range(3):
        levels.append(F.avg_pool2d(levels[-1], 2, stride=2))
    return levels


def lookup(levels, coords, radius=4):
    """Correlation features [P][324][h][w] at coords [P][2][h][w]: channel l * 81 + i * 9 + j samples level l at
    (x / 2^l + i - radius, y / 2^l + j - radius), bilinear, align_corners=True, zeros outside."""
    P, _, h, w = coords.shape
    d = torch.arange(-radius, radius + 1, dtype=coords.dtype, device=coords.device)
    di, dj = torch.meshgrid(d, d, indexing="ij")
    c = coords.permute(0, 2, 3, 1).reshape(P * h * w, 1, 1, 2)
    out = []
    for lv in levels:
        hl, wl = lv.shape[-2:]
        x = c[..., :1] + di[None, :, :, None]
        y = c[..., 1:] + dj[None, :, :, None]
        grid = torch.cat([2 * x / (wl - 1) - 1, 2 * y / (hl - 1) - 1], dim=-1)
        out.append(F.grid_sample(lv, grid, mode="bilinear", padding_mode="zeros", align_corners=True).view(P, h, w, -1))
        c = c / 2
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2)


def _gru(sd, key, h, x, pad):
    hx = torch.cat([h, x], dim=1)
    z = torch.sigmoid(_conv(sd, key + ".convz", hx, padding=pad))
    r = torch.sigmoid(_conv(sd, key + ".convr", hx, padding=pad))
    q = torch.tanh(_conv(sd, key + ".convq", torch.cat([r * h, x], dim=1), padding=pad))
    return (1 - z) * h + z * q


def flows(sd, enc, pairs, num_flow_updates):
    """Full-resolution flows [P][2][8h][8w] of the pairs (i, j) of an encoding (fmap, hidden, context)."""
    fmap, hidden, context = enc
    i = torch.tensor([p[0] for p in pairs], device=fmap.device)
    levels = pyramid(fmap, pairs)
    h, ctx = hidden[i], context[i]
    P, _, hh, ww = h.shape
    ys, xs = torch.meshgrid(torch.arange(hh, device=fmap.device), torch.arange(ww, device=fmap.device), indexing="ij")
    coords0 = torch.stack([xs, ys]).to(fmap.dtype)[None].expand(P, -1, -1, -1)
    coords1 = coords0.clone()
    me = "update_block.motion_encoder."
    for _ in range(num_flow_updates):
        corr = lookup(levels, coords1)
        flow = coords1 - coords0
        c = F.relu(_conv(sd, me + "convcorr1.0", corr))
        c = F.relu(_conv(sd, me + "convcorr2.0", c))
        f = F.relu(_conv(sd, me + "convflow1.0", flow))
        f = F.relu(_conv(sd, me + "convflow2.0", f))
        m = F.relu(_conv(sd, me + "conv.0", torch.cat([c, f], dim=1)))
        x = torch.cat([ctx, m, flow], dim=1)
        h = _gru(sd, "update_block.recurrent_block.convgru1", h, x, (0, 2))
        h = _gru(sd, "update_block.recurrent_block.convgru2", h, x, (2, 0))
        delta = _conv(sd, "update_block.flow_head.conv2", F.relu(_conv(sd, "update_block.flow_head.conv1", h)))
        coords1 = coords1 + delta
    mask = 0.25 * _conv(sd, "mask_predictor.conv", F.relu(_conv(sd, "mask_predictor.convrelu.0", h)))
    mask = torch.softmax(mask.view(P, 1, 9, 8, 8, hh, ww), dim=2)
    up = F.unfold(8 * (coords1 - coords0), kernel_size=3, padding=1).view(P, 2, 9, 1, 1, hh, ww)
    return torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3).reshape(P, 2, 8 * hh, 8 * ww)


def torchvision_flow(model, a01, b01, num_flow_updates):
    """torchvision's ``model((a - 0.5) / 0.5, (b - 0.5) / 0.5, n)[-1]`` in the frames' dtype: its coordinate grids are
    made in float32, so for float64 they are made in float64 (the only change)."""
    from torchvision.models.optical_flow import raft as tvr
    make = tvr.make_coords_grid
    tvr.make_coords_grid = lambda *a, **k: make(*a, **k).to(a01.dtype)
    try:
        with torch.no_grad():
            return model((a01 - 0.5) / 0.5, (b01 - 0.5) / 0.5, num_flow_updates=num_flow_updates)[-1]
    finally:
        tvr.make_coords_grid = make


def seeded_model(seed=0, flow_gain=8.0):
    """raft_large with seeded init, random eval BatchNorm statistics and the flow head scaled so that the flows move by
    several pixels."""
    from torchvision.models.optical_flow import raft_large
    torch.manual_seed(seed)
    m = raft_large(weights=None, progress=False).eval()
    with torch.no_grad():
        for mod in m.context_encoder.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.uniform_(-0.2, 0.2)
                mod.running_var.uniform_(0.5, 2.0)
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)
        m.update_block.flow_head.conv2.weight.mul_(flow_gain)
    return m


def textured_pair(H, W, shift=(2.5, -1.5), seed=0):
    """A smooth random texture a [1][3][H][W] in [0, 1] and b = a moved by ``shift`` px (bilinear)."""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, H // 4 + 3, W // 4 + 3, generator=g), size=(H + 16, W + 16), mode="bicubic",
                         align_corners=False).clamp(0, 1)
    a = base[..., 8:8 + H, 8:8 + W]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    grid = torch.stack([(xs + 8 + shift[0]) / (W + 15) * 2 - 1, (ys + 8 + shift[1]) / (H + 15) * 2 - 1], -1)[None]
    b = F.grid_sample(base, grid, align_corners=True, padding_mode="border")
    return a, b

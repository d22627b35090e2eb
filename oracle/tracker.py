"""Oracle restatement of the tracker forward (SURVEY.md 8a rows a3..a8).

Test infrastructure (see ``oracle/__init__.py``).  Plain PyTorch fp32; the explicit formulas
below are also the specification the CUDA kernels follow.  Device-agnostic: every tensor is
created on the device of the inputs, so the same code is the CPU oracle (goldens, small cases)
and -- on ``cuda`` with TF32 off (``oracle.use_exact_fp32()``) -- the fp32 oracle for
BASELINE.json's full-size configurations and the reference's PyTorch-CUDA comparator.
"""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

EPS = 1e-08  # models/tracker.py:14


@dataclass(frozen=True)
class Geometry:
    """Video / token-grid geometry (models/extractor.py:171-177, models/tracker.py:77-94)."""
    H: int = 476
    W: int = 854
    patch: int = 14
    stride: int = 7
    radius: int = 35  # models/networks/tracker_head.py:47 (argmax_radius)

    @property
    def h(self) -> int:
        return 1 + (self.H - self.patch) // self.stride

    @property
    def w(self) -> int:
        return 1 + (self.W - self.patch) // self.stride

    @property
    def P(self) -> int:
        return self.h * self.w

    def point_affine(self):
        """(aw, ah, bw, bh) of models/tracker.py:84-93, computed in Python doubles
        exactly as the reference does, then stored as fp32 by ``torch.tensor``."""
        p, s = self.patch, self.stride
        last_h = ((self.H - p) // s) * s + (p / 2)
        last_w = ((self.W - p) // s) * s + (p / 2)
        ah = 2 / (last_h - (p / 2))
        aw = 2 / (last_w - (p / 2))
        bh = 1 - last_h * 2 / (last_h - (p / 2))
        bw = 1 - last_w * 2 / (last_w - (p / 2))
        return aw, ah, bw, bh


# --------------------------------------------------------------------------- a4
def normalize_points_for_sampling(points: torch.Tensor, geo: Geometry) -> torch.Tensor:
    """models/tracker.py:77-94 -- ``a * points + b`` with a=[aw,ah,1], b=[bw,bh,0] in fp32."""
    aw, ah, bw, bh = geo.point_affine()
    a = torch.tensor([[aw, ah, 1]], dtype=torch.float32, device=points.device)
    b = torch.tensor([[bw, bh, 0]], dtype=torch.float32, device=points.device)
    return a * points + b


def _unnormalize_clip(coord: torch.Tensor, size: int) -> torch.Tensor:
    # ATen grid_sampler, align_corners=True: ((coord + 1) / 2) * (size - 1), then
    # padding_mode='border': clip to [0, size-1].
    x = ((coord + 1.0) / 2.0) * float(size - 1)
    return torch.clamp(x, min=0.0, max=float(size - 1))


def sample_descriptors(features: torch.Tensor, points: torch.Tensor, frames_set=None) -> torch.Tensor:
    """models/tracker.py:96-111 + utils.py:75-101 (5-D ``grid_sample``), restated explicitly.

    features: N x C x h x w (the frame set).  points: B x 3 = (x_n, y_n, idx) with
    x_n, y_n already in [-1, 1] and idx the (float) index into the frame set.
    Returns B x C.  The time coordinate is normalised ``idx / (N-1) * 2 - 1``
    (utils.py:96-99, skipped division when N == 1) and un-normalised again inside
    ``grid_sample``; in fp32 that round trip is not exact, which leaks O(1e-6) of
    weight onto a neighbouring frame -- reproduced here (SURVEY.md 8a row a4).
    Trilinear weights and the corner accumulation order follow ATen's
    ``grid_sampler_3d`` (tnw, tne, tsw, tse, bnw, bne, bsw, bse).

    ``frames_set`` (optional, N ints): ``features`` is then the WHOLE video and slot z of the
    frame set is ``features[frames_set[z]]`` -- the same values as sampling the gathered copy
    ``features[frames_set]`` (models/tracker.py:316), without materialising it.

    The weights are always computed in fp32 (the leak is part of what the kernels reproduce);
    float64 ``features`` are weighted and summed in float64.
    """
    _, C, h, w = features.shape
    N = features.shape[0] if frames_set is None else frames_set.shape[0]
    pts = points.to(torch.float32)
    tn = pts[:, 2].clone()
    if N > 1:
        tn = tn / (N - 1)
    tn = tn * 2 - 1
    ix = _unnormalize_clip(pts[:, 0], w)
    iy = _unnormalize_clip(pts[:, 1], h)
    iz = _unnormalize_clip(tn, N)
    x0 = torch.floor(ix); y0 = torch.floor(iy); z0 = torch.floor(iz)
    x1 = x0 + 1; y1 = y0 + 1; z1 = z0 + 1
    corners = [  # (xi, yi, zi, weight) in ATen order
        (x0, y0, z0, (x1 - ix) * (y1 - iy) * (z1 - iz)),
        (x1, y0, z0, (ix - x0) * (y1 - iy) * (z1 - iz)),
        (x0, y1, z0, (x1 - ix) * (iy - y0) * (z1 - iz)),
        (x1, y1, z0, (ix - x0) * (iy - y0) * (z1 - iz)),
        (x0, y0, z1, (x1 - ix) * (y1 - iy) * (iz - z0)),
        (x1, y0, z1, (ix - x0) * (y1 - iy) * (iz - z0)),
        (x0, y1, z1, (x1 - ix) * (iy - y0) * (iz - z0)),
        (x1, y1, z1, (ix - x0) * (iy - y0) * (iz - z0)),
    ]
    out = torch.zeros(pts.shape[0], C, dtype=features.dtype, device=features.device)
    fs = None if frames_set is None else frames_set.long()
    for xi, yi, zi, wt in corners:
        ok = (xi >= 0) & (xi <= w - 1) & (yi >= 0) & (yi <= h - 1) & (zi >= 0) & (zi <= N - 1)
        xi = xi.clamp(0, w - 1).long(); yi = yi.clamp(0, h - 1).long(); zi = zi.clamp(0, N - 1).long()
        vals = features[zi if fs is None else fs[zi], :, yi, xi]  # B x C
        out = out + torch.where(ok[:, None], vals * wt[:, None], torch.zeros_like(vals))
    return out


# --------------------------------------------------------------------------- a5
def corr_maps(source_desc: torch.Tensor, frames: torch.Tensor, target_idx: torch.Tensor,
              faithful_einsum: bool = False, frames_set=None) -> torch.Tensor:
    """models/tracker.py:158-169.  source_desc B x C, frames N x C x h x w, target_idx B.

    corr[b] = <s_b, F[tgt_b][:, r, c]> / max(|s_b| * |F[tgt_b][:, r, c]|, 1e-8)  -> B x 1 x h x w.
    ``faithful_einsum=True`` reproduces the reference's cost profile (all B x N maps,
    then the diagonal pick); the default computes only the B needed maps.  With
    ``frames_set`` the target of map b is ``frames[frames_set[target_idx[b]]]`` (``frames`` =
    the whole video, no gathered copy) and maps sharing a target frame are one matrix product.
    """
    tgt = target_idx.long()
    if frames_set is not None and not faithful_einsum:
        tf = frames_set.long()[tgt]
        B = source_desc.shape[0]
        _, C, h, w = frames.shape
        corr = torch.empty(B, h, w, dtype=source_desc.dtype, device=frames.device)
        fnorm = torch.empty(B, h, w, dtype=source_desc.dtype, device=frames.device)
        for f in torch.unique(tf).tolist():
            sel = tf == f
            corr[sel] = (source_desc[sel] @ frames[f].reshape(C, h * w)).reshape(-1, h, w)
            fnorm[sel] = frames[f].norm(dim=0)
    elif faithful_einsum:
        vol = torch.einsum("bc,nchw->bnhw", source_desc, frames)
        corr = vol[torch.arange(source_desc.shape[0], device=vol.device), tgt]
        fnorm = frames.norm(dim=1)[tgt]
    else:
        sel = frames[tgt]  # B x C x h x w
        corr = torch.einsum("bc,bchw->bhw", source_desc, sel)
        fnorm = sel.norm(dim=1)
    snorm = source_desc.norm(dim=1)[:, None, None]
    corr = corr / torch.clamp(snorm * fnorm, min=EPS)
    return corr[:, None]


# --------------------------------------------------------------------------- a7
def normalized_conv_weight(weight: torch.Tensor) -> torch.Tensor:
    """models/networks/conv_norm.py:34-46: every (out, in) 3x3 kernel divided by its
    spatial sum; |sum| < 1e-8 -> sign(sum) * 1e-8 (sign(0) = 0 -> division by zero, as
    in the reference)."""
    w_sum = weight.sum(dim=[2, 3])[:, :, None, None].clone()
    unstable = w_sum.abs() < 1e-8
    if unstable.sum() > 0:
        w_sum[unstable] = torch.sign(w_sum[unstable]) * 1e-8
    return weight / w_sum


def refiner(cost: torch.Tensor, head_sd: dict, normalized: bool = False) -> torch.Tensor:
    """models/networks/tracker_head.py:54-58: NormalizedConv2d(1,16,3,pad 1) -> ReLU ->
    NormalizedConv2d(16,1,3,pad 1).  ``normalized=True``: the weights of ``head_sd`` are already
    the normalised ones (what the CUDA head and its reverse pass take)."""
    w1, w2 = head_sd["cnn_refiner.0.weight"], head_sd["cnn_refiner.2.weight"]
    if not normalized:
        w1, w2 = normalized_conv_weight(w1), normalized_conv_weight(w2)
    x = F.conv2d(cost, w1, bias=head_sd["cnn_refiner.0.bias"], stride=1, padding=1)
    x = torch.relu(x)
    return F.conv2d(x, w2, bias=head_sd["cnn_refiner.2.bias"], stride=1, padding=1)


# ---------------------------------------------------------------------- a6, a8
def token_pixel_grid(geo: Geometry):
    """models/networks/tracker_head.py:72-77 -> (xs[w], ys[h]) integer pixel centres."""
    hs = geo.patch // 2
    h_end = ((geo.H - 2 * hs) // geo.stride) * geo.stride + hs + math.ceil(geo.stride / 2)
    w_end = ((geo.W - 2 * hs) // geo.stride) * geo.stride + hs + math.ceil(geo.stride / 2)
    ys = torch.arange(hs, h_end, geo.stride)
    xs = torch.arange(hs, w_end, geo.stride)
    return xs, ys


def head_forward(cost_relu: torch.Tensor, head_sd: dict, geo: Geometry, return_aux: bool = False,
                 amax=None, fb=None, normalized: bool = False):
    """models/networks/tracker_head.py:107-121 (+ soft_argmax :68-98, softmax :100-105).

    cost_relu: B x 1 x h x w (already ReLU'd, models/tracker.py:173).  Returns B x 2 in
    [-1, 1] (RangeNormalizer((W, H)), dst=(-1,1): x / (W-1, H-1), * 2, + (-1);
    data/dataset.py:33-35).

    ``amax`` / ``fb`` (optional, B each): pin the arg-max token and the stability branch to
    given decisions (e.g. a kernel's ``aux``) instead of taking them from this evaluation, so
    that a higher-precision evaluation of a near-tie stays on the kernel's piecewise branch.
    The aux dict then also holds this evaluation's own decisions ("own_argmax",
    "own_fallback").  ``normalized``: see ``refiner``.
    """
    B, _, h, w = cost_relu.shape
    flat = cost_relu[:, 0].reshape(B, -1)
    own_amax = torch.argmax(flat, dim=1)  # first maximal index
    amax = own_amax if amax is None else amax.to(own_amax)
    row, col = amax // w, amax % w
    z = refiner(cost_relu, head_sd, normalized)
    p = torch.softmax(z.reshape(B, 1, -1), dim=2).reshape(B, h, w)
    xs, ys = token_pixel_grid(geo)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    grid = torch.stack((gx, gy), -1).to(cost_relu.device)  # h x w x 2 (x, y), int64
    hs = geo.patch // 2
    centre = torch.stack((col * geo.stride + hs, row * geo.stride + hs), dim=-1)  # B x 2
    mask = torch.norm((grid[None] - centre[:, None, None]).to(torch.float32), dim=-1) <= geo.radius
    hm = p * mask
    s = hm.sum(dim=(1, 2))
    own_fb = s < 1e-8
    fb = own_fb if fb is None else fb.to(own_fb)
    if fb.any():  # numerical-stability branch, tracker_head.py:87-94
        uniform = 1 / mask[fb].sum(dim=(1, 2))
        hm[fb] = (hm[fb] + uniform[:, None, None]) * mask[fb]
        s[fb] = hm[fb].sum(dim=(1, 2))
    point = (grid[None] * hm[..., None]).sum(dim=(1, 2)) / s[:, None]
    norm = torch.tensor([geo.W, geo.H], dtype=torch.float32, device=point.device) - 1
    out = point / norm
    out = (1 - (-1)) * out + (-1)
    if return_aux:
        return out, {"argmax": amax, "fallback": fb, "logits": z[:, 0], "point_px": point,
                     "own_argmax": own_amax, "own_fallback": own_fb}
    return out


def unnormalize_xy(coords: torch.Tensor, geo: Geometry) -> torch.Tensor:
    """RangeNormalizer.unnormalize(src=(-1,1), dims=[0,1]) (data/dataset.py:39-53) as
    called in models/model_inference.py:52,144: (v - (-1)) / (1 - (-1)) * (W-1, H-1)."""
    norm = torch.tensor([geo.W, geo.H], dtype=torch.float32, device=coords.device) - 1
    x = (coords - (-1)) / (1 - (-1))
    return x * norm


# ---------------------------------------------------------------------- a3 + forward
def tracker_forward(features: torch.Tensor, inp, head_sd: dict, geo: Geometry,
                    faithful: bool = False) -> torch.Tensor:
    """models/tracker.py:303-325 with cached refined features (the inference path).

    features: T x C x h x w (refined).  inp = (source_points B x 3 px, source_frame_indices B,
    target_frame_indices B, frames_set_t N).  Returns B x 2 in [-1, 1].
    """
    src_pts, src_idx, tgt_idx, frames_set_t = inp
    pn = normalize_points_for_sampling(src_pts.to(torch.float32), geo)
    pts = torch.cat([pn[:, :-1], src_idx[:, None].to(torch.float32)], dim=1)
    if faithful:   # the reference's cost profile: two gathered copies of the frame set, B x N einsum
        frames = features[frames_set_t.long()]  # models/tracker.py:316 (gather copy)
        _ = features[frames_set_t.long()]  # models/tracker.py:317: second, unused gather
        desc = sample_descriptors(frames, pts)
        corr = corr_maps(desc, frames, tgt_idx, faithful_einsum=True)
    else:          # same values, frame set addressed through its index vector
        desc = sample_descriptors(features, pts, frames_set_t)
        corr = corr_maps(desc, features, tgt_idx, frames_set=frames_set_t)
    return head_forward(torch.relu(corr), head_sd, geo)

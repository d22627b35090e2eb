"""The tracker node's reverse pass in float64, for the CPU and GPU tests of ``dinotrk_track_backward``.

``oracle_coords`` is the oracle chain (sample -> cosine maps -> ReLU -> refiner -> soft-argmax) in the dtype of its
inputs, with the arg-max, the stability branch and the ReLU of the maps pinned to given decisions; autograd through
it is the reference gradient.  ``abs_reverse`` evaluates the same reverse chain with every operand replaced by its
absolute value (forward quantities by their absolute-value evaluations) and every sum taken over absolute values:
per output element it gives M, the scale of the rounding error any evaluation order of the chain can make, so that
|kernel - reference| <= kappa * 2^-24 * M.  See tests/test_train_backward_gpu.py for the derivation.
"""
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from oracle import tracker as ot

U = 2.0 ** -24
# pre-activations of the refiner's hidden layer this close to the ReLU's kink (relative to their absolute-value
# evaluation) may take either branch in fp32: the bound then covers both (see abs_reverse).  The kernel's pre-activation
# is b1 + 9 fused multiply-adds on maps that are themselves fp32-faithful: within ~16 u of exact, 2^-20; doubled.
KINK = 2.0 ** -19


def head_sd(w1, b1, w2, b2):
    return {"cnn_refiner.0.weight": w1, "cnn_refiner.0.bias": b1, "cnn_refiner.2.weight": w2, "cnn_refiner.2.bias": b2}


def normalized_weights(head, dtype=torch.float32, device="cpu"):
    """(w1n 16x1x3x3, b1 16, w2n 1x16x3x3, b2 1) as the kernels take them: normalised in fp32, then cast."""
    w1 = ot.normalized_conv_weight(head["cnn_refiner.0.weight"].float())
    w2 = ot.normalized_conv_weight(head["cnn_refiner.2.weight"].float())
    return tuple(t.to(device=device, dtype=dtype) for t in (w1, head["cnn_refiner.0.bias"], w2, head["cnn_refiner.2.bias"]))


def worst_ratio(err, bound):
    """max of err / bound; an element with bound 0 must have err 0 (else inf)."""
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return r.max().item() if r.numel() else 0.0


def draw_grad_out(B, gen):
    """d loss / d coords, B x 2 fp32: both signs, magnitudes spread over 1e-3 .. 1e3 across maps (a wrong map is then
    invisible to any bar relative to a tensor maximum), every 7th map exactly 0 in x, every 11th in both coordinates."""
    mag = 10.0 ** (torch.rand(B, 1, generator=gen) * 6 - 3)
    g = torch.randn(B, 2, generator=gen) * mag
    g[::7, 0] = 0
    g[::11] = 0
    return g.float()


def sampling_points(pts, geo):
    """pts B x 3 = (x_px, y_px, slot) -> (x_n, y_n, slot) in fp32, exactly as the kernels normalise."""
    return ot.normalize_points_for_sampling(pts.to(torch.float32), geo)


def oracle_coords(feats, pts_n, tgt_slot, frames_set, wts, geo, amax=None, fb=None, relu_mask=None):
    """B x 2 normalised coordinates and the head's aux.  feats T x C x h x w (any float dtype; the whole video, slot z
    of the frame set is feats[frames_set[z]]), pts_n B x 3 from ``sampling_points``, wts the normalised refiner weights.
    relu_mask (B x 1 x h x w bool, optional) replaces relu(corr) by corr * relu_mask."""
    desc = ot.sample_descriptors(feats, pts_n, frames_set)
    corr = ot.corr_maps(desc, feats, tgt_slot, frames_set=frames_set)
    m = torch.relu(corr) if relu_mask is None else corr * relu_mask
    return ot.head_forward(m, head_sd(*wts), geo, return_aux=True, amax=amax, fb=fb, normalized=True)


def reference_gradients(feats, pts_n, tgt_slot, frames_set, wts, geo, grad_out, amax, fb, relu_mask):
    """Autograd through ``oracle_coords`` in the dtype of feats: (d/dfeats T x C x h x w, d/dw 305, coords, aux)."""
    f = feats.detach().clone().requires_grad_(True)
    w = [t.detach().to(feats.dtype).clone().requires_grad_(True) for t in wts]
    out, aux = oracle_coords(f, pts_n, tgt_slot, frames_set, w, geo, amax, fb, relu_mask)
    gf, *gw = torch.autograd.grad(out, [f] + w, grad_out.to(out.dtype))
    return gf, torch.cat([g.reshape(-1) for g in gw]), out.detach(), aux


@torch.no_grad()
def abs_reverse(feats, pts_n, tgt_slot, frames_set, wts, geo, grad_out, amax, fb, relu_mask, kappa, full_softmax=False):
    """M for d/dfeats (T x C x h x w) and d/dw (305), float64, plus per-map diagnostics.

    Forward quantities enter by their absolute-value evaluations: |s|.|F| / D for the map, |b1| + |w1| * m_abs for the
    hidden layer, |b2| + |w2| * h_abs for the logits.  The softmax is exact up to the error of its exp argument,
    relative (1 + z_abs + z_abs_max) u; the per-map factor fz = 1 + 2 max_p z_abs multiplies the map's d/dlogits.
    The soft-argmax point (px, py) is a q-weighted mean over the disc: relative errors of q up to fz u move it by at
    most fz u times the disc's diameter 2 r, its fp32 sums by a few u px; so |gx - px| enters as |gx - px| + 2 r +
    px / fz (the factor fz is applied once, on d/dlogits).

    Two terms are not rounding errors of the kernel and enter with weights that make kappa u M cover them in full:
    a hidden pre-activation within KINK of its kink may take the other ReLU branch in fp32 (its |d/dhidden|, formed
    from |d/dlogits| without the error factors above, weight 1 / (kappa u)); off the disc of a map not on the stability branch the exact d/dlogits is 0 (sum_q p_q dL/dp_q = 0),
    which the kernel uses and float64 autograd reproduces only up to its rounding (sum_q p_q |dL/dp_q|, weight
    2^-45 / (kappa u)).  ``full_softmax``: bound an fp32 evaluation that forms that sum for every map, as autograd
    does (weight 1)."""
    T, C, h, w = feats.shape
    P = h * w
    B = pts_n.shape[0]
    feats = feats.double()
    A = feats.abs()
    w1, b1, w2, b2 = (t.double() for t in wts)
    fs = frames_set.long()
    tf = fs[tgt_slot.long()]
    desc = ot.sample_descriptors(feats, pts_n, frames_set)
    desc_a = ot.sample_descriptors(A, pts_n, frames_set)           # trilinear weights are >= 0
    dot = torch.empty(B, P, dtype=torch.float64, device=feats.device)
    dot_a = torch.empty_like(dot)
    for f in torch.unique(tf).tolist():
        sel = tf == f
        dot[sel] = desc[sel] @ feats[f].reshape(C, P)
        dot_a[sel] = desc_a[sel] @ A[f].reshape(C, P)
    sn = desc.norm(dim=1)
    fn = feats.norm(dim=1).reshape(T, P)[tf]                          # B x P
    prod = sn[:, None] * fn
    D = prod.clamp_min(ot.EPS)
    free = prod > ot.EPS                                              # clamp inactive
    rm = relu_mask.reshape(B, P).double()
    relu_moved = (dot > 0) != relu_mask.reshape(B, P)
    m = (dot / D * rm).reshape(B, 1, h, w)
    m_a = (dot_a / D * rm).reshape(B, 1, h, w)
    del dot, dot_a
    pre1 = F.conv2d(m, w1, b1, padding=1)
    h_a = F.conv2d(m_a, w1.abs(), b1.abs(), padding=1)
    z = F.conv2d(torch.relu(pre1), w2, b2, padding=1).reshape(B, P)
    z_a = F.conv2d(h_a, w2.abs(), b2.abs(), padding=1)
    fz = 1 + 2 * z_a.reshape(B, P).amax(dim=1)
    p = torch.softmax(z, dim=1)
    # soft-argmax on the (pinned) disc
    xs, ys = ot.token_pixel_grid(geo)
    gx = xs.double().to(feats.device).repeat(h)
    gy = ys.double().to(feats.device).repeat_interleave(w)
    hs = geo.patch // 2
    am = amax.long().to(feats.device)
    cx = (am % w) * geo.stride + hs
    cy = (am // w) * geo.stride + hs
    disc = ((gx[None] - cx[:, None]) ** 2 + (gy[None] - cy[:, None]) ** 2) <= geo.radius ** 2
    fbd = fb.to(device=feats.device, dtype=torch.bool)
    uni = fbd.double() / disc.sum(1)
    q = (p + uni[:, None]) * disc
    s2 = q.sum(1)
    px, py = (gx * q).sum(1) / s2, (gy * q).sum(1) / s2
    g = grad_out.double().abs()
    dpx, dpy = g[:, 0] * 2 / (geo.W - 1), g[:, 1] * 2 / (geo.H - 1)
    d2 = 2 * geo.radius
    ex = (gx[None] - px[:, None]).abs() + d2 + px[:, None] / fz[:, None]
    ey = (gy[None] - py[:, None]).abs() + d2 + py[:, None] / fz[:, None]
    dq = disc * (ex * dpx[:, None] + ey * dpy[:, None]) / s2[:, None]
    dot_q = (p * dq).sum(1)
    real = torch.where(fbd | full_softmax, 1.0, 0.0)
    dz_real = (fz[:, None] * p * (dq + (dot_q * real)[:, None])).reshape(B, 1, h, w)
    dz = dz_real + (fz * dot_q * (1 - real) * 2.0 ** -45 / (kappa * U))[:, None, None, None] * p.reshape(B, 1, h, w)
    # |d/dlogits| itself (no error factors): a flipped ReLU branch changes the gradient by at most |d/dhidden|
    dq_t = disc * ((gx[None] - px[:, None]).abs() * dpx[:, None] + (gy[None] - py[:, None]).abs() * dpy[:, None]) / s2[:, None]
    dz_t = (p * (dq_t + ((p * dq_t).sum(1) * fbd)[:, None])).reshape(B, 1, h, w)
    del q, dq, dq_t, p, ex, ey, dz_real
    # refiner backward
    dhid = conv2d_input(h_a.shape, w2.abs(), dz, padding=1)
    dhid_t = conv2d_input(h_a.shape, w2.abs(), dz_t, padding=1)
    kink = (pre1.abs() <= KINK * h_a) & (dhid_t > 0)
    n_kink = int(kink.sum().item())
    dpre = dhid * (pre1 > 0) + dhid_t * kink / (kappa * U)
    del pre1, kink, dhid_t, dz_t
    gw2 = conv2d_weight(h_a, w2.shape, dz, padding=1)
    gb2 = dz.sum().reshape(1)
    gw1 = conv2d_weight(m_a, w1.shape, dpre, padding=1)
    gb1 = dpre.sum(dim=(0, 2, 3))
    dm = conv2d_input(m_a.shape, w1.abs(), dpre, padding=1).reshape(B, P) * rm
    del dhid, dpre, h_a
    # cosine backward: d/ds = g (F / D - corr s / |s|^2), d/dF = g (s / D - corr F / |F|^2), second terms where free
    corr_a = m_a.reshape(B, P)
    la = dm / D
    lb = torch.where(free, dm * corr_a / fn.clamp_min(1e-300) ** 2, torch.zeros_like(dm))
    selfc = torch.where(sn > 0, (dm * corr_a * free).sum(1) / sn.clamp_min(1e-300) ** 2, torch.zeros_like(sn))
    ddesc = selfc[:, None] * desc_a
    M = torch.zeros(T, P, C, dtype=torch.float64, device=feats.device)
    for f in torch.unique(tf).tolist():
        sel = tf == f
        Af = A[f].reshape(C, P)
        ddesc[sel] += la[sel] @ Af.T
        M[f] += la[sel].T @ desc_a[sel] + lb[sel].sum(0)[:, None] * Af.T
    del la, lb, dm
    # trilinear scatter of d/ddescriptor
    leaf = torch.zeros_like(feats).requires_grad_(True)
    with torch.enable_grad():
        (Ms,) = torch.autograd.grad(ot.sample_descriptors(leaf, pts_n, frames_set), leaf, ddesc)
    M = M.reshape(T, h, w, C).permute(0, 3, 1, 2) + Ms
    Mw = torch.cat([gw1.reshape(-1), gb1, gw2.reshape(-1), gb2])
    return M, Mw, {"fz": fz, "n_kink": n_kink, "n_relu": int(relu_moved.sum()), "n_relu_maps": int(relu_moved.any(1).sum())}


def sample_abs(feats_shape, pts_n, frames_set, grad_desc, dtype=torch.float64):
    """M of the sampling backward alone: the trilinear weights (>= 0) applied to |grad_desc|."""
    leaf = torch.zeros(feats_shape, dtype=dtype, device=grad_desc.device, requires_grad=True)
    (M,) = torch.autograd.grad(ot.sample_descriptors(leaf, pts_n, frames_set), leaf, grad_desc.abs().to(dtype))
    return M

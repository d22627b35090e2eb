"""Seeded synthetic inputs shared by the golden generator, the tests and bench.py.

Test/bench infrastructure (see ``oracle/__init__.py``).  Everything is drawn from
``numpy.random.RandomState`` (bit-stable legacy generator) so that fixtures can be
regenerated from a seed on any box.
"""
import numpy as np
import torch


def shifted_field_features(T, C, h, w, seed=0, noise=0.15, max_shift=3, smooth=True):
    """A smooth random descriptor field that translates by a few tokens per frame plus noise:
    tracks are non-trivial, most frames pass the 0.7 anchor cos-sim threshold (SURVEY.md 8d).
    Returns (features T x C x h x w fp32, shifts T x 2 int (dy, dx))."""
    rs = np.random.RandomState(seed)
    pad = max_shift * 2 + 2
    base = rs.standard_normal((C, h + 2 * pad, w + 2 * pad)).astype(np.float32)
    if smooth:
        b = base.copy()
        b[:, 1:-1, 1:-1] = (base[:, 1:-1, 1:-1] * 0.5 + 0.125 * (base[:, :-2, 1:-1] + base[:, 2:, 1:-1]
                            + base[:, 1:-1, :-2] + base[:, 1:-1, 2:]))
        base = b
    shifts = np.zeros((T, 2), dtype=np.int64)
    for t in range(1, T):
        shifts[t] = np.clip(shifts[t - 1] + rs.randint(-1, 2, size=2), -max_shift, max_shift)
    feats = np.empty((T, C, h, w), dtype=np.float32)
    for t in range(T):
        dy, dx = shifts[t]
        feats[t] = base[:, pad + dy: pad + dy + h, pad + dx: pad + dx + w]
        feats[t] += noise * rs.standard_normal((C, h, w)).astype(np.float32)
    return torch.from_numpy(feats), torch.from_numpy(shifts)


def random_features(T, C, h, w, seed=0):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.standard_normal((T, C, h, w)).astype(np.float32))


def random_video(T, H, W, seed=0):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.random_sample((T, 3, H, W)).astype(np.float32))


def head_weights(kind="well", seed=0):
    """Head state dict (keys of models/networks/tracker_head.py:54-58).
    'well': U(0.2, 1) for all four tensors (kernel sums far from 0, SURVEY.md 8d);
    'default': PyTorch-default-like init -> kernel sums ~0 -> huge logits -> every map takes the
               numerical-stability fallback branch; 'mixed': mixed-sign but non-degenerate sums."""
    rs = np.random.RandomState(1000 + seed)
    def u(lo, hi, *shape):
        return torch.from_numpy(rs.uniform(lo, hi, size=shape).astype(np.float32))
    if kind == "well":
        sd = {"cnn_refiner.0.weight": u(0.2, 1, 16, 1, 3, 3), "cnn_refiner.0.bias": u(0.2, 1, 16),
              "cnn_refiner.2.weight": u(0.2, 1, 1, 16, 3, 3), "cnn_refiner.2.bias": u(0.2, 1, 1)}
    elif kind == "default":
        # mixed-sign kernels whose spatial sums are tiny (like PyTorch-default init in the probe of
        # SURVEY.md 8d): normalisation blows the gain up, the softmax collapses onto a spot unrelated
        # to the pre-CNN arg-max, and the disc mass drops below 1e-8 -> fallback branch.
        def tiny_sum(o, i, total):
            r = u(-1, 1, o, i, 3, 3)
            return r - r.mean(dim=(2, 3), keepdim=True) + total / 9
        sd = {"cnn_refiner.0.weight": tiny_sum(16, 1, 0.05), "cnn_refiner.0.bias": u(-1 / 3, 1 / 3, 16),
              "cnn_refiner.2.weight": tiny_sum(1, 16, 0.05), "cnn_refiner.2.bias": u(-1 / 12, 1 / 12, 1)}
    elif kind == "mixed":
        w1 = u(-0.5, 1, 16, 1, 3, 3); w2 = u(-0.5, 1, 1, 16, 3, 3)
        sd = {"cnn_refiner.0.weight": w1, "cnn_refiner.0.bias": u(-0.2, 0.2, 16),
              "cnn_refiner.2.weight": w2, "cnn_refiner.2.bias": u(-0.2, 0.2, 1)}
    elif kind == "sharp":
        # 'well' with a large gain folded in: kernel sums stay O(1) after normalisation, but the
        # centre tap dominates -> peaked softmax (closer to a trained head)
        w1 = u(0.0, 0.05, 16, 1, 3, 3); w1[:, :, 1, 1] += 1.0
        w2 = u(0.0, 0.05, 1, 16, 3, 3); w2[:, :, 1, 1] += 1.0
        sd = {"cnn_refiner.0.weight": w1, "cnn_refiner.0.bias": u(-0.05, 0.05, 16),
              "cnn_refiner.2.weight": w2, "cnn_refiner.2.bias": u(-0.05, 0.05, 1)}
    else:
        raise ValueError(kind)
    return sd


def scaled(feats, k):
    """feats * 2^k.  Exact in fp32 while no element leaves the normal range, so every cosine -- and the oracle's output,
    as long as |d| |F| stays above its 1e-8 clamp -- is unchanged bit for bit; only the kernels' fp16 operands notice."""
    return feats * (2.0 ** k)


def massive_channels(feats, n_big=4, seed=0):
    """Per-channel range like DINOv2's massive activations: `n_big` channels scaled by 2^8 .. 2^10, the rest by 2^-6
    (powers of two: exact).  feats T x C x h x w."""
    rs = np.random.RandomState(2000 + seed)
    C = feats.shape[1]
    e = np.full(C, -6.0)
    e[rs.choice(C, n_big, replace=False)] = rs.randint(8, 11, size=n_big)
    return feats * torch.from_numpy(2.0 ** e).to(feats.dtype).view(1, C, 1, 1)


def twin_peak(feats, src, dst, gaps, seed=0):
    """Far-apart twins: in frame t (t = 0 .. len(gaps) - 1) token `dst` becomes a copy of token `src` (row, col) of the
    same frame plus a component orthogonal to every token of the 3 x 3 neighbourhoods of `src` in all frames, so that
    for every descriptor d bilinearly sampled inside those neighbourhoods (float64)
        cos(d, copy) = cos(d, orig) / sqrt(1 + eta_t)   with   eta_t chosen so that  1 - 1/sqrt(1 + eta_t) = gaps[t]:
    a descriptor whose cosine with the original is c sees a second peak c * gaps[t] lower, far away.  Returns a copy of
    feats (T x C x h x w fp32; storing it in fp32 moves each gap by up to ~3e-8, see the construction test)."""
    T, C, h, w = feats.shape
    f = feats.double().clone()
    r0, c0 = src
    nb = f[:, :, max(r0 - 1, 0):r0 + 2, max(c0 - 1, 0):c0 + 2].permute(1, 0, 2, 3).reshape(C, -1)
    assert nb.shape[1] < C, "the orthogonal complement of the neighbourhoods is empty: use more channels"
    q, _ = torch.linalg.qr(nb)
    rs = np.random.RandomState(3000 + seed)
    for t, gap in enumerate(gaps):
        o = f[t, :, r0, c0]
        v = torch.from_numpy(rs.standard_normal(C))
        v = v - q @ (q.t() @ v)
        v = v - q @ (q.t() @ v)
        eta = 1.0 / (1.0 - gap) ** 2 - 1.0
        f[t, :, dst[0], dst[1]] = o + v * (o.norm() * np.sqrt(eta) / v.norm())
    return f.float()


def rounding_aligned_twin(feats, src, dst, gap, seed=0):
    """Twins the fp16 rounding orders against their exact order.  Token `src` (row, col) becomes, in every frame, a vector o
    whose components all sit 2^-6 fp16 ulp BELOW a rounding midpoint (rn_fp16 shrinks each by ~2^-11 relative), token `dst`
    a vector c whose components sit 2^-6 ulp ABOVE one (rn_fp16 grows each), c = o + up to 190 fp16 ulps per
    component, with the float64 cos(o, c) = 1 - g, g as close to `gap` as the ulp grid allows.  For a descriptor equal to o
    the single-pass fp16 cosines are then about 1 - 2 r for o (r ~ 2^-11 / 1.19, the relative rounding at these mantissas)
    and 1 - g for c: the coarse pass reverses the twins when g < ~8e-4 (never more than 2^-10: inside XW_EPS).
    Returns (feats fp32 copy, g).  The components are exact in fp32 (16 significant bits)."""
    T, C, h, w = feats.shape
    rs = np.random.RandomState(4000 + seed)
    ulp = 2.0 ** -10
    e = np.floor(np.log2(np.abs(rs.standard_normal(C)) + 0.25))
    sgn = np.where(rs.random_sample(C) < 0.5, -1.0, 1.0)
    j = rs.randint(192, 200, size=C)
    o = sgn * 2.0 ** e * (1 + (j + 0.5) * ulp - 2.0 ** -16)
    u = rs.uniform(-1, 1, size=C)

    def copy(lam):
        m = np.round(lam * u)
        return sgn * 2.0 ** e * (1 + (j + m + 0.5) * ulp + 2.0 ** -16)

    def g_of(c):
        return 1.0 - o @ c / (np.linalg.norm(o) * np.linalg.norm(c))

    lo, hi = 0.0, 190.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if g_of(copy(mid)) < gap else (lo, mid)
    c = copy(hi)
    f = feats.clone()
    f[:, :, src[0], src[1]] = torch.from_numpy(o).to(f.dtype)
    f[:, :, dst[0], dst[1]] = torch.from_numpy(c).to(f.dtype)
    return f, float(g_of(c))


def lattice_query_points(n_side_x, n_side_y, H, W, t_q=0, margin=20.0, jitter_seed=None):
    xs = np.linspace(margin, W - 1 - margin, n_side_x, dtype=np.float32)
    ys = np.linspace(margin, H - 1 - margin, n_side_y, dtype=np.float32)
    gx, gy = np.meshgrid(xs, ys)
    pts = np.stack([gx.reshape(-1), gy.reshape(-1)], -1)
    if jitter_seed is not None:
        pts = pts + np.random.RandomState(jitter_seed).uniform(-3, 3, size=pts.shape).astype(np.float32)
    t = np.full((pts.shape[0], 1), float(t_q), dtype=np.float32) if np.isscalar(t_q) else \
        np.asarray(t_q, dtype=np.float32).reshape(-1, 1)
    return torch.from_numpy(np.concatenate([pts, t], 1).astype(np.float32))

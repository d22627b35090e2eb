"""GPU tests: the tracker node's reverse pass (``dinotrk_track_backward``, csrc/train.cu) and ``dinotrk_sample_backward``
element by element against float64, at the shape the training step ships (config/train.yaml: 476 x 854 frames, a
67 x 121 token grid, N = 4, B = 512, C = 1024) and at the edges where the kernels clip, clamp or branch.

Forward.  ``train.track_forward`` -- the production forward of the tracker node (grouping, sorting, the head with aux)
-- gives desc, desc_norm, maps and aux; the tests then call ``dinotrk_track_backward`` directly.  The case with a
non-identity frame set calls the C ABI for the forward too.

Reference.  Autograd through the oracle chain (oracle/tracker.py) in float64, fed the same fp32 inputs (embeddings,
normalised refiner weights, points, grad_out) and pinned to the kernel's decisions: arg-max and stability branch from
``aux``, the ReLU of the maps from ``maps > 0``.  The trilinear weights stay fp32 (the temporal leak included): they
are part of what the kernel reproduces.  Maps whose own float64 arg-max or branch differs from ``aux`` are counted and
printed; they are compared on the kernel's branch.

Bound.  ``track_reverse.abs_reverse`` runs the reverse chain again in float64 with every operand replaced by its
absolute value and every sum taken over absolute values, giving M per output element.  An fp32 evaluation of the
chain in any order (atomics included) errs by at most a small multiple of u M, u = 2^-24, for every operation
whose result is rounded contributes at most u times the absolute value of what it sums.  Two effects are not of that
form and are carried into M by construction: the softmax is exact only up to the error of its exp argument, which is
relative, (1 + |z| + |z_max|) u with z the logits (taken at their absolute-value evaluation, per map, as a factor on the
map's d/dlogits); and a hidden pre-activation within 2^-19 of the ReLU's kink may take the other branch.  The
gradient buffers start with a pattern of the size of M (never subnormal: global fp32 atomics flush subnormals to
zero); the kernel adds into it, so what is compared is
(result - pattern) against the reference, within kappa u (M + |pattern|).  kappa is measured and pinned below.

Exact checks (no tolerance): elements no map can reach keep the pattern bit for bit (a map off the stability branch
reaches its +-7-token window in the target frame and its sampling corners; a map on it the whole target frame); the
slots after the 305 weight gradients stay untouched; grad_tpc = NULL leaves grad_w within its bound; B = 0 writes
nothing; host-side argument errors return DINOTRK_EINVAL before any launch.
"""
import ctypes
import time
import zlib

import pytest
import torch

from dino_tracker_b200 import _lib
from dino_tracker_b200 import train as dtrain
from oracle import synth
from oracle.tracker import Geometry

import track_reverse as tr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHIPPED = Geometry(H=476, W=854)
SMALL = Geometry(H=154, W=210)
EINVAL = -22                  # DINOTRK_EINVAL
# Worst error / (u (M + |pattern|)) measured on an H100 80GB HBM3 (700 W power limit) over every case of this file:
# grad_tpc 9.6 (shipped, "sharp", fp16x3), grad_w 8.9 (shipped, "well", fp32), dinotrk_sample_backward 13.9 (4,096
# clustered points); pinned with more than 3x headroom.
KAPPA_TPC = 32.0
KAPPA_W = 28.0
KAPPA_SAMPLE = 48.0


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _tpc(feats):
    T, C, h, w = feats.shape
    return feats.permute(0, 2, 3, 1).reshape(T, h * w, C)


def _tracker(geo, feats, precision):
    from dino_tracker_b200 import Tracker
    T, C = feats.shape[:2]
    return Tracker(video=torch.zeros(T, 3, geo.H, geo.W, device=DEV), dino_embed_video=feats, device=DEV,
                   delta_channels=[3, 4, 4, 4, C], corr_precision=precision)


def _backward(feat, geom, hw, pts, fs, desc, dn, tgt_frame, maps, aux, g, grad_w, grad_tpc, ws_short=0, B=None):
    lib = _lib.load()
    C = desc.shape[1]
    B = desc.shape[0] if B is None else B
    ws_bytes = lib.dinotrk_track_backward_workspace_bytes(B, C, ctypes.byref(geom))
    ws = torch.empty(max(ws_bytes, 1), device=DEV, dtype=torch.uint8)
    return lib.dinotrk_track_backward(ctypes.byref(feat), ctypes.byref(geom), ctypes.byref(hw), _lib.ptr(pts), _lib.ptr(fs),
                                      fs.shape[0], _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(tgt_frame), _lib.ptr(maps), _lib.ptr(aux),
                                      _lib.ptr(g), B, _lib.ptr(grad_w), _lib.ptr(grad_tpc), _lib.ptr(ws), ws_bytes - ws_short,
                                      _lib.stream_ptr())


def _pattern(M, gen):
    """fp32 prefill: random signs, magnitude 0.5 .. 1 times M (1 where M is 0), never below 2^-100.  Global fp32 atomics
    flush subnormals to zero, so the values the kernel adds into must stay in the normal range."""
    r = torch.rand(M.shape, generator=gen, dtype=torch.float64).to(M.device)
    sign = torch.where(torch.rand(M.shape, generator=gen).to(M.device) < 0.5, -1.0, 1.0)
    return (sign * (0.5 + 0.5 * r) * torch.where(M > 0, M, torch.ones_like(M)).clamp_min(2.0 ** -100)).float()


def _reachable(T, h, w, tgt_frame, amax, fb, pts_n, fs):
    """Tokens (T x P) a map may write: its +-7-token window in the target frame (the whole frame on the stability
    branch) and its sampling corners of non-zero weight."""
    R = torch.zeros(T, h, w, dtype=torch.bool)
    for f, a, b in zip(tgt_frame.tolist(), amax.tolist(), fb.tolist()):
        if b:
            R[f] = True
        else:
            r, c = divmod(a, w)
            R[f, max(r - 7, 0):r + 8, max(c - 7, 0):c + 8] = True
    S = tr.sample_abs((T, 1, h, w), pts_n, fs, torch.ones(pts_n.shape[0], 1, device=pts_n.device)) > 0
    return R.to(S.device).reshape(T, h * w) | S.reshape(T, h * w)


def _worst(label, got, pattern, ref, M, kappa):
    d = got.double() - pattern.double()
    bound = tr.U * (M + pattern.double().abs())
    err = (d - ref).abs()
    ratio = tr.worst_ratio(err, bound) / kappa
    print(f"  [{label}] worst error / bound = {ratio:.4f} (error / (u (M + |pattern|)) = {ratio * kappa:.3f})")
    if ratio > 1:
        i = torch.argmax(torch.where(bound > 0, err / bound.clamp_min(1e-300), err * 1e300)).item()
        at = [int(v) for v in torch.unravel_index(torch.tensor(i), tuple(ref.shape))]
        print(f"    worst at {at}: got {d.flatten()[i].item():.6g}, reference {ref.flatten()[i].item():.6g}, "
              f"M {M.flatten()[i].item():.3g}")
    return ratio


def _seen(label, ref, pattern, M, kappa):
    """Worst |ref| / bound: above 1 means a kernel that left this gradient out would fail the bound somewhere."""
    r = tr.worst_ratio(ref.abs(), tr.U * (M + pattern.double().abs())) / kappa
    print(f"  [{label}] reference / bound reaches {r:.3g}")
    return r


def check_track_backward(label, feats, fs, pts_sorted, tgt_slot_sorted, wts, geo, g_sorted, maps, aux, feat, geom, hw,
                         desc, dn, must_see=None):
    """Reference, bound, prefilled kernel call and every check of the module docstring for one forward.  Non-vacuity:
    the reference gradient must exceed the bound on some element of grad_tpc and of grad_w, and so must the gradient of
    the maps selected by each mask of ``must_see`` (sorted order) alone, on grad_tpc."""
    t0 = time.time()
    T, C, h, w = feats.shape
    P = h * w
    B = desc.shape[0]
    f64 = feats.to(DEV, torch.float64)
    fs = fs.to(DEV)
    tgt_frame = fs.long()[tgt_slot_sorted.long()].to(torch.int32).contiguous()
    pts_n = tr.sampling_points(pts_sorted, geo)
    amax, fb = aux[:, 0].long(), aux[:, 1].bool()
    rm = (maps[:, :P] > 0).reshape(B, 1, h, w)
    wts64 = tuple(t.to(DEV, torch.float64) for t in wts)
    ref_f, ref_w, _, oaux = tr.reference_gradients(f64, pts_n, tgt_slot_sorted, fs, wts64, geo, g_sorted, amax, fb, rm)
    moved = int(((oaux["own_argmax"] != amax) | (oaux["own_fallback"] != fb)).sum())
    M, Mw, info = tr.abs_reverse(f64, pts_n, tgt_slot_sorted, fs, wts64, geo, g_sorted, amax, fb, rm,
                                 min(KAPPA_TPC, KAPPA_W))
    del f64
    ref_t, M_t = _tpc(ref_f), _tpc(M)
    del ref_f, M
    reach = _reachable(T, h, w, tgt_frame.cpu(), amax.cpu(), fb.cpu(), pts_n, fs)
    gen = _gen(label)
    pat_t, pat_w = _pattern(M_t, gen), _pattern(torch.cat([Mw, torch.zeros(64, device=DEV, dtype=torch.float64)]), gen)
    grad_tpc, grad_w = pat_t.clone(), pat_w.clone()
    g32 = g_sorted.to(DEV, torch.float32).contiguous()
    pts32 = pts_sorted.to(DEV, torch.float32).contiguous()
    _lib.check(_backward(feat, geom, hw, pts32, fs, desc, dn, tgt_frame, maps, aux, g32, grad_w, grad_tpc), "track_backward")
    grad_w_null = pat_w.clone()
    _lib.check(_backward(feat, geom, hw, pts32, fs, desc, dn, tgt_frame, maps, aux, g32, grad_w_null, None), "track_backward")
    torch.cuda.synchronize()
    print(f"[{label}] B = {B}, stability-branch maps {int(fb.sum())}, float64 arg-max / branch differing from aux: {moved}, "
          f"hidden pre-activations at the ReLU kink: {info['n_kink']}, max logit factor {info['fz'].max().item():.3g}, "
          f"map elements whose float64 ReLU decision differs from maps > 0: {info['n_relu']} (in {info['n_relu_maps']} maps)")
    if fb.any():
        print(f"  stability-branch maps: target frames {tgt_frame[fb].tolist()}, arg-max {amax[fb].tolist()}")
    unreached = ~reach
    assert torch.equal(grad_tpc[unreached].view(torch.int32), pat_t[unreached].view(torch.int32)), \
        "grad_tpc changed where no map reaches"
    assert torch.equal(grad_w[305:].view(torch.int32), pat_w[305:].view(torch.int32)), "grad_w written past entry 305"
    assert torch.equal(grad_w_null[305:].view(torch.int32), pat_w[305:].view(torch.int32))
    r_t = _worst(label + " grad_tpc", grad_tpc, pat_t, ref_t, M_t, KAPPA_TPC)
    r_w = _worst(label + " grad_w", grad_w[:305], pat_w[:305], ref_w, Mw, KAPPA_W)
    r_n = _worst(label + " grad_w, grad_tpc = NULL", grad_w_null[:305], pat_w[:305], ref_w, Mw, KAPPA_W)
    assert r_t <= 1 and r_w <= 1 and r_n <= 1, (r_t, r_w, r_n)
    assert _seen(label + " grad_tpc", ref_t, pat_t, M_t, KAPPA_TPC) > 1, "the bound cannot see the whole gradient"
    assert _seen(label + " grad_w", ref_w, pat_w[:305], Mw, KAPPA_W) > 1, "the bound cannot see the whole gradient"
    for name, sel in (must_see or {}).items():
        part, _, _, _ = tr.reference_gradients(feats.to(DEV, torch.float64), pts_n, tgt_slot_sorted, fs, wts64, geo,
                                               g_sorted * sel[:, None], amax, fb, rm)
        assert _seen(f"{label} grad_tpc, {name} alone", _tpc(part), pat_t, M_t, KAPPA_TPC) > 1, \
            f"the bound cannot see the {name}"
        del part
    print(f"  [{label}] {time.time() - t0:.1f} s")
    return {"ref_t": ref_t, "M_t": M_t, "fb": fb, "amax": amax, "tgt_frame": tgt_frame}


def run_production(label, geo, feats, head, precision, pts, tgt_slot, gout):
    """train.track_forward on a Tracker (the production forward), then check_track_backward."""
    m = _tracker(geo, feats, precision)
    wts = tr.normalized_weights(head, device=DEV)
    emb = _tpc(feats.to(DEV)).contiguous()
    out, hw, saved = dtrain.track_forward(m, emb, *wts, pts.to(DEV), tgt_slot.to(DEV))
    emb, norms, pts_sorted, desc, dn, tgt_sorted, maps, aux, order, slots = saved
    feat = _lib.make_features(emb, norms)
    g_sorted = gout.to(DEV)[order]
    res = check_track_backward(label, feats, slots, pts_sorted, tgt_sorted, wts, geo, g_sorted, maps, aux, feat, m._geom,
                               hw, desc, dn)
    res.update(order=order, aux=aux)
    return res


def _batch(geo, N, B, gen):
    pts = torch.rand(B, 3, generator=gen) * torch.tensor([geo.W - 1.0, geo.H - 1.0, 0.0])
    pts[:, 2] = torch.randint(0, N, (B,), generator=gen).float()
    return pts, torch.randint(0, N, (B,), generator=gen), tr.draw_grad_out(B, gen)


@pytest.mark.parametrize("precision", ["fp16x3", "fp32"])
@pytest.mark.parametrize("kind", ["sharp", "well"])
def test_shipped_shape(kind, precision):
    """The bench.py train_step workload: 476 x 854, N = 4, B = 512, C = 1024."""
    geo = SHIPPED
    feats, _ = synth.shifted_field_features(4, 1024, geo.h, geo.w, seed=101, noise=0.2, max_shift=2)
    gen = _gen("shipped", kind, precision)
    pts, tgt, gout = _batch(geo, 4, 512, gen)
    run_production(f"shipped {kind} {precision}", geo, feats, synth.head_weights(kind, seed=101), precision, pts, tgt, gout)


def test_stability_mix():
    """Stability-branch and normal maps in one launch under a well-conditioned head ("well": logit factor ~50, so the
    bound resolves the branch's dot term, uniform weight and full-frame rows).  8 maps are built to land on the branch:
    their source points lie inside a 4 x 4 block of equal tokens of slot 0 (descriptor s exactly), and target slot 3
    holds s at one token, vectors with negative cosine within 7 tokens of it, and cosine-0.99 copies of s everywhere
    else.  The raw arg-max is the lone token, but the refined logits of the plateau exceed those of the disc by ~16,
    so the disc keeps less than 1e-8 of the softmax.  56 random maps complete the launch (B = 64: every branch map costs
    P x C atomics)."""
    geo = SHIPPED
    h, w = geo.h, geo.w
    N, C, n_fb = 4, 1024, 8
    feats, _ = synth.shifted_field_features(N, C, h, w, seed=103, noise=0.2, max_shift=2)
    gen = _gen("stability")
    r0, c0, ar, ac = 20, 30, 40, 80
    s = feats[0, :, r0, c0].clone()
    feats[0, :, r0 - 1:r0 + 3, c0 - 1:c0 + 3] = s[:, None, None]
    noise = torch.randn(C, h, w, generator=gen)
    noise -= s[:, None, None] * ((s @ noise.reshape(C, -1)) / (s @ s)).reshape(1, h, w)
    noise *= s.norm() / noise.norm(dim=0, keepdim=True)
    frame = s[:, None, None] + 0.14 * noise
    frame[:, ar - 7:ar + 8, ac - 7:ac + 8] = -0.5 * s[:, None, None] + noise[:, ar - 7:ar + 8, ac - 7:ac + 8]
    frame[:, ar, ac] = s
    feats[3] = frame
    hs = geo.patch // 2
    f = torch.rand(n_fb, 2, generator=gen)
    planted = torch.stack([hs + (c0 + f[:, 0]) * geo.stride, hs + (r0 + f[:, 1]) * geo.stride, torch.zeros(n_fb)], 1)
    pts, tgt, gout = _batch(geo, N, 64, gen)
    pts[:n_fb], tgt[:n_fb] = planted, 3
    wanted = torch.zeros(64, dtype=torch.bool)
    wanted[:n_fb] = True
    m = _tracker(geo, feats, "fp16x3")
    wts = tr.normalized_weights(synth.head_weights("well", seed=103), device=DEV)
    emb = _tpc(feats.to(DEV)).contiguous()
    _, hw, saved = dtrain.track_forward(m, emb, *wts, pts.to(DEV), tgt.to(DEV))
    emb, norms, pts_sorted, desc, dn, tgt_sorted, maps, aux, order, slots = saved
    fb = aux[:, 1].bool().cpu()
    planted_sorted = wanted[order.cpu()]
    assert fb[planted_sorted].all(), "the planted maps must take the stability branch"
    assert (~fb).sum() > 0, "normal maps must share the launch"
    assert (aux[:, 0].cpu()[planted_sorted] == ar * w + ac).all()
    check_track_backward("stability mix", feats, slots, pts_sorted, tgt_sorted, wts, geo, gout.to(DEV)[order], maps, aux,
                         _lib.make_features(emb, norms), m._geom, hw, desc, dn,
                         must_see={"stability-branch maps": fb.to(DEV).double()})


def _border_targets(h, w):
    pos = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (0, w // 2), (h - 1, w // 2), (h // 2, 0), (h // 2, w - 1)]
    for d in range(1, 8):
        pos += [(d, w // 2 + 4 * d), (h - 1 - d, w // 2 - 4 * d), (h // 2 + 3 * d, d), (h // 2 - 3 * d, w - 1 - d),
                (d, d), (h - 1 - d, w - 1 - d)]
    return pos


def test_borders():
    """Arg-max planted at the corners, on every border and 1-7 tokens from a border: the disc, the 11 x 11 box and the
    +-8-row window are clipped.  Planted by copying the source token's vector into the target token."""
    geo = SHIPPED
    h, w = geo.h, geo.w
    N = 4
    feats, _ = synth.shifted_field_features(N, 1024, h, w, seed=105, noise=0.2, max_shift=2)
    targets = _border_targets(h, w)
    gen = _gen("borders")
    B = len(targets)
    src_tok = torch.randperm((h - 20) * (w - 20), generator=gen)[:B]
    sr, sc = src_tok // (w - 20) + 10, src_tok % (w - 20) + 10
    tgt = torch.tensor([1 + k % 3 for k in range(B)])
    for k, (r, c) in enumerate(targets):
        feats[tgt[k], :, r, c] = feats[0, :, sr[k], sc[k]]
    hs = geo.patch // 2
    pts = torch.stack([(sc * geo.stride + hs).float(), (sr * geo.stride + hs).float(), torch.zeros(B)], 1)
    gout = tr.draw_grad_out(B, gen)
    res = run_production("borders", geo, feats, synth.head_weights("well", seed=105), "fp16x3", pts, tgt, gout)
    want = torch.tensor([r * w + c for r, c in targets], device=DEV)[res["order"]]
    assert torch.equal(res["amax"], want), "planted arg-max not where the kernel's aux puts it"


def test_clamp():
    """Tokens with |s| |F| just above / below the 1e-8 clamp inside the window of map 2's arg-max: they carry gradient,
    so the clamp branch of the cosine backward runs.  Maps 0 (a zero descriptor) and 1 (zero target tokens around its
    arg-max) have relu(corr) = 0 there, hence zero incoming gradient: they only check that such maps write nothing
    but finite values where they reach."""
    geo = SMALL
    h, w = geo.h, geo.w
    N, C = 4, 256
    feats, _ = synth.shifted_field_features(N, C, h, w, seed=107, noise=0.2, max_shift=2)
    hs = geo.patch // 2
    # map 0: source on zero tokens (every slot: the leak reads them too) -> zero descriptor
    feats[:, :, 4:6, 4:6] = 0
    # map 1: target frame 2 with a block of zero tokens around the (planted) arg-max
    feats[2, :, 10:13, 20:23] = 0
    feats[2, :, 11, 24] = feats[0, :, 15, 8]
    # map 2: tiny source token (slot 0, token (6, 14)); target frame 3: a copy at (14, 20), around it tiny tokens
    v = feats[0, :, 6, 14].clone()
    feats[:, :, 6, 14] = 0
    feats[0, :, 6, 14] = v * (1e-4 / v.norm())
    feats[3, :, 14, 20] = v
    pts = torch.tensor([[4.5 * geo.stride + hs, 4.5 * geo.stride + hs, 0], [8 * geo.stride + hs, 15 * geo.stride + hs, 0],
                        [14 * geo.stride + hs, 6 * geo.stride + hs, 0]], dtype=torch.float32)
    tgt = torch.tensor([1, 2, 3])
    sn = tr.ot.sample_descriptors(feats, tr.sampling_points(pts[2:], geo))[0].double().norm().item()
    gen = _gen("clamp")
    k = 0
    for r in range(12, 17):
        for c in range(17, 24):
            if (r, c) == (14, 20):
                continue
            t = (v + 0.3 * v.norm() / C ** 0.5 * torch.randn(C, generator=gen)).double()
            f = 1e-8 * (1.01 if k % 2 else 0.99) / sn
            feats[3, :, r, c] = (t * (f / t.norm())).float()
            k += 1
    gout = torch.tensor([[0.7, -1.3], [2.0, 0.5], [-3.0, 1.5]])
    res = run_production("clamp", geo, feats, synth.head_weights("well", seed=107), "fp32", pts, tgt, gout)
    fn = feats[3].norm(dim=0).double() * sn
    near = (fn > 0.98e-8) & (fn < 1.02e-8)
    assert int(near.sum()) == k and bool((fn[near] < 1e-8).any()) and bool((fn[near] > 1e-8).any())
    # the clamped tokens carry gradient: they lie in the window of map 2's arg-max
    assert res["ref_t"][3].reshape(h, w, C)[near.to(DEV)].abs().sum() > 0


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5, 7])
def test_sampling_edges(N):
    """Points on exact token centres (zero-weight corners skipped), on the frame border and outside it (border clip),
    source slots 0 and N - 1."""
    geo = SMALL
    feats, _ = synth.shifted_field_features(N, 128, geo.h, geo.w, seed=109 + N, noise=0.2, max_shift=2)
    hs = geo.patch // 2
    xy = [(hs + 3 * geo.stride, hs + 5 * geo.stride), (hs, hs), (geo.W - 1 - hs - 0.0, 40.0), (0.0, 70.0), (geo.W - 1.0, 30.0),
          (90.0, 0.0), (120.0, geo.H - 1.0), (-6.0, 50.0), (geo.W + 9.0, 60.0), (100.0, -5.0), (60.0, geo.H + 11.0),
          (-20.0, -20.0), (geo.W + 3.0, geo.H + 3.0), (hs + 7 * geo.stride, 55.5), (33.3, hs + 2 * geo.stride)]
    pts = torch.tensor([[x, y, float(s)] for x, y in xy for s in sorted({0, N - 1})])
    gen = _gen("edges", N)
    tgt = torch.randint(0, N, (pts.shape[0],), generator=gen)
    gout = tr.draw_grad_out(pts.shape[0], gen)
    run_production(f"sampling edges N={N}", geo, feats, synth.head_weights("well", seed=109), "fp16x3", pts, tgt, gout)


def test_leak_only_tokens():
    """N = 7: slot 1 normalises to 1.0000001, so its samples leak ~1e-7 of weight onto slot 2.  Every map samples
    slot 1 and targets slot 1: tokens of slot 2 get gradient only through the leak."""
    geo = SMALL
    N = 7
    feats, _ = synth.shifted_field_features(N, 128, geo.h, geo.w, seed=111, noise=0.2, max_shift=2)
    gen = _gen("leak")
    B = 24
    pts = torch.rand(B, 3, generator=gen) * torch.tensor([geo.W / 3, geo.H - 1.0, 0.0])
    pts[:, 2] = 1
    tgt = torch.ones(B, dtype=torch.long)
    gout = tr.draw_grad_out(B, gen)
    res = run_production("leak only", geo, feats, synth.head_weights("well", seed=111), "fp16x3", pts, tgt, gout)
    leak = res["ref_t"][2]
    assert (leak != 0).any() and leak.abs().max() < 1e-5 * res["ref_t"][1].abs().max()


def test_frame_map_abi():
    """The C ABI with a non-identity frame set: T = 6 frames, slots -> frames [4, 1, 5, 1] (frame 1 twice), tgt_frame
    given as frames; frames 0, 2, 3 are used by no slot and must stay untouched."""
    geo = SMALL
    T, C, B = 6, 128, 40
    lib = _lib.load()
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=113, noise=0.2, max_shift=2)
    fs = torch.tensor([4, 1, 5, 1], dtype=torch.int32, device=DEV)
    gen = _gen("abi")
    pts, tgt_slot, gout = _batch(geo, 4, B, gen)
    head = synth.head_weights("sharp", seed=113)
    wts = tr.normalized_weights(head, device=DEV)
    geom = _lib.make_geom(geo.H, geo.W)
    emb = _tpc(feats.to(DEV)).contiguous()
    P = geo.P
    norms = torch.empty(T, P, device=DEV)
    st = _lib.stream_ptr()
    _lib.check(lib.dinotrk_token_norms(_lib.ptr(emb), _lib.ptr(norms), T, C, P, st), "token_norms")
    feat = _lib.make_features(emb, norms)
    tf = fs.long()[tgt_slot.to(DEV)]
    order = torch.argsort(tf, stable=True)
    tf_sorted = tf[order].to(torch.int32).contiguous()
    pts_sorted = pts.to(DEV)[order].contiguous()
    desc = torch.empty(B, C, device=DEV)
    dn = torch.empty(B, device=DEV)
    _lib.check(lib.dinotrk_sample_descriptors(_lib.ptr(emb), T, C, ctypes.byref(geom), _lib.ptr(pts_sorted), B, _lib.ptr(fs),
                                              4, 0, _lib.ptr(desc), _lib.ptr(dn), st), "sample_descriptors")
    uniq, counts = torch.unique_consecutive(tf_sorted, return_counts=True)
    row0 = (torch.cumsum(counts, 0) - counts).to(torch.int32)
    grp = torch.stack([uniq.to(torch.int32), row0, counts.to(torch.int32), row0]).contiguous()
    maps = torch.empty(B, lib.dinotrk_map_stride(ctypes.byref(geom)), device=DEV)
    ws_bytes = lib.dinotrk_corr_maps_workspace_bytes(B, int(uniq.shape[0]), C)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    _lib.check(lib.dinotrk_corr_maps(ctypes.byref(feat), ctypes.byref(geom), _lib.ptr(desc), _lib.ptr(dn), _lib.ptr(grp[0]),
                                     _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), int(uniq.shape[0]), B, int(counts.max()),
                                     _lib.ptr(maps), _lib.ptr(ws), ws_bytes, st), "corr_maps")
    hw = dtrain._head_struct(*wts)
    out = torch.empty(B, 2, device=DEV)
    aux = torch.empty(B, 2, device=DEV, dtype=torch.int32)
    _lib.check(lib.dinotrk_head(_lib.ptr(maps), B, ctypes.byref(geom), ctypes.byref(hw), None, _lib.ptr(out), 2, 1, _lib.ptr(aux),
                                None, st), "head")
    slot_sorted = tgt_slot.to(DEV)[order]
    res = check_track_backward("frame map", feats, fs, pts_sorted, slot_sorted, wts, geo, gout.to(DEV)[order], maps, aux, feat,
                               geom, hw, desc, dn)
    assert res["ref_t"][[0, 2, 3]].abs().max() == 0


def test_sample_backward():
    """dinotrk_sample_backward alone at C = 1024: normalised points, some outside [-1, 1], and 4,096 points clustered on
    a few tokens (atomic contention)."""
    geo = SHIPPED
    T, C = 4, 1024
    lib = _lib.load()
    h, w = geo.h, geo.w
    gen = _gen("sample")
    spread = torch.rand(1024, 3, generator=gen) * torch.tensor([2.6, 2.6, 0.0]) - torch.tensor([1.3, 1.3, 0.0])
    spread[:, 2] = torch.randint(0, T, (1024,), generator=gen).float()
    cx = torch.tensor([0.1, -0.5, 0.7])[torch.randint(0, 3, (4096,), generator=gen)]
    cy = torch.tensor([0.2, 0.9, -0.4])[torch.randint(0, 3, (4096,), generator=gen)]
    clustered = torch.stack([cx + 1e-3 * torch.rand(4096, generator=gen), cy + 1e-3 * torch.rand(4096, generator=gen),
                             torch.randint(0, T, (4096,), generator=gen).float()], 1)
    pts = torch.cat([spread, clustered]).to(DEV).contiguous()
    B = pts.shape[0]
    gd = (torch.randn(B, C, generator=gen) * 10.0 ** (torch.rand(B, 1, generator=gen) * 6 - 3)).to(DEV)
    fs = torch.arange(T, dtype=torch.int32, device=DEV)
    leaf = torch.zeros(T, C, h, w, dtype=torch.float64, device=DEV, requires_grad=True)
    (ref,) = torch.autograd.grad(tr.ot.sample_descriptors(leaf, pts, fs), leaf, gd.double())
    M = tr.sample_abs((T, C, h, w), pts, fs, gd)
    ref_t, M_t = _tpc(ref), _tpc(M)
    pat = _pattern(M_t, gen)
    got = pat.clone()
    geom = _lib.make_geom(geo.H, geo.W)
    _lib.check(lib.dinotrk_sample_backward(T, C, ctypes.byref(geom), _lib.ptr(pts), B, _lib.ptr(fs), T, 1, _lib.ptr(gd),
                                           _lib.ptr(got), _lib.stream_ptr()), "sample_backward")
    torch.cuda.synchronize()
    reach = M_t > 0
    assert torch.equal(got[~reach].view(torch.int32), pat[~reach].view(torch.int32))
    assert _worst("sample_backward", got, pat, ref_t, M_t, KAPPA_SAMPLE) <= 1


def test_host_checks_and_empty_batch():
    """B = 0 returns DINOTRK_OK and writes nothing; radius > 5 tokens, a workspace one byte short and a 1080 x 1920 grid
    (5 P floats over the shared memory) return DINOTRK_EINVAL before any launch."""
    lib = _lib.load()
    geo = SMALL
    T, C, B = 2, 64, 4
    feats = synth.random_features(T, C, geo.h, geo.w, seed=115)
    emb = _tpc(feats.to(DEV)).contiguous()
    norms = emb.norm(dim=2).contiguous()
    feat = _lib.make_features(emb, norms)
    hw = dtrain._head_struct(*tr.normalized_weights(synth.head_weights("well")))
    fs = torch.arange(T, dtype=torch.int32, device=DEV)
    pts = torch.zeros(B, 3, device=DEV)
    desc, dn = torch.ones(B, C, device=DEV), torch.ones(B, device=DEV)
    tgt = torch.zeros(B, dtype=torch.int32, device=DEV)
    aux = torch.zeros(B, 2, dtype=torch.int32, device=DEV)
    g = torch.ones(B, 2, device=DEV)
    gw0 = torch.randn(305, device=DEV)
    gt0 = torch.randn(T, geo.P, C, device=DEV)
    geom = _lib.make_geom(geo.H, geo.W)
    maps = torch.zeros(B, lib.dinotrk_map_stride(ctypes.byref(geom)), device=DEV)
    gw, gt = gw0.clone(), gt0.clone()
    assert _backward(feat, geom, hw, pts, fs, desc, dn, tgt, maps, aux, g, gw, gt, B=0) == 0
    assert lib.dinotrk_sample_backward(T, C, ctypes.byref(geom), _lib.ptr(pts), 0, _lib.ptr(fs), T, 1, _lib.ptr(desc), _lib.ptr(gt),
                                       _lib.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.equal(gw, gw0) and torch.equal(gt, gt0)
    n0 = _lib.launch_count()
    far = _lib.make_geom(geo.H, geo.W, radius=42)
    assert _backward(feat, far, hw, pts, fs, desc, dn, tgt, maps, aux, g, gw, gt) == EINVAL
    assert _backward(feat, geom, hw, pts, fs, desc, dn, tgt, maps, aux, g, gw, gt, ws_short=1) == EINVAL
    big = _lib.make_geom(1080, 1920)
    big_maps = torch.zeros(B, lib.dinotrk_map_stride(ctypes.byref(big)), device=DEV)
    assert big.h * big.w * 5 * 4 > 227 * 1024
    assert _backward(feat, big, hw, pts, fs, desc, dn, tgt, big_maps, aux, g, gw, gt) == EINVAL
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0, "an argument error must return before any launch"
    assert torch.equal(gw, gw0) and torch.equal(gt, gt0)

"""Delta-DINO's training node (``train.DeltaTrainFunction``, ``csrc/delta_train.cu``) against float64 autograd.

The reference computation is delta_dino.py:22-61 with BatchNorm on the batch statistics (train) or the running statistics
(eval), and the bilinear alignment of models/utils.py:7-45, evaluated in float64 here (``_cnn64`` restates
``oracle.delta_dino.delta_cnn`` with the float64 BlurPool filter the oracle does not build).

Bars: measured on the H100 and pinned with at least 3x headroom; the worst error measured is written beside each constant.
Errors are relative to the largest entry of the float64 reference tensor.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import delta_dino as od
from oracle import synth
from oracle import tracker as ot
from oracle.tracker import Geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHIPPED = [3, 64, 128, 256, 1024]
# Worst errors measured on an H100 80GB HBM3 at a 400 W power limit; forward_graph (cuDNN fp32) beside them for the record.
FWD_TOL = 5e-5        # residual: 1.65e-5 (cuDNN fp32: 7.0e-6)
RULE_TOL = 1e-6       # running-statistics update on the node's own batch statistics: 5.9e-8
STAT_TOL = 1.5e-4     # batch mean / unbiased variance vs float64, 1 x 34 x 34: 4.4e-5 (they follow the conv outputs)
CANCEL_TOL = 3e-4     # frames 0.5 + 1e-3 noise: residual 9.7e-5 (cuDNN fp32: 9.8e-5), batch statistics 4.0e-5
# (weights / BN tensors, conv biases as described in _check_grads)
TRAIN_TOL = (4e-2, 1e-6)    # train mode, 4 x 476 x 854: 1.25e-2 (cuDNN fp32: 1.06e-2 .. 1.24e-2), 2.5e-7
EVAL_TOL = (2e-3, 2.5e-3)   # eval mode, 4 x 238 x 427: 5.4e-4 (cuDNN fp32: 1.0e-4 .. 1.2e-4), 7.4e-4
STEP_TOL = (1.2e-2, 6e-7)   # whole training step: 3.4e-3, 1.6e-7
WIDE_TOL = (3e-5, 3e-6)     # widths [3, 8, 8, 8, 4096], 1 x 34 x 34: 8.1e-6, 7.5e-7
HEAD_TOL = 2e-5       # refiner gradients through both nodes, relative to the largest: 4.4e-6
XY_TOL = 1e-3
CONV_BIASES = {f"layers.{i}.bias" for i in od.CONV_IDX}


def _report(name, value):
    print(f"[delta-train] {name}: {value:.3e}")


def _sd(chans, seed, last_std=0.01):
    return od.random_state_dict(chans, torch.Generator().manual_seed(seed), last_std=last_std)


def _module(chans, sd, training):
    from dino_tracker_b200.networks import DeltaDINO
    m = DeltaDINO(channels=chans, vit_stride=7).to(DEV)
    m.load_state_dict(sd)
    m.train(training)
    return m


def _vit_hw(H, W):
    return 1 + (H - 14) // 7, 1 + (W - 14) // 7


def _node(m, frames):
    """The module's forward with a graph (frames B x 3 x H x W on the GPU) -> residual B x C x h x w."""
    h, w = _vit_hw(*frames.shape[-2:])
    with torch.enable_grad():
        return m(frames, torch.empty(frames.shape[0], m.channels[-1], h, w, device=DEV))


def _sd64(sd, grad=True):
    out = {}
    for k, v in sd.items():
        if v.dtype.is_floating_point:
            v = v.to(DEV, torch.float64)
            if grad and "running" not in k and "filt" not in k:
                v.requires_grad_(True)
        out[k] = v.to(DEV)
    return out


def _cnn64(frames, sd, bn_training, stats=None):
    """od.delta_cnn in float64; ``stats``: list receiving (batch mean, biased batch var, rows) per layer."""
    x = frames.to(DEV, torch.float64)
    for li, (ci, bi, dil) in enumerate(zip(od.CONV_IDX, od.BN_IDX, od.DILATIONS)):
        pad = 2 * dil
        x = F.conv2d(F.pad(x, (pad,) * 4, mode="reflect"), sd[f"layers.{ci}.weight"], sd[f"layers.{ci}.bias"], dilation=dil)
        if stats is not None:
            stats.append((x.mean(dim=(0, 2, 3)).detach(), x.var(dim=(0, 2, 3), unbiased=False).detach(), x.numel() // x.shape[1]))
        if bn_training:
            x = F.batch_norm(x, None, None, sd[f"layers.{bi}.weight"], sd[f"layers.{bi}.bias"], training=True, eps=od.BN_EPS)
        else:
            x = F.batch_norm(x, sd[f"layers.{bi}.running_mean"], sd[f"layers.{bi}.running_var"], sd[f"layers.{bi}.weight"],
                             sd[f"layers.{bi}.bias"], training=False, eps=od.BN_EPS)
        if li < 3:
            x = torch.relu(x)
            C = x.shape[1]
            x = F.conv2d(F.pad(x, (1, 2, 1, 2), mode="reflect"), sd[f"layers.{ci + 3}.filt"].to(DEV, torch.float64), stride=2,
                         groups=C)
    return x


def _align64(cnn, vit_hw):
    """od.align_cnn_to_vit with the reference's fp32 grid, sampled in float64."""
    vh, vw = vit_hw
    ch, cw = cnn.shape[-2:]
    c_br = [(ch - 1) * 8, (cw - 1) * 8]
    vx = torch.arange(vw, dtype=torch.float32, device=DEV) * 7 + 7.0
    vy = torch.arange(vh, dtype=torch.float32, device=DEV) * 7 + 7.0
    gx, gy = torch.meshgrid(-1.0 - (1.0 / c_br[1]) + (2.0 * vx / c_br[1]), -1 - (1.0 / c_br[0]) + (2.0 * vy / c_br[0]),
                            indexing="xy")
    grid = torch.stack([gx, gy], dim=-1)[None].expand(cnn.shape[0], -1, -1, -1).to(torch.float64)
    return F.grid_sample(cnn, grid, mode="bilinear", padding_mode="border", align_corners=True)


def _residual64(frames, sd64, bn_training, stats=None):
    return _align64(_cnn64(frames, sd64, bn_training, stats), _vit_hw(*frames.shape[-2:]))


def _rel(a, b):
    b = b.to(torch.float64)
    return ((a.to(torch.float64) - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


def _frames(B, H, W, seed):
    return synth.random_video(B, H, W, seed=seed).to(DEV)


def _check_grads(m, sd64, label, tol):
    """Every delta-DINO parameter gradient against float64 autograd: relative to the tensor's largest entry, conv biases
    (mathematically 0 before a train-mode BatchNorm) absolutely, against the scale of the layer's gamma / beta gradients."""
    got = dict(m.named_parameters())
    errs, bias_errs = {}, {}
    for ci, bi in zip(od.CONV_IDX, od.BN_IDX):
        for key in (f"layers.{ci}.weight", f"layers.{bi}.weight", f"layers.{bi}.bias"):
            errs[key] = _rel(got[key].grad, sd64[key].grad)
        key = f"layers.{ci}.bias"
        scale = max(sd64[f"layers.{bi}.weight"].grad.abs().max().item(), sd64[f"layers.{bi}.bias"].grad.abs().max().item())
        bias_errs[key] = (got[key].grad.double() - sd64[key].grad).abs().max().item() / scale
    for k, e in list(errs.items()) + list(bias_errs.items()):
        _report(f"{label} {k}", e)
    assert max(errs.values()) <= tol[0], errs
    assert max(bias_errs.values()) <= tol[1], bias_errs


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [4, 8])
def test_shipped_shape_forward(B):
    import oracle
    H, W = 476, 854
    sd = _sd(SHIPPED, 11 + B)
    frames = _frames(B, H, W, seed=B)
    m = _module(SHIPPED, sd, True)
    res = _node(m, frames).detach()
    with torch.no_grad():
        ref = _residual64(frames, _sd64(sd, grad=False), True)
    e = _rel(res, ref)
    _report(f"forward B={B} node", e)
    oracle.use_exact_fp32()
    g = _module(SHIPPED, sd, True)
    with torch.no_grad():
        eg = _rel(g.forward_graph(frames, _vit_hw(H, W)), ref)
    _report(f"forward B={B} forward_graph (cuDNN fp32)", eg)
    assert e <= FWD_TOL


def test_running_statistics_train_and_eval():
    """Two train-mode calls update the running statistics as torch.nn.BatchNorm2d does; eval mode leaves them alone.

    The update rule is checked on the node's own batch statistics, which a twin module with momentum 1 stores (mean and
    unbiased variance): within RULE_TOL.  Those batch statistics are checked against float64 on maps small enough
    (1 frame of 34 x 34: 1156 .. 25 rows per channel) that writing the biased variance, 1/(n-1) away, fails STAT_TOL at
    every layer -- the test asserts that too."""
    H, W, B = 34, 34, 1
    sd = _sd(SHIPPED, 21)
    m, twin = _module(SHIPPED, sd, True), _module(SHIPPED, sd, True)
    for bi in od.BN_IDX:
        twin.layers[bi].momentum = 1.0
    for call in (1, 2):
        old = {bi: (m.layers[bi].running_mean.double(), m.layers[bi].running_var.double()) for bi in od.BN_IDX}
        frames = _frames(B, H, W, seed=30 + call)
        _node(m, frames)
        _node(twin, frames)
        stats = []
        with torch.no_grad():
            _cnn64(frames, _sd64(sd, grad=False), True, stats)
        rule, batch = 0.0, 0.0
        for li, bi in enumerate(od.BN_IDX):
            bn, tw = m.layers[bi], twin.layers[bi]
            rule = max(rule, _rel(bn.running_mean, 0.9 * old[bi][0] + 0.1 * tw.running_mean.double()),
                       _rel(bn.running_var, 0.9 * old[bi][1] + 0.1 * tw.running_var.double()))
            mean, var, n = stats[li]
            unbiased = var * n / (n - 1)
            batch = max(batch, _rel(tw.running_mean, mean), _rel(tw.running_var, unbiased))
            as_biased = _rel(tw.running_var.double() * (n - 1) / n, unbiased)
            _report(f"call {call} layer {li + 1}: biased variance would be off by", as_biased)
            assert as_biased > STAT_TOL, (li, as_biased)
            assert bn.num_batches_tracked.item() == call and tw.num_batches_tracked.item() == call
        _report(f"running statistics after call {call}: update rule", rule)
        _report(f"running statistics after call {call}: batch statistics vs float64", batch)
        assert rule <= RULE_TOL, call
        assert batch <= STAT_TOL, call
    m.eval()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    _node(m, _frames(B, H, W, seed=40))
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k


def _backward_case(H, W, B, training, seed):
    sd = _sd(SHIPPED, seed)
    frames = _frames(B, H, W, seed=seed + 1)
    h, w = _vit_hw(H, W)
    gr = (torch.randn(B, SHIPPED[-1], h, w, generator=torch.Generator().manual_seed(seed + 2)) * 2.5e-8).to(DEV)
    m = _module(SHIPPED, sd, training)
    res = _node(m, frames)
    assert type(res.grad_fn).__name__ == "DeltaTrainFunctionBackward"
    (res * gr).sum().backward()
    sd64 = _sd64(sd)
    (_residual64(frames, sd64, training) * gr.double()).sum().backward()
    import oracle
    oracle.use_exact_fp32()
    g = _module(SHIPPED, sd, training)
    with torch.enable_grad():
        (g.forward_graph(frames, (h, w)) * gr).sum().backward()
    worst = max(_rel(p.grad, sd64[k].grad) for k, p in g.named_parameters() if k not in CONV_BIASES)
    _report(f"backward {'train' if training else 'eval'} {B}x{H}x{W} forward_graph (cuDNN fp32) worst weight", worst)
    return m, sd64


def test_shipped_shape_backward():
    m, sd64 = _backward_case(476, 854, 4, True, 50)
    _check_grads(m, sd64, "backward train 4x476x854", TRAIN_TOL)


def test_eval_mode_with_gradients():
    m, sd64 = _backward_case(238, 427, 4, False, 60)
    _check_grads(m, sd64, "backward eval 4x238x427", EVAL_TOL)


def test_gradient_scale_invariance_is_exact():
    H, W, B = 98, 126, 2
    chans = [3, 16, 16, 16, 32]
    m = _module(chans, _sd(chans, 70), True)
    res = _node(m, _frames(B, H, W, seed=71))
    params = list(m.parameters())
    gr = torch.randn(res.shape, generator=torch.Generator().manual_seed(72)).to(DEV) * 1e-7
    base = torch.autograd.grad(res, params, grad_outputs=gr, retain_graph=True)
    for k in (-40, -20, 10):
        got = torch.autograd.grad(res, params, grad_outputs=gr * 2.0 ** k, retain_graph=True)
        for a, b in zip(got, base):
            assert torch.equal(a, b * 2.0 ** k), k


def test_forward_backward_is_deterministic():
    H, W, B = 238, 427, 4
    sd = _sd(SHIPPED, 80)
    frames = _frames(B, H, W, seed=81)
    runs = []
    for _ in range(2):
        m = _module(SHIPPED, sd, True)
        res = _node(m, frames)
        gr = torch.randn(res.shape, generator=torch.Generator().manual_seed(82)).to(DEV) * 1e-7
        (res * gr).sum().backward()
        runs.append([res.detach().clone()] + [b.clone() for b in m.buffers()] + [p.grad.clone() for p in m.parameters()])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_batch_statistics_without_cancellation():
    """Frames = 0.5 + 1e-3 noise: conv outputs whose mean is ~1e3 x their spread (E[x^2] - E[x]^2 in fp32 fails here)."""
    H, W, B = 238, 427, 4
    sd = _sd(SHIPPED, 90)
    noise = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(91))
    frames = (0.5 + 1e-3 * noise).to(DEV)
    m = _module(SHIPPED, sd, True)
    for bi in od.BN_IDX:
        m.layers[bi].momentum = 1.0          # running statistics = this batch's statistics
    res = _node(m, frames).detach()
    stats = []
    with torch.no_grad():
        ref = _residual64(frames, _sd64(sd, grad=False), True, stats)
    worst = 0.0
    for li, bi in enumerate(od.BN_IDX):
        mean, var, n = stats[li]
        assert (mean.abs() / var.sqrt()).max().item() > 10 or li > 0
        bn = m.layers[bi]
        worst = max(worst, _rel(bn.running_mean, mean), _rel(bn.running_var.double() * (n - 1) / n, var))
    _report("cancellation: batch statistics", worst)
    e = _rel(res, ref)
    _report("cancellation: residual", e)
    import oracle
    oracle.use_exact_fp32()
    with torch.no_grad():
        eg = _rel(_module(SHIPPED, sd, True).forward_graph(frames, _vit_hw(H, W)), ref)
    _report("cancellation: residual of forward_graph (cuDNN fp32)", eg)
    assert worst <= CANCEL_TOL and e <= CANCEL_TOL


def test_whole_step_through_tracker():
    """config/train.yaml's shape: 4 frames of 476x854, C = 1024, shipped widths, 512 points, Huber loss plus the norm
    regulariser, in train mode, against float64 autograd through the restated delta-DINO and oracle.tracker."""
    from dino_tracker_b200 import Tracker
    geo = Geometry(H=476, W=854)
    T, C, B = 4, 1024, 512
    feats = synth.random_features(T, C, geo.h, geo.w, seed=100)
    feats = feats / feats.norm(dim=1, keepdim=True)
    head = synth.head_weights("well", seed=100)
    sd = _sd(SHIPPED, 101, last_std=0.02)
    video = synth.random_video(T, geo.H, geo.W, seed=102).to(DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=SHIPPED)
    m.tracker_head.load_state_dict(head)
    m.delta_dino.load_state_dict(sd)
    m.train()
    g = torch.Generator().manual_seed(103)
    pts = torch.rand(B, 3, generator=g) * torch.tensor([geo.W - 1.0, geo.H - 1.0, 0.0])
    src, tgt = torch.randint(0, T, (B,), generator=g), torch.randint(0, T, (B,), generator=g)
    labels = (torch.rand(B, 2, generator=g) * 2 - 1).to(DEV)
    fs = torch.arange(T, dtype=torch.int32)
    inp = (pts.to(DEV), src.to(DEV), tgt.to(DEV), fs.to(DEV))
    huber = torch.nn.HuberLoss(delta=1 / 32)
    c = m(inp)
    fn, seen = m.residual_embeddings.grad_fn, set()
    stack = [fn]
    while stack:
        f = stack.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        stack += [n for n, _ in f.next_functions]
    assert any(type(f).__name__ == "DeltaTrainFunctionBackward" for f in seen)
    reg = (m.frame_embeddings.norm(dim=1) / m.raw_embeddings.norm(dim=1) - 1).abs().mean()
    (huber(c, labels) + 1e-4 * reg).backward()

    sd64 = _sd64(sd)
    head64 = {k: v.to(DEV, torch.float64).requires_grad_(True) for k, v in head.items()}
    raw = feats.to(DEV, torch.float64)
    refined = raw + _residual64(video, sd64, True)
    c64 = ot.tracker_forward(refined, (inp[0], inp[1], inp[2], torch.arange(T, dtype=torch.int32, device=DEV)), head64, geo)
    reg64 = (refined.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
    (huber(c64, labels.double()) + 1e-4 * reg64).backward()
    scale = torch.tensor([geo.W - 1, geo.H - 1], device=DEV) / 2
    exy = ((c.detach().double() - c64.detach()).abs() * scale).max().item()
    _report("whole step: coordinates (px)", exy)
    assert exy <= XY_TOL
    _check_grads(m.delta_dino, sd64, "whole step", STEP_TOL)
    # relative to the largest head gradient: d b2 is mathematically 0 (the soft-argmax ignores a constant logit offset)
    head_scale = max(g.grad.abs().max().item() for g in head64.values())
    for k, p in m.tracker_head.named_parameters():
        e = (p.grad.double() - head64[k].grad).abs().max().item() / head_scale
        _report(f"whole step head {k}", e)
        assert e <= HEAD_TOL, k


def test_wide_last_layer():
    """A 4096-channel last layer: legal widths whose input-gradient im2col needs more scratch than the forward's."""
    chans = [3, 8, 8, 8, 4096]
    sd = _sd(chans, 115)
    frames = _frames(1, 34, 34, seed=116)
    m = _module(chans, sd, True)
    res = _node(m, frames)
    gr = torch.randn(res.shape, generator=torch.Generator().manual_seed(117)).to(DEV) * 1e-7
    (res * gr).sum().backward()
    sd64 = _sd64(sd)
    (_residual64(frames, sd64, True) * gr.double()).sum().backward()
    _check_grads(m, sd64, "wide last layer 1x34x34", WIDE_TOL)


def test_routing_by_width():
    frames = _frames(2, 98, 126, seed=110)
    for chans, node in (([3, 4, 4, 4, 32], False), ([3, 8, 8, 8, 32], True)):
        m = _module(chans, _sd(chans, 111), True)
        res = _node(m, frames)
        assert (type(res.grad_fn).__name__ == "DeltaTrainFunctionBackward") == node, chans


def test_abi_argument_errors_launch_nothing():
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    B, H, W, h, w = 2, 98, 126, 13, 17
    chans = [3, 8, 8, 8, 32]
    ch = (ctypes.c_int * 5)(*chans)
    frames = _frames(B, H, W, seed=121)
    buf = lambda n: torch.zeros(max(n, 1), device=DEV, dtype=torch.uint8)
    saved_b, fws_b = lib.dinotrk_delta_train_saved_bytes(B, H, W, ch), lib.dinotrk_delta_train_forward_workspace_bytes(B, H, W, ch)
    bws_b = lib.dinotrk_delta_train_backward_workspace_bytes(B, H, W, ch)
    saved, fws, bws = buf(saved_b), buf(fws_b), buf(bws_b)
    v = lambda n, val=0.0: torch.full((n,), val, device=DEV)
    his = [torch.zeros(c, 208, device=DEV, dtype=torch.float16) for c in chans[1:]]
    vecs = [v(c, 1.0) for c in chans[1:]]
    arr = lambda ts: (ctypes.c_void_p * 4)(*[t.data_ptr() if t is not None else None for t in ts])
    ixs, iys = v(w), v(h)
    res = v(B * h * w * 32, 7.0)
    grads = [v(c * 208, 7.0) for c in chans[1:]]

    def fwd(Bn=B, Hn=H, Wn=W, chn=ch, fr=frames, wts=his, sb=saved_b, wb=fws_b):
        return lib.dinotrk_delta_train_forward(_lib.ptr(fr), Bn, Hn, Wn, chn, arr(wts), arr(his), arr(vecs), arr(vecs), arr(vecs),
                                               arr(vecs), arr(vecs), 1, 0.1, 1e-5, _lib.ptr(ixs), _lib.ptr(iys), h, w,
                                               _lib.ptr(res), _lib.ptr(saved), sb, _lib.ptr(fws), wb, _lib.stream_ptr())

    def bwd(Bn=B, Hn=H, Wn=W, chn=ch, wb=bws_b):
        return lib.dinotrk_delta_train_backward(_lib.ptr(frames), Bn, Hn, Wn, chn, arr(his), arr(his), arr(vecs), arr(vecs), 1,
                                                _lib.ptr(ixs), _lib.ptr(iys), h, w, _lib.ptr(res), _lib.ptr(saved), saved_b,
                                                arr(grads), arr(vecs), arr(vecs), arr(vecs), _lib.ptr(bws), wb, _lib.stream_ptr())
    n0 = _lib.launch_count()
    assert fwd(fr=None) == -22
    assert fwd(wts=[his[0], None, his[2], his[3]]) == -22
    assert fwd(chn=(ctypes.c_int * 5)(3, 8, 12, 8, 32)) == -22          # not a multiple of 8
    assert fwd(sb=saved_b - 1) == -22 and fwd(wb=fws_b - 1) == -22      # short buffers
    assert fwd(Hn=28, Wn=40) == -22                                     # layer 4's map is 4 rows: too small for pad 4
    assert bwd(wb=bws_b - 1) == -22 and bwd(chn=(ctypes.c_int * 5)(3, 8, 8, 8, 36)) == -22
    assert _lib.launch_count() == n0
    assert fwd(Bn=0) == 0 and bwd(Bn=0) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert (res == 7.0).all() and all((g == 7.0).all() for g in grads)

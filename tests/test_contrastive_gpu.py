"""GPU suite: the best-buddy contrastive node (dinotrk_bb_contrastive_forward / _backward) and the drop-in losses
(dino_tracker_b200/contrastive.py) against float64 autograd through the oracle (oracle/contrastive.py).  Each test prints
the node's error next to fp32 torch's (cuBLAS, TF32 off) on the same inputs; the bars hold at least 3x the node's error
measured on an H100."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import contrastive as oc
from oracle import make_golden_contrastive as mg

pytestmark = pytest.mark.gpu

DEV = "cuda"


def smooth_frames(N, C, h, w, seed, noise=0.05):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    freq = torch.rand(C, 2, generator=g) * 0.3
    phase = torch.rand(C, generator=g) * 6.28
    fr = [torch.sin(freq[:, 0, None, None] * (xx + 1.3 * i) + freq[:, 1, None, None] * yy + phase[:, None, None])
          + noise * torch.randn(C, h, w, generator=g) for i in range(N)]
    return torch.stack(fr)


def tok(x):
    return x.reshape(x.shape[0], x.shape[1], -1).transpose(1, 2).contiguous()


def oracle_node(E, S, U, groups, tau):
    """Per group the oracle's get_bb_pairs_contrastive_loss: (cl1 [B], cl2 [B], bb_mean [G], c_mean [G])."""
    B = S.shape[0]
    cl1 = torch.zeros(B, dtype=E.dtype, device=E.device)
    cl2 = torch.zeros(B, dtype=E.dtype, device=E.device)
    bbm, cm = [], []
    for s, t, r0, n in groups:
        a, b, m1, m2 = oc.get_bb_pairs_contrastive_loss(None, S[r0:r0 + n], U[r0:r0 + n], E[s], E[t], temp=tau)
        cl1 = cl1.index_put((torch.arange(r0, r0 + n, device=E.device),), a)
        cl2 = cl2.index_put((torch.arange(r0, r0 + n, device=E.device),), b)
        bbm.append(m1)
        cm.append(m2)
    return cl1, cl2, torch.stack(bbm), torch.stack(cm)


def run_both(E, S, U, groups, tau, seed=0):
    """Outputs and gradients of the node, of fp32 torch and of float64 torch under the same random upstream gradients."""
    from dino_tracker_b200.contrastive import bb_contrastive
    g = torch.Generator(device=DEV).manual_seed(seed)
    B, G = S.shape[0], len(groups)
    ups = [torch.randn(B, device=DEV, generator=g), torch.randn(B, device=DEV, generator=g),
           torch.randn(G, device=DEV, generator=g), torch.randn(G, device=DEV, generator=g)]
    res = {}
    for name, dt in (("node", torch.float32), ("fp32", torch.float32), ("f64", torch.float64)):
        x = [t.detach().to(dt).clone().requires_grad_(True) for t in (E, S, U)]
        outs = bb_contrastive(*x, groups, tau) if name == "node" else oracle_node(*x, groups, tau)
        torch.autograd.backward(list(outs), [u.to(dt) for u in ups])
        res[name] = [o.detach().double() for o in outs] + [t.grad.double() for t in x]
    return res


NAMES = ["cl1", "cl2", "bb_mean", "c_mean", "dE", "dS", "dU"]


def rel_errors(res, which):
    out = {}
    for k, a, b in zip(NAMES, res[which], res["f64"]):
        assert torch.equal(a.isnan(), b.isnan()), k        # the mean of an empty group is NaN, as in torch
        ok = ~b.isnan()
        out[k] = float((a[ok] - b[ok]).abs().max() / b[ok].abs().max().clamp_min(1e-30))
    return out


def check(res, bars, label):
    node, ref = rel_errors(res, "node"), rel_errors(res, "fp32")
    for k in NAMES:
        print(f"{label} {k}: node {node[k]:.2e}  fp32 torch {ref[k]:.2e}  bar {bars[k]:.0e}")
    for k in NAMES:
        assert node[k] <= bars[k], (label, k, node[k], bars[k])


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def shipped_inputs(seed=0):
    N, C, h, w = 4, 1024, 67, 121
    E = tok(smooth_frames(N, C, h, w, seed)).to(DEV)
    P = h * w
    g = torch.Generator().manual_seed(seed + 1)
    groups = [(0, 1, 0, 256), (2, 2, 256, 256), (3, 0, 512, 256), (1, 3, 768, 256)]
    S, U = [], []
    for s, t, _, n in groups:
        S.append(E[s][torch.randint(P, (n,), generator=g).to(DEV)])
        U.append(E[t][torch.randint(P, (n,), generator=g).to(DEV)])
    return E, torch.cat(S), torch.cat(U), groups


# max error / max |value| against float64, measured on an H100 (node | fp32 torch): cl1 3.5e-6 | 1.1e-7, cl2 3.5e-6 | 9.9e-8,
# bb_mean 3.9e-8 | 3.9e-8, c_mean 6.3e-6 | 8.4e-8, dE 2.2e-5 | 3.4e-6, dS 9.2e-6 | 5.3e-7, dU 6.4e-6 | 4.6e-7
BARS_SHIPPED = {"cl1": 1.5e-5, "cl2": 1.5e-5, "bb_mean": 2e-7, "c_mean": 2e-5, "dE": 1e-4, "dS": 3e-5, "dU": 3e-5}


# small shapes with clamped / zero / duplicate rows and with more groups than frames, measured at most: cl1 2.3e-7,
# cl2 2.5e-7, bb_mean 9.8e-8, c_mean 3.3e-7, dE 1.5e-6, dS 1.5e-6, dU 1.5e-6
BARS_CLAMPED = {"cl1": 1e-6, "cl2": 1e-6, "bb_mean": 4e-7, "c_mean": 1e-6, "dE": 5e-6, "dS": 5e-6, "dU": 5e-6}


def test_node_shipped_shape_against_float64():
    E, S, U, groups = shipped_inputs()
    check(run_both(E, S, U, groups, 0.1), BARS_SHIPPED, "shipped")


def test_node_clamped_zero_and_duplicate():
    N, C, h, w = 3, 64, 13, 17
    E = tok(smooth_frames(N, C, h, w, 3)).to(DEV)
    P = h * w
    E[1, 5] = 0.0                       # a zero token: every cosine against it hits the clamp
    E[2, 7] = E[2, 8]                   # duplicate tokens
    g = torch.Generator().manual_seed(4)
    groups = [(0, 1, 0, 20), (2, 2, 20, 12), (1, 0, 32, 0), (1, 2, 32, 10)]   # a self-pair and an empty group
    S = E[0][torch.randint(P, (42,), generator=g).to(DEV)].clone()
    U = E[1][torch.randint(P, (42,), generator=g).to(DEV)].clone()
    S[20:32] = E[2][7]                  # the duplicate token as every source of the self-pair
    U[20:32] = E[2][8]
    S[3] = 0.0                          # zero descriptors: bb and every row cosine clamped
    U[35] = 0.0
    S[5] *= 1e-10                       # non-zero but clamped: |S_5| |E_n| ~ 6e-9 < 1e-8 for every token
    check(run_both(E, S, U, groups, 0.1), BARS_CLAMPED, "clamped")


def test_node_more_groups_than_frames():
    """Six pairs over a frame set of two (more groups than frames + 1): the workspace queries cover the group tables."""
    N, C, h, w = 2, 64, 13, 17
    E = tok(smooth_frames(N, C, h, w, 11)).to(DEV)
    P = h * w
    g = torch.Generator().manual_seed(12)
    groups = [(0, 1, 0, 20), (1, 0, 20, 20), (0, 0, 40, 20), (1, 1, 60, 20), (0, 1, 80, 7), (1, 0, 87, 13)]
    S = E[0][torch.randint(P, (100,), generator=g).to(DEV)]
    U = E[1][torch.randint(P, (100,), generator=g).to(DEV)]
    check(run_both(E, S, U, groups, 0.1), BARS_CLAMPED, "groups > frames")


def test_node_determinism_and_power_of_two_invariance():
    from dino_tracker_b200.contrastive import bb_contrastive
    E, S, U, groups = shipped_inputs(seed=5)
    g = torch.Generator(device=DEV).manual_seed(1)
    ups = [torch.randn(S.shape[0], device=DEV, generator=g) for _ in range(2)] + \
          [torch.randn(len(groups), device=DEV, generator=g) for _ in range(2)]

    def run(scale):
        x = [(t * scale).clone().requires_grad_(True) for t in (E, S, U)]
        outs = bb_contrastive(*x, groups, 0.1)
        torch.autograd.backward(list(outs), ups)
        return [o.detach() for o in outs], [t.grad for t in x]
    o1, g1 = run(1.0)
    o2, g2 = run(1.0)
    for a, b in zip(o1 + g1, o2 + g2):
        assert torch.equal(a, b)
    o3, g3 = run(2.0 ** 5)
    for a, b in zip(o1[:3], o3[:3]):
        assert torch.equal(a, b)
    for a, b in zip(g1, g3):
        assert torch.equal(a, b * 2.0 ** 5)


def test_node_argument_errors_and_empty():
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    N, P, C, B = 2, 100, 12, 4
    E = torch.zeros(N, P, C, device=DEV)
    S = torch.zeros(B, C, device=DEV)
    cos = torch.zeros(2 * B, 104, device=DEV)
    out = torch.zeros(7, B, device=DEV)
    ws = torch.zeros(1 << 20, device=DEV, dtype=torch.uint8)
    before = _lib.launch_count()

    def fwd(C_, grp, nbytes=ws.numel()):
        g = torch.tensor(grp, dtype=torch.int32).reshape(-1, 4).t().contiguous()
        return lib.dinotrk_bb_contrastive_forward(_lib.ptr(E), N, P, C_, _lib.ptr(S), _lib.ptr(S), B,
                                                  *(ctypes.c_void_p(g[i].data_ptr()) for i in range(4)), g.shape[1], 0.1,
                                                  _lib.ptr(cos), _lib.ptr(out), _lib.ptr(ws), nbytes, _lib.stream_ptr())
    assert fwd(12, [(0, 1, 0, 4)]) == -22                 # C not a multiple of 8
    assert fwd(8, [(0, 2, 0, 4)]) == -22                  # slot out of range
    assert fwd(8, [(0, 1, 2, 4)]) == -22                  # rows out of range
    assert fwd(8, [(0, 1, 0, 4)], nbytes=16) == -22       # short workspace
    assert fwd(8, [(0, 1, 0, 0)]) == 0                    # only empty groups: nothing to do
    assert _lib.launch_count() == before

    g_row = torch.zeros(B, device=DEV)
    g_grp = torch.zeros(1, device=DEV)
    dS = torch.zeros(B, 8, device=DEV)
    dE = torch.zeros(N, P, 8, device=DEV)

    def bwd(C_, grp, nbytes=None):
        g = torch.tensor(grp, dtype=torch.int32).reshape(-1, 4).t().contiguous()
        gp = [ctypes.c_void_p(g[i].data_ptr()) for i in range(4)]
        q = lib.dinotrk_bb_contrastive_backward_workspace_bytes(N, P, C_, B, *gp, g.shape[1])
        rc = lib.dinotrk_bb_contrastive_backward(_lib.ptr(E), N, P, C_, _lib.ptr(S), _lib.ptr(S), B, *gp, g.shape[1], 0.1,
                                                 _lib.ptr(cos), _lib.ptr(out), _lib.ptr(g_row), _lib.ptr(g_row), _lib.ptr(g_grp),
                                                 _lib.ptr(g_grp), _lib.ptr(dS), _lib.ptr(dS), _lib.ptr(dE), _lib.ptr(ws),
                                                 ws.numel() if nbytes is None else nbytes, _lib.stream_ptr())
        return q, rc
    assert bwd(12, [(0, 1, 0, 4)]) == (0, -22)            # C not a multiple of 8: the query reports 0
    assert bwd(8, [(0, 2, 0, 4)]) == (0, -22)             # slot out of range
    assert bwd(8, [(0, 1, 2, 4)]) == (0, -22)             # rows out of range
    q, _ = bwd(8, [(0, 1, 0, 4)], nbytes=0)
    assert q > 0 and bwd(8, [(0, 1, 0, 4)], nbytes=q - 1)[1] == -22   # one byte short
    assert _lib.launch_count() == before


def test_dropin_losses_empty_selection_return_zero_without_launch():
    from dino_tracker_b200 import _lib
    from dino_tracker_b200 import contrastive as c
    cfg = dict(mg.CONFIG)
    tr = type("T", (), {})()
    tr.config = cfg
    tr.fg_masks = torch.zeros(4, 98, 126)
    tr.dino_bb_pairs = {f"{s}_{t}": {"source_coords": None, "target_coords": None} for s in range(4) for t in range(4)}
    model = oc.ModelStandIn(torch.zeros(4, 3, 98, 126), torch.randn(4, 32, 13, 17, device=DEV))
    before = _lib.launch_count()
    loss = c.get_dino_bb_contrastive_loss(tr, model, torch.arange(4))
    assert float(loss) == 0.0 and _lib.launch_count() == before
    # refined loss: best buddies, but 0 points per pair -> every selection empty, no node launch
    calls = []
    orig = c.BBContrastiveFunction.apply
    c.BBContrastiveFunction.apply = lambda *a: calls.append(a) or orig(*a)
    try:
        loss = c.get_refined_bb_contrastive_loss(tr, model, torch.arange(4), model.frame_embeddings, 4, 0, 0.7, 0.1, 900)
    finally:
        c.BBContrastiveFunction.apply = orig
    assert float(loss) == 0.0 and not calls


def fixture_setup():
    z = np.load(mg.OUT)
    emb = torch.from_numpy(z["emb"])
    tr = mg.trainer_standin(type("T", (), {}), torch.from_numpy(z["masks"]), mg.load_bb(z))
    video = torch.zeros(mg.T, 3, *z["video_hw"].tolist())
    return z, emb, tr, video


@pytest.mark.parametrize("which", ["dino", "refined"])
def test_dropin_losses_reproduce_fixture(which):
    from dino_tracker_b200 import contrastive as c
    z, emb0, tr, video = fixture_setup()
    seed = int(z[f"{which}_seed"])
    fs = torch.from_numpy(z["frames"])
    cfg = mg.CONFIG
    emb = emb0.to(DEV).requires_grad_(True)
    model = oc.ModelStandIn(video, emb, stride=mg.STRIDE)
    kw = dict(batch_size=cfg["cl_n_frames"], points_per_pair=cfg["cl_points_per_pair"], fg_points_ratio=cfg["cl_fg_points_ratio"])
    torch.manual_seed(seed)
    if which == "dino":
        drawn = c.draw_dino_bb_pairs(tr, model, fs)
        pairs = np.array([(s, t, len(sel)) for s, t, sel, _ in drawn])
        src = np.concatenate([sel.numpy() for _, _, sel, _ in drawn])
        tgt = src
    else:
        drawn = c.draw_refined_pairs(tr, model, fs, emb, **kw)
        pairs = np.array([(s, t, len(a)) for s, t, a, _, _ in drawn])
        src = np.concatenate([a.cpu().numpy() for _, _, a, _, _ in drawn])
        tgt = np.concatenate([b.cpu().numpy() for _, _, _, b, _ in drawn])
    assert np.array_equal(pairs, z[f"{which}_pairs"])
    assert np.array_equal(src, z[f"{which}_src"]) and np.array_equal(tgt, z[f"{which}_tgt"])
    torch.manual_seed(seed)
    if which == "dino":
        loss = c.get_dino_bb_contrastive_loss(tr, model, fs)
    else:
        loss = c.get_refined_bb_contrastive_loss(tr, model, fs, emb, temp=cfg["cl_temp"], cl_div=cfg["cl_div_ref_bb"], **kw)
    loss.backward()
    ref_loss = float(z[f"{which}_loss"])
    ref_grad = torch.from_numpy(z[f"{which}_grad"]).to(DEV)
    le = abs(loss.item() - ref_loss) / abs(ref_loss)
    ge = float((emb.grad - ref_grad).abs().max() / ref_grad.abs().max())
    print(f"fixture {which}: loss rel err {le:.2e}, grad rel err {ge:.2e}")
    assert le <= 1e-5 and ge <= 5e-5   # measured: loss 3.1e-7, gradient 7.5e-6 (refined)


def test_search_self_pairs_duplicates_and_rescaled():
    from dino_tracker_b200.contrastive import refined_best_buddies
    N, C, h, w = 3, 64, 13, 17
    H, W = (h - 1) * 7 + 14, (w - 1) * 7 + 14
    fr = smooth_frames(N, C, h, w, 9, noise=0.2)
    fr[1, :, 2, 3] = fr[1, :, 4, 5]                      # duplicate tokens
    pairs = [(0, 1), (1, 1), (2, 2), (2, 0)]
    for scale in (1.0, 3e5):                             # 3e5: outside the fp16 split's range (the rescaled path)
        emb = (fr * scale).to(DEV)
        mutual, partner, cos_at = refined_best_buddies(emb, pairs, H, W)
        for k, (s, t) in enumerate(pairs):
            a, b = tok(emb.double())[s], tok(emb.double())[t]
            m64, p64, aff = oc.refined_best_buddies(a, b)
            top2 = aff.topk(2, dim=1).values
            clear = (top2[:, 0] - top2[:, 1]) >= 2e-4      # float64 arg-max gap at least delta_bb
            clear_t = aff.topk(2, dim=0).values
            clear_t = (clear_t[0] - clear_t[1]) >= 2e-4
            ok = clear & clear_t[p64]
            assert torch.equal(partner[k][ok], p64[ok]), (s, t, scale)
            assert torch.equal(mutual[k][ok], m64[ok]), (s, t, scale)
            assert torch.allclose(cos_at[k][ok].double(), aff[torch.arange(aff.shape[0], device=DEV), p64][ok], atol=1e-5)
        # self-pair: every token with a unique maximum is its own best buddy
        own = torch.arange(h * w, device=DEV)
        uniq = torch.ones(h * w, dtype=torch.bool, device=DEV)
        uniq[[2 * w + 3, 4 * w + 5]] = False
        assert torch.equal(partner[1][uniq], own[uniq]) and bool(mutual[1][uniq].all())


# measured on an H100: total loss 7.8e-8, parameter gradients 6.4e-5 to 7.1e-5, dino-BB term 1e-7, refined term 1.1e-4 against float64
# (fp32 torch: 6.5e-7).  The refined term is dominated by self-pair rows, where loss = lse - bb / tau ~ 0.3 is a
# difference of two numbers near 10: the node's absolute cosine error (~4e-6 at C = 1024, wgmma accumulation) shows
# there relative to a small result.
ITER_LOSS_TOL, ITER_GRAD_TOL, ITER_TERM_TOL = 5e-7, 2.5e-4, 3.5e-4


def test_whole_training_iteration_dropin_against_torch_losses():
    """dino_tracker.py:405-427 after iteration 5000 at train.yaml's shape (4 frames of 476 x 854, C = 1024, shipped
    delta-DINO widths, 512 tracked points, both contrastive terms with 4 pairs x 256 points): the drop-in Tracker in train
    mode, once with the library's contrastive losses and once with the oracle's torch losses on the same draws (the
    oracle's refined loss takes the library's arg-max through its ``search`` hook, so near-ties pick the same buddies).
    Total loss and every delta-DINO and refiner parameter gradient.  The cycle-consistency term is left out: it is the same
    model code on both sides and has its own fixture test."""
    from test_delta_train_gpu import SHIPPED, _sd
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200 import contrastive as c
    from oracle import synth
    H, W, T, C, B = 476, 854, 4, 1024, 512
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    feats = synth.random_features(T, C, h, w, seed=200)
    video = synth.random_video(T, H, W, seed=201).to(DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=SHIPPED)
    m.tracker_head.load_state_dict(synth.head_weights("well", seed=202))
    m.delta_dino.load_state_dict(_sd(SHIPPED, 203, last_std=0.02))
    m.train()
    cfg = dict(mg.CONFIG, cl_points_per_pair=256, lambda_cl_dino_bb=0.00025, lambda_cl_ref_bb=0.00005,
               lambda_emb_norm=0.0001, lambda_angle=0.0001)
    g = torch.Generator().manual_seed(204)
    masks = torch.zeros(T, H, W)
    masks[:, 120:360, 250:600] = 1
    coords = oc.get_vit_feature_coords_from_mask(H, W, 7, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                n = 1500
                bb[f"{s}_{t}"] = {"source_coords": coords[torch.randperm(h * w, generator=g)[:n]],
                                  "target_coords": coords[torch.randint(h * w, (n,), generator=g)],
                                  "cos_sims": torch.rand(n, generator=g) * 0.6 + 0.4, "r": torch.rand(n, generator=g) * 0.4}
    tr = type("Trainer", (), {})()
    tr.config, tr.fg_masks, tr.dino_bb_pairs = cfg, masks, bb
    pts = torch.rand(B, 3, generator=g) * torch.tensor([W - 1.0, H - 1.0, 0.0])
    src, tgt = torch.randint(0, T, (B,), generator=g), torch.randint(0, T, (B,), generator=g)
    labels = (torch.rand(B, 2, generator=g) * 2 - 1).to(DEV)
    fs = torch.arange(T, device=DEV)
    inp = (pts.to(DEV), src.to(DEV), tgt.to(DEV), fs)
    huber = torch.nn.HuberLoss(delta=1 / 32, reduction="none")

    def iteration(lib):
        m.zero_grad()
        coords_pred = m(inp)
        loss = huber(coords_pred, labels).mean()
        emb = m.frame_embeddings
        torch.manual_seed(205)
        kw = dict(batch_size=cfg["cl_n_frames"], points_per_pair=cfg["cl_points_per_pair"],
                  fg_points_ratio=cfg["cl_fg_points_ratio"], temp=cfg["cl_temp"], cl_div=cfg["cl_div_ref_bb"])
        if lib:
            ref_l = c.get_refined_bb_contrastive_loss(tr, m, fs, emb, **kw)
        else:
            def search(s, t):
                mutual, partner, _ = c.refined_best_buddies(emb, [(s, t)], H, W)
                return mutual[0], partner[0]
            ref_l = oc.get_refined_bb_contrastive_loss(tr, m, fs, emb, search=search, **kw)
        loss = loss + cfg["lambda_cl_ref_bb"] * ref_l
        dino_l = (c if lib else oc).get_dino_bb_contrastive_loss(tr, m, fs)
        raw = m.raw_embeddings
        norm_reg = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
        angle_reg = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
        loss = loss + cfg["lambda_cl_dino_bb"] * dino_l + cfg["lambda_emb_norm"] * norm_reg + cfg["lambda_angle"] * angle_reg
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in list(m.delta_dino.named_parameters()) +
                 [("head." + k, p) for k, p in m.tracker_head.named_parameters()]}
        if not lib:   # the refined term once more in float64 on the same draws
            torch.manual_seed(205)
            emb64 = emb.detach().double()
            ref64 = oc.get_refined_bb_contrastive_loss(tr, m, fs, emb64, search=search, **kw).item()
        return loss.item(), ref_l.item(), dino_l.item(), grads, (ref64 if not lib else None)

    lib = iteration(True)
    ref = iteration(False)
    print(f"iteration: refined term vs float64: library {abs(lib[1] - ref[4]) / abs(ref[4]):.2e}, "
          f"fp32 torch {abs(ref[1] - ref[4]) / abs(ref[4]):.2e}")
    assert ref[1] != 0.0 and ref[2] != 0.0, "both contrastive terms must be active"
    le = abs(lib[0] - ref[0]) / abs(ref[0])
    print(f"iteration: total loss {lib[0]:.6g} vs {ref[0]:.6g} (rel {le:.2e}); refined {lib[1]:.6g} vs {ref[1]:.6g}; "
          f"dino-BB {lib[2]:.6g} vs {ref[2]:.6g}")
    scale = max(v.abs().max().item() for v in ref[3].values())
    worst = 0.0
    for k, v in ref[3].items():
        e = (lib[3][k] - v).abs().max().item() / max(v.abs().max().item(), 1e-3 * scale)
        worst = max(worst, e)
    print(f"iteration: worst parameter gradient error {worst:.2e} (relative to the tensor's largest entry)")
    assert abs(lib[1] - ref[4]) <= ITER_TERM_TOL * abs(ref[4]) and abs(lib[2] - ref[2]) <= ITER_TERM_TOL * abs(ref[2])
    assert le <= ITER_LOSS_TOL and worst <= ITER_GRAD_TOL

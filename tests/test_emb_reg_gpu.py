"""The embedding regularisers as one CUDA node (``train.RegularisersFunction``, csrc/emb_reg.cu) against float64 torch
of the reference's expressions (dino_tracker.py:136-146, models/utils.py:79-84).

Bars: both scalars within 1e-6 relative; dE within 2e-3 of the float64 gradient's largest entry (the training-step bar of
test_train_gpu.py).  At |x - 1|'s kink (E == R, as at iteration -1 of a fresh run) both terms' own gradients are
rounding noise, so there dE is held to 2e-3 of the gradient ONE active term gives, g / (nP) max_p |E_p|_inf / (a b):
a node that let the norm term through at its kink would miss it by 500 times.
"""
import pytest
import torch

from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REL = 1e-6
GRAD_TOL = 2e-3
G_NORM, G_ANGLE = 0.75, -1.25      # upstream gradients (the sign of g_angle exercises both branches of each term)


def _inputs(n, P, C, seed):
    g = torch.Generator().manual_seed(seed)
    R = torch.randn(n, P, C, generator=g)
    scale = 1 + 0.3 * torch.randn(n, P, 1, generator=g)
    E = R * scale + 0.4 * torch.randn(n, P, C, generator=g)
    return E.to(DEV), R.to(DEV)


def _ref64(E, R):
    """float64 norm_reg, angle_reg and dE of G_NORM * norm_reg + G_ANGLE * angle_reg, through the chw views the
    reference reads."""
    n, P, C = E.shape
    e = E.double().view(n, P, 1, C).permute(0, 3, 1, 2).detach().requires_grad_(True)
    r = R.double().view(n, P, 1, C).permute(0, 3, 1, 2)
    a, b = e.norm(dim=1), r.norm(dim=1)
    norm_reg = (a / b - 1).abs().mean()
    angle_reg = (torch.einsum("bchw,bchw->bhw", e, r) / (a * b) - 1).abs().mean()
    (G_NORM * norm_reg + G_ANGLE * angle_reg).backward()
    return norm_reg.item(), angle_reg.item(), e.grad.permute(0, 2, 3, 1).reshape(n, P, C)


def _node(E, R):
    from dino_tracker_b200.train import RegularisersFunction
    e = E.detach().clone().requires_grad_(True)
    norm_reg, angle_reg = RegularisersFunction.apply(e, R)
    (G_NORM * norm_reg + G_ANGLE * angle_reg).backward()
    torch.cuda.synchronize()
    return norm_reg, angle_reg, e.grad


def _rel(x, ref):
    return abs(x - ref) / abs(ref)


# (n, P, C): train.yaml's frame set (4 frames of 67 x 121 tokens, ViT-L's 1024), a narrow and a ViT-g width, and
# P = 37 x 29 = 1073, not a multiple of 32
SHAPES = [(4, 67 * 121, 1024), (3, 221, 32), (2, 500, 1536), (3, 37 * 29, 64)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_node_matches_float64(shape):
    E, R = _inputs(*shape, seed=sum(shape))
    n_ref, a_ref, g_ref = _ref64(E, R)
    norm_reg, angle_reg, dE = _node(E, R)
    assert _rel(norm_reg.item(), n_ref) <= REL, (norm_reg.item(), n_ref)
    assert _rel(angle_reg.item(), a_ref) <= REL, (angle_reg.item(), a_ref)
    err = (dE.double() - g_ref).abs().max().item() / g_ref.abs().max().item()
    assert err <= GRAD_TOL, err


def _one_term_scale(E, R, g):
    a, b = E.double().norm(dim=-1), R.double().norm(dim=-1)
    return (g / E[..., 0].numel() * E.double().abs().amax(dim=-1) / (a * b)).max().item()


def _check_kink(E, R):
    norm_reg, angle_reg, dE = _node(E, R)
    assert norm_reg.item() == 0.0
    assert abs(angle_reg.item()) <= 1e-6
    # what autograd gives in the reference's own precision, and in float64
    e = E.detach().clone().requires_grad_(True)
    emb, raw = e.view(*E.shape[:2], 1, E.shape[2]).permute(0, 3, 1, 2), R.view(*R.shape[:2], 1, R.shape[2]).permute(0, 3, 1, 2)
    nr = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
    ar = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
    (G_NORM * nr + G_ANGLE * ar).backward()
    _, _, g64 = _ref64(E, R)
    bar = GRAD_TOL * _one_term_scale(E, R, max(abs(G_NORM), abs(G_ANGLE)))
    assert (dE - e.grad).abs().max().item() <= bar
    assert (dE.double() - g64).abs().max().item() <= bar


def test_kink_equal_embeddings():
    _, R = _inputs(4, 67 * 121, 1024, seed=11)
    _check_kink(R.clone(), R)


def test_kink_fresh_delta_dino_through_tracker_forward():
    """A fresh delta-DINO (zero last convolution) in train mode adds exactly 0: frame_embeddings == raw_embeddings."""
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200.train import token_rows
    H, W, T, C = 98, 126, 4, 32
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    model = Tracker(video=synth.random_video(T, H, W, seed=3).to(DEV), dino_embed_video=synth.random_features(T, C, h, w, seed=4),
                    device=DEV, delta_channels=[3, 8, 8, 8, C])
    model.train()
    g = torch.Generator().manual_seed(5)
    B = 16
    pts = (torch.rand(B, 3, generator=g) * torch.tensor([W - 1.0, H - 1.0, 0.0])).to(DEV)
    inp = (pts, torch.randint(0, T, (B,), generator=g).to(DEV), torch.randint(0, T, (B,), generator=g).to(DEV),
           torch.arange(T, dtype=torch.int32, device=DEV))
    model(inp)
    E, R = token_rows(model.frame_embeddings), token_rows(model.raw_embeddings)
    assert torch.equal(E, R)
    _check_kink(E.detach(), R)


def test_bit_identical_runs():
    E, R = _inputs(4, 67 * 121, 1024, seed=21)
    first = _node(E, R)
    second = _node(E, R)
    for x, y in zip(first, second):
        assert torch.equal(x, y)


def test_rejects_width_not_multiple_of_4():
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.train import RegularisersFunction
    lib = _lib.load()
    n, P, C = 2, 40, 6
    E, R = _inputs(n, P, C, seed=1)
    out = torch.empty(2, device=DEV)
    aux = torch.empty(n * P, 3, device=DEV)
    ws_bytes = lib.dinotrk_emb_reg_workspace_bytes(n, P)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    st = _lib.stream_ptr()
    assert lib.dinotrk_emb_reg_forward(_lib.ptr(E), _lib.ptr(R), n, P, C, _lib.ptr(out), _lib.ptr(aux), _lib.ptr(ws), ws_bytes,
                                       st) == -22   # DINOTRK_EINVAL
    g = torch.ones((), device=DEV)
    dE = torch.empty_like(E)
    assert lib.dinotrk_emb_reg_backward(_lib.ptr(E), _lib.ptr(R), n, P, C, _lib.ptr(aux), _lib.ptr(g), _lib.ptr(g), _lib.ptr(dE),
                                        st) == -22
    with pytest.raises(_lib.DinotrkError):
        RegularisersFunction.apply(E.requires_grad_(True), R)
    with pytest.raises(ValueError):
        RegularisersFunction.apply(E, R.clone().requires_grad_(True))


def test_shipped_layout_reads_embeddings_in_place():
    """The training forward's frame_embeddings / raw_embeddings are token-major in memory: the node reads them through
    views, without a copy."""
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200.train import token_rows
    from oracle import delta_dino as od
    H, W, T, C = 98, 126, 6, 64
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    chans = [3, 8, 8, 8, C]
    model = Tracker(video=synth.random_video(T, H, W, seed=6).to(DEV), dino_embed_video=synth.random_features(T, C, h, w, seed=7),
                    device=DEV, delta_channels=chans)
    model.delta_dino.load_state_dict(od.random_state_dict(chans, torch.Generator().manual_seed(8), last_std=0.1))
    model.train()
    B = 8
    inp = (torch.zeros(B, 3, device=DEV) + 20, torch.zeros(B, dtype=torch.long, device=DEV),
           torch.ones(B, dtype=torch.long, device=DEV), torch.tensor([1, 3, 4, 5], dtype=torch.int32, device=DEV))
    model(inp)
    for emb in (model.frame_embeddings, model.raw_embeddings):
        rows = token_rows(emb)
        assert rows.is_contiguous() and rows.data_ptr() == emb.data_ptr()
        assert rows.contiguous().data_ptr() == emb.data_ptr()

"""GPU tests: every stage of a ViT block on its own (dinotrk_vit_stage, the forward's own launch code) at the widths and
token counts the project ships, against float64 computed from the same fp16 operands the kernel reads.

Shapes.  One 854x476 frame (67 x 121 tokens + cls: N1 = 8108 rows) and two frames per call (16216 rows = 63 x 256 + 88:
the rank-1 CTA of the last CTA-pair tile has no valid row; with one frame it has 44).  Widths ViT-S/14 (384, 6 heads:
a 128-column N tail in qkv, proj and fc2), ViT-B/14 (768, 12), ViT-L/14 (1024, 16) and ViT-g/14 (1536, 24).  At these
sizes every CTA of the persistent GEMMs runs several tiles, so the ring's stage / phase carried from tile to tile and the
producer running into the next tile during the epilogue are exercised, in CTA-pair and in single-CTA mode.

Bounds.  With the operand rounding taken out of the comparison, what remains is the fp32 tensor-core accumulation, the
fp32 epilogue and the output rounding.  A GEMM stage with reference c = sum_k a_k w_k (+ bias, position embedding) is
held to
    |got - ref| <= gamma(K) * (sum_k |a_k w_k| + |bias| (+ |pos|)) * |scale| + r
where r is half an fp16 ulp of the output for fp16 outputs (q, k, v^T, h; taken at the larger of |got| and |ref|, so that
a result rounded across a power of two is covered) and half an fp32 ulp of the updated residual stream for proj / fc2,
whose check is x_new - x_old against ls * (acc + bias).  gamma(K) covers the accumulation over K and the two or three
fp32 operations of the epilogue; its constant is measured and pinned with headroom (GAMMA_C below).  fc1 adds the erf
fit of the GELU (1.5e-7, Abramowitz-Stegun 7.1.26) and its fp32 evaluation, times 0.5 |v|, and |gelu'(v)| times the
accumulation term.  LayerNorm is held to its derived fp32 rounding bound (see test_layernorm_stage).  For fp16 outputs
the printed worst error / bound sits just under 1 by construction: the output rounding alone reaches half an ulp.

Every output buffer is filled with NaN first: slots the stage must write are checked to be finite, slots it must leave
alone (the cls row under the patch embedding, the v^T padding columns, rows past B * N1) to still be NaN.  CTA-pair and
single-CTA runs issue the same wgmma sequence per output row, so their results must be bit-identical."""
import ctypes
import math
import zlib

import pytest
import torch

from dino_tracker_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FRAME_H, FRAME_W = 476, 854
N1 = 67 * 121 + 1                 # tokens per frame incl. cls
P = N1 - 1
KP = 592                          # 3 * 14 * 14 = 588 rounded up to 8: the last 64-wide K block holds 16 columns
WIDTHS = {"vits14": (384, 6), "vitb14": (768, 12), "vitl14": (1024, 16), "vitg14": (1536, 24)}
LAYERNORM, PATCH, QKV, PROJ, FC1, FC2 = range(6)   # DINOTRK_VIT_* of include/dinotrk.h
U24 = 2.0 ** -24
# Accumulation + epilogue constant of the GEMM stages: GAMMA(K) = GAMMA_C sqrt(K) 2^-23.  The fp32 tensor-core
# accumulation rounds once per K step on partial sums of size ~sqrt(K) (random-sign operands), so what the data needs
# grows like sqrt(K) relative to sum |a w|.  Measured on an H100 80GB HBM3 (400 W power limit) over every stage and shape of
# this file: at most 0.150 sqrt(K) 2^-23 (patch 0.150, fc2 0.143, proj 0.133, qkv 0.083, fc1 0.074; e.g. 10.8 x 2^-23 for
# ViT-g fc2 at K = 6144); pinned at 0.5, over 3x headroom.
GAMMA_C = 0.5
GELU_ERF = 1.5e-7 + 2.0 ** -21    # erf fit + its fp32 evaluation (rcp.approx, ex2.approx, five FMAs)
QSCALE = 0.125 * float(torch.tensor(1.4426950408889634, dtype=torch.float32))   # the kernel's fp32 64^-1/2 log2(e)
CANARY = 512                      # rows past the output that must stay NaN

shapes = pytest.mark.parametrize("width,frames", [(w, f) for w in WIDTHS for f in (1, 2)])


def _half_ulp(t, mant_bits, min_exp):
    """Half an ulp of |t| in a binary format with `mant_bits` stored significand bits and smallest normal 2^min_exp."""
    _, e = torch.frexp(t.double().abs())
    e = torch.where(t == 0, torch.full_like(e, min_exp + 1), e.clamp_min(min_exp + 1))
    return torch.ldexp(torch.ones_like(t, dtype=torch.float64), e - 2 - mant_bits)


def half_ulp16(t):
    return _half_ulp(t, 10, -14)


def half_ulp32(t):
    return _half_ulp(t, 23, -126)


def _stage(stage, dim, heads, frames, inp, w=None, p0=None, p1=None, outs=(), pair=True):
    lib = _lib.load()
    cfg = _lib.VitConfig(1, dim, heads, 0, 14, 7, 0, 1, 1 if pair else 0)
    geom = _lib.make_geom(FRAME_H, FRAME_W)
    assert geom.h * geom.w + 1 == N1
    ws = torch.empty(4096, dtype=torch.uint8, device=DEV)
    o = list(outs) + [None] * (3 - len(outs))
    _lib.check(lib.dinotrk_vit_stage(stage, ctypes.byref(cfg), ctypes.byref(geom), frames, _lib.ptr(inp), _lib.ptr(w),
                                     _lib.ptr(p0), _lib.ptr(p1), _lib.ptr(o[0]), _lib.ptr(o[1]), _lib.ptr(o[2]), _lib.ptr(ws),
                                     ws.numel(), _lib.stream_ptr()), "vit_stage")
    torch.cuda.synchronize()


def _gemm64(a16, w16):
    """float64 a . w^T and |a| . |w|^T from the fp16 operands."""
    a, w = a16.double(), w16.double()
    return a @ w.T, a.abs() @ w.abs().T


def gamma(K):
    return GAMMA_C * math.sqrt(K) * 2.0 ** -23


def _check(label, got, ref, bound, K=None, acc_scale=None, rest=None):
    """Every element within its bound; prints the worst error / bound and, for GEMM stages, the accumulation constant
    the data needed (error beyond `rest` over the accumulation scale, in units of sqrt(K) 2^-23)."""
    got = got.double()
    assert torch.isfinite(got).all(), f"{label}: {int((~torch.isfinite(got)).sum())} outputs not written or not finite"
    err = (got - ref).abs()
    ratio = (err / bound).max().item()
    msg = f"[{label}] worst error / bound = {ratio:.4f}"
    if K is not None:
        seen = ((err - rest).clamp_min(0) / acc_scale.clamp_min(1e-30)).max().item() / gamma(K) * GAMMA_C
        msg += f", accumulation constant seen = {seen:.3f} (pinned {GAMMA_C:g}) x sqrt({K}) 2^-23"
    print(msg)
    assert ratio <= 1.0, msg


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _randn(g, *shape, std=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * std


def _bits_equal(a, b):
    """torch.equal on the bit patterns (NaN canaries included)."""
    iv = torch.int16 if a.element_size() == 2 else torch.int32
    return torch.equal(a.view(iv), b.view(iv))


@shapes
def test_layernorm_stage(width, frames):
    """fp16 LayerNorm of the fp32 residual stream (warp per row, the row in registers) against float64
    (x - mu) / sqrt(var + 1e-6) * w + b.  Every fifth row carries a common offset around 1e3, every fifth (another) one
    channel around +-1e4 -- the very large channels of DINOv2 residual streams.  The bound is the kernel's fp32 rounding,
    derived: the row sum runs D / 128 + 2 additions deep per lane plus a 5-level warp tree, so
    |mu~ - mu| <= d u mean|x| with d = D / 128 + 8, u = 2^-24; the variance adds d u relative and the shift error
    squared, rsqrtf two ulps; the output a few more roundings, then half an fp16 ulp."""
    D, heads = WIDTHS[width]
    rows = frames * N1
    g = _gen("ln", D, frames)
    x = _randn(g, rows, D)
    x[1::5] += 1e3 * (1 + 0.1 * torch.rand(x[1::5].shape[0], 1, generator=g, device=DEV))
    sel = torch.arange(3, rows, 5, device=DEV)
    ch = torch.randint(0, D, (sel.numel(),), generator=g, device=DEV)
    x[sel, ch] = 1e4 * torch.sign(_randn(g, sel.numel()))
    gw = 1 + _randn(g, D, std=0.2)
    gb = _randn(g, D, std=0.1)
    y = _nan(rows + CANARY, D, dtype=torch.half)
    _stage(LAYERNORM, D, heads, frames, x, None, gw, gb, (y,))
    got = y[:rows]

    x64, w64, b64 = x.double(), gw.double(), gb.double()
    mu = x64.mean(1, keepdim=True)
    xc = x64 - mu
    rstd = 1.0 / torch.sqrt((xc * xc).mean(1, keepdim=True) + 1e-6)
    ref = xc * rstd * w64 + b64
    d = D // 128 + 8
    dmu = d * U24 * x64.abs().mean(1, keepdim=True)
    t = (xc * rstd * w64).abs()
    bound = (U24 * ((d + 8) * t + b64.abs()) + w64.abs() * rstd * dmu + t * (dmu * rstd) ** 2
             + half_ulp16(torch.maximum(ref.abs(), got.double().abs())))
    _check(f"layernorm {width} x{frames}", got, ref, bound)
    assert y[rows:].isnan().all(), "LayerNorm wrote rows past B * N1"


@shapes
def test_patch_embedding_stage(width, frames):
    """Patch GEMM (K = 592, 16 live columns in the last K block) + bias + position embedding into x[b][1 + p]; the cls
    row x[b][0] and the rows past the call stay untouched."""
    D, heads = WIDTHS[width]
    g = _gen("patch", D, frames)
    cols = ((torch.rand(frames * P, KP, generator=g, device=DEV) - 0.45) / 0.225).half()   # ImageNet-normalised pixels
    w = _randn(g, D, KP, std=588 ** -0.5).half()
    bias = _randn(g, D, std=0.05)
    pos = _randn(g, P, D, std=0.1)
    x = _nan(frames * N1 + CANARY, D)
    _stage(PATCH, D, heads, frames, cols, w, bias, pos, (x,))
    acc, aabs = _gemm64(cols, w)
    pos_all = pos.double().repeat(frames, 1)
    ref = acc + bias.double() + pos_all
    scale = aabs + bias.double().abs() + pos_all.abs()
    xv = x[:frames * N1].view(frames, N1, D)
    _check(f"patch {width} x{frames}", xv[:, 1:].reshape(frames * P, D), ref, gamma(KP) * scale, KP, scale, 0.0)
    assert xv[:, 0].isnan().all(), "the patch embedding wrote the cls row"
    assert x[frames * N1:].isnan().all(), "the patch embedding wrote rows past the call"


def _heads_major(t, frames, heads):
    """[frames * N1][heads * 64] -> [frames * heads][N1][64]"""
    return t.reshape(frames, N1, heads, 64).permute(0, 2, 1, 3).reshape(frames * heads, N1, 64)


@shapes
def test_qkv_stage(width, frames):
    """qkv GEMM with the fused-attention scatter: q (x 64^-1/2 log2 e), k [b][head][n][64] and v^T [b][head][64][n] with
    row pitch N1 rounded up to 8 (8112: four padding columns that must stay unwritten), fp16."""
    D, heads = WIDTHS[width]
    rows, BH, N1p8 = frames * N1, frames * heads, (N1 + 7) // 8 * 8
    g = _gen("qkv", D, frames)
    y = _randn(g, rows, D).half()
    w = _randn(g, 3 * D, D, std=D ** -0.5).half()
    bias = _randn(g, 3 * D, std=0.05)
    res = {}
    for pair in (True, False):
        q, k = _nan(BH * N1 * 64 + CANARY, dtype=torch.half), _nan(BH * N1 * 64 + CANARY, dtype=torch.half)
        vT = _nan(BH * 64 * N1p8 + CANARY, dtype=torch.half)
        _stage(QKV, D, heads, frames, y, w, bias, None, (q, k, vT), pair)
        res[pair] = (q, k, vT)
    acc, aabs = _gemm64(y, w)
    ref, scale = acc + bias.double(), aabs + bias.double().abs()
    refs = {"q": (_heads_major(ref[:, :D], frames, heads) * QSCALE, _heads_major(scale[:, :D], frames, heads) * QSCALE),
            "k": (_heads_major(ref[:, D:2 * D], frames, heads), _heads_major(scale[:, D:2 * D], frames, heads)),
            "v": (_heads_major(ref[:, 2 * D:], frames, heads).transpose(1, 2), _heads_major(scale[:, 2 * D:], frames, heads).transpose(1, 2))}
    for pair, (q, k, vT) in res.items():
        mode = "pair" if pair else "single"
        vv = vT[:BH * 64 * N1p8].view(BH, 64, N1p8)
        got = {"q": q[:BH * N1 * 64].view(BH, N1, 64), "k": k[:BH * N1 * 64].view(BH, N1, 64), "v": vv[:, :, :N1]}
        for name in ("q", "k", "v"):
            r, s = refs[name]
            r16 = half_ulp16(torch.maximum(r.abs(), got[name].double().abs()))
            _check(f"qkv.{name} {width} x{frames} {mode}", got[name], r, gamma(D) * s + r16, D, s, r16)
        assert vv[:, :, N1:].isnan().all(), "v^T padding columns written"
        assert q[BH * N1 * 64:].isnan().all() and k[BH * N1 * 64:].isnan().all() and vT[BH * 64 * N1p8:].isnan().all()
    for a, b, name in zip(res[True], res[False], "qkv"):
        assert _bits_equal(a, b), f"qkv.{name}: CTA-pair and single-CTA results differ"


def _residual_case(stage, width, frames):
    D, heads = WIDTHS[width]
    K = D if stage == PROJ else 4 * D
    rows = frames * N1
    g = _gen("residual", stage, D, frames)
    if stage == PROJ:      # attention output: convex combinations of v rows
        a = _randn(g, rows, K, std=0.5).half()
    else:                  # GELU output
        a = torch.nn.functional.gelu(_randn(g, rows, K)).half()
    w = _randn(g, D, K, std=K ** -0.5).half()
    bias = _randn(g, D, std=0.05)
    ls = _randn(g, D, std=0.3)
    x0 = _nan(rows + CANARY, D)
    x0[:rows] = _randn(g, rows, D)           # a missing read-before-write shows up against these
    out = {}
    for pair in (True, False):
        x = x0.clone()
        _stage(stage, D, heads, frames, a, w, bias, ls, (x,), pair)
        out[pair] = x
    acc, aabs = _gemm64(a, w)
    ls64 = ls.double()
    ref = ls64 * (acc + bias.double())
    scale = ls64.abs() * (aabs + bias.double().abs())
    label = "proj" if stage == PROJ else "fc2"
    for pair, x in out.items():
        xn = x[:rows].double()
        r = half_ulp32(xn)
        _check(f"{label} {width} x{frames} {'pair' if pair else 'single'}", xn - x0[:rows].double(), ref, gamma(K) * scale + r,
               K, scale, r)
        assert x[rows:].isnan().all(), f"{label} wrote rows past B * N1"
    assert _bits_equal(out[True], out[False]), f"{label}: CTA-pair and single-CTA results differ"


@shapes
def test_proj_stage(width, frames):
    """proj GEMM (K = D) + bias, LayerScale and the residual add into the fp32 stream."""
    _residual_case(PROJ, width, frames)


@shapes
def test_fc2_stage(width, frames):
    """fc2 GEMM (K = 4 D: 4096 for ViT-L, 6144 for ViT-g) + bias, LayerScale and the residual add."""
    _residual_case(FC2, width, frames)


@shapes
def test_fc1_stage(width, frames):
    """fc1 GEMM + bias + exact GELU (erf by the 1.5e-7 fit) to fp16; the coalesced epilogue (single CTA) and the
    thread-per-row one (CTA pairs) must agree bit for bit."""
    D, heads = WIDTHS[width]
    rows = frames * N1
    g = _gen("fc1", D, frames)
    y = _randn(g, rows, D).half()
    w = _randn(g, 4 * D, D, std=D ** -0.5).half()
    bias = _randn(g, 4 * D, std=0.05)
    out = {}
    for pair in (True, False):
        h = _nan(rows + CANARY, 4 * D, dtype=torch.half)
        _stage(FC1, D, heads, frames, y, w, bias, None, (h,), pair)
        out[pair] = h
    acc, aabs = _gemm64(y, w)
    v = acc + bias.double()
    ref = 0.5 * v * (1 + torch.special.erf(v / math.sqrt(2)))
    dgelu = 0.5 * (1 + torch.special.erf(v / math.sqrt(2))) + v * torch.exp(-0.5 * v * v) / math.sqrt(2 * math.pi)
    scale = dgelu.abs() * (aabs + bias.double().abs())
    for pair, h in out.items():
        got = h[:rows]
        rest = 0.5 * v.abs() * GELU_ERF + half_ulp16(torch.maximum(ref.abs(), got.double().abs()))
        _check(f"fc1 {width} x{frames} {'pair' if pair else 'single'}", got, ref, gamma(D) * scale + rest, D, scale, rest)
        assert h[rows:].isnan().all(), "fc1 wrote rows past B * N1"
    assert _bits_equal(out[True], out[False]), "fc1: CTA-pair and single-CTA results differ"

"""GPU: the int8 coarse pass of the anchor phase (csrc/xwin.cu, tcgemm.cuh TcMode::S8).

The coarse values only decide which exact values get computed, so the int8 pass must (1) quantise exactly as specified
(include/dinotrk.h: dinotrk_quantise_s8), (2) produce the keys of its own int8 operands -- maximum, first token holding it,
second value -- and (3) stay within the per-map bound eps it reports of the exact cosine.  End to end, forcing either coarse
pass or the full-map pipeline gives the same trajectories and occlusion masks bit for bit, and a video whose features carry outlier channels runs the
fp16 pass in the automatic mode."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import synth
from oracle.tracker import Geometry

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 128
HERE = os.path.dirname(os.path.abspath(__file__))


def _keys_module():
    spec = importlib.util.spec_from_file_location("coarse_keys_cases", os.path.join(HERE, "test_coarse_keys_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _outliers(x, n_ch=4, scale=30.0, axis=-1):
    """A few channels `scale` times larger than the rest (the channel outliers of some ViT features)."""
    x = x.copy()
    idx = [slice(None)] * x.ndim
    idx[axis] = slice(0, n_ch)
    x[tuple(idx)] *= scale
    return x


def _quant_ref(x):
    """numpy reference of dinotrk_quantise_s8 on rows of x (float32): q, s, fac, rho64 (unrounded)."""
    x = x.astype(np.float32)
    mx = np.abs(x).max(-1)
    s = (mx / np.float32(127)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(s[..., None] > 0, np.clip(np.rint(x / s[..., None]), -127, 127), 0).astype(np.int8)
    norm = np.sqrt((x.astype(np.float64) ** 2).sum(-1))
    res = np.sqrt(((x.astype(np.float64) - s[..., None].astype(np.float64) * q) ** 2).sum(-1))
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = np.where(norm > 0, res / norm, 0.0)
    return q, s, norm, rho


def _quantise(x_np, rows_per_group):
    from dino_tracker_b200 import _lib
    x = torch.from_numpy(x_np).to(DEV)
    norms = x.norm(dim=-1).contiguous()
    q, fac, rho, rho_max = _lib.quantise_s8(x, norms, rows_per_group, _lib.stream_ptr())
    torch.cuda.synchronize()
    return x, norms, q, fac, rho, rho_max


@pytest.mark.parametrize("kind", ["gauss", "outlier"])
def test_quantiser_matches_numpy(kind):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((3, 700, 256), dtype=np.float32)
    if kind == "outlier":
        x = _outliers(x)
    x[1, 17] = 0.0                                   # a zero row: q = 0, rho = 0
    x[2, 3] = 0.0
    x[2, 3, 9] = -2.5                                # a one-hot row: q = -127 at channel 9, 0 elsewhere
    _, norms, q, fac, rho, rho_max = _quantise(x, 700)
    rq, s, _, rrho = _quant_ref(x)
    assert np.array_equal(q.cpu().numpy(), rq)
    nf = norms.cpu().numpy()
    assert np.array_equal(fac.cpu().numpy(), (s / np.maximum(nf, np.float32(1e-4))).astype(np.float32))
    g = rho.cpu().numpy().astype(np.float64)
    assert (g >= rrho).all(), "rho not rounded up"
    up = np.nextafter(rrho.astype(np.float32), np.float32(np.inf)).astype(np.float64)
    assert (g <= up).all(), "rho more than one float above its float64 value"
    assert g[1, 17] == 0.0 and rq[2, 3, 9] == -127 and not rq[2, 3, :9].any()
    assert np.array_equal(rho_max.cpu().numpy(), rho.cpu().numpy().max(1))


def _run_keys_i8(cs):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    h, w = cs["hw"]
    g = _lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
    P = cs["P"]
    feats, norms, fq, ffac, _, frho = _quantise(cs["feats"], P)
    desc, dnorm, dq, dfac, drho, _ = _quantise(cs["desc"], cs["desc"].shape[0])
    fs = _lib.make_features(feats, norms, quant=(fq, ffac, frho))
    gf, gr, gm = (torch.from_numpy(cs[k]).to(DEV) for k in ("frame", "row0", "m"))
    rows, n_groups = desc.shape[0], len(cs["m"])
    key1 = torch.zeros((rows, cs["n_tiles"]), dtype=torch.int64, device=DEV)
    max2 = torch.zeros((rows, cs["n_tiles"]), dtype=torch.float32, device=DEV)
    eps = torch.full((rows,), -1.0, dtype=torch.float32, device=DEV)
    nb = lib.dinotrk_xw_coarse_keys_workspace_bytes(cs["T"], n_groups, ctypes.byref(g))
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    _lib.check(lib.dinotrk_xw_coarse_keys_i8(ctypes.byref(fs), ctypes.byref(g), _lib.ptr(dq), _lib.ptr(dfac), _lib.ptr(drho), rows,
                                             _lib.ptr(gf), _lib.ptr(gr), _lib.ptr(gm), n_groups, _lib.ptr(key1), _lib.ptr(max2),
                                             _lib.ptr(eps), _lib.ptr(ws), nb, _lib.stream_ptr()), "xw_coarse_keys_i8")
    torch.cuda.synchronize()
    return dict(key1=key1.cpu().numpy(), max2=max2.cpu().numpy(), eps=eps.cpu().numpy(), feats=feats, norms=norms, fq=fq,
                ffac=ffac, desc=desc, dnorm=dnorm, dq=dq, dfac=dfac)


CASES = {   # name: (make_case arguments of test_coarse_keys_gpu, outlier channels)
    "gauss_c1024": ((11, (67, 121), 3, 1024, (1, 255, 256, 257, 655), (0, 1, 2, 1, 0)), False),
    "gauss_odd_c64": ((14, (13, 25), 4, 64, (257, 255, 1, 655, 256), (1, 2, 3, 0, 2)), False),
    "outlier_c1024": ((13, (13, 25), 4, 1024, (655, 1, 257, 256, 255), (3, 0, 1, 2, 3)), True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_int8_keys_match_int_reference_and_bound(name):
    """Every case holds exact duplicate tokens (test_coarse_keys_gpu's construction): the key must name the first one."""
    args, outl = CASES[name]
    cs = _keys_module().make_case(*args)
    if outl:
        cs["feats"] = _outliers(cs["feats"])
        cs["desc"] = _outliers(cs["desc"])
    r = _run_keys_i8(cs)
    key1, max2, eps = r["key1"], r["max2"], r["eps"]
    P, nt = cs["P"], cs["n_tiles"]
    kmax = (key1.view(np.uint64) >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    ktok = 0x7FFFFFFF - (key1.view(np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)
    fq, dq = r["fq"].double(), r["dq"].double()           # integer products are exact in float64 (C 127^2 < 2^53)
    ffac, dfac = r["ffac"].double(), r["dfac"].double()
    fx, dx = r["feats"].double(), r["desc"].double()
    fn, dn = r["norms"].double(), r["dnorm"].double()
    tiles = np.arange(nt)[None, :]
    n_dup = 0
    for r0, m, f in zip(cs["row0"], cs["m"], cs["frame"]):
        sl = slice(int(r0), int(r0 + m))
        ints = dq[sl] @ fq[f].T
        coarse = ints * dfac[sl, None] * ffac[f][None, :]                         # the pass's values (pre-ReLU)
        exact = (dx[sl] @ fx[f].T) / (dn[sl, None] * fn[f][None, :]).clamp_min(1e-8)
        # the bound the plan relies on, for every token of every map
        gap = (coarse.clamp_min(0) - exact.clamp_min(0)).abs().max(1).values.cpu().numpy()
        assert (eps[sl] > 0).all() and (gap <= eps[sl]).all(), (gap.max(), eps[sl].min())
        pad = torch.full((m, nt * TILE - P), -np.inf, dtype=torch.float64, device=DEV)
        v = torch.cat([coarse, pad], 1).view(m, nt, TILE).cpu().numpy()
        iv = torch.cat([ints, pad], 1).view(m, nt, TILE).cpu().numpy()
        srt = -np.sort(-v, axis=2)
        top1, top2 = srt[..., 0], srt[..., 1]
        km, kt, k2 = kmax[sl], ktok[sl], max2[sl].astype(np.float64)
        tol = 4 * 2.0 ** -24 * np.maximum(np.abs(top1), 1.0)                     # a few fp32 roundings of the epilogue
        assert np.abs(km - np.maximum(top1, 0)).max() <= tol.max(), "tile maximum off"
        assert np.abs(k2 - np.maximum(top2, 0)).max() <= tol.max(), "second value off"
        first = v.argmax(axis=2) + tiles * TILE
        sure = top1 - top2 > 2 * tol
        assert (kt[sure] == first[sure]).all(), "token is not the first arg-max of a clear tile maximum"
        # exact duplicates holding the maximum: identical int8 rows and factors, so an exact tie -> the first token
        isrt = -np.sort(-iv, axis=2)
        tie = (isrt[..., 0] == isrt[..., 1]) & (top1 == top2) & (top1 > 0.5)
        assert (kt[tie] == first[tie]).all() and (k2[tie] == km[tie]).all(), "exact tie not resolved to the first token"
        n_dup += int(tie.sum())
    assert n_dup >= len(cs["m"])


def _tracker(feats, head, geo):
    from dino_tracker_b200 import ModelInference, Tracker
    T = feats.shape[0]
    m = Tracker(video=torch.zeros(T, 3, geo.H, geo.W, device=DEV), dino_embed_video=feats, device=DEV,
                delta_channels=[3, 4, 4, 4, feats.shape[1]])
    m.tracker_head.load_state_dict(head)
    return ModelInference(m, m.range_normalizer, 0.7, 0.6)


def _infer(mi, q, path, coarse):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    try:
        assert lib.dinotrk_infer_set_path(path) == 0 and lib.dinotrk_infer_set_coarse(coarse) == 0
        r = mi.infer_all(q.to(DEV))
        torch.cuda.synchronize()
        stats = _lib.infer_stats()
    finally:
        lib.dinotrk_infer_set_path(-1)
        lib.dinotrk_infer_set_coarse(-1)
    return {k: v.clone() for k, v in r.items()}, stats


def _same(a, b):
    """traj / occ / cos_sims bit for bit.  Anchor points to the parity bar: a map the looser int8 bound queues is finished by
    the full-map head instead of the exact-window head, whose softmax sums differ in the last bits (test_xwin_gpu.py)."""
    for k in ("traj", "occ", "cos_sims"):
        assert torch.equal(a[k], b[k]), k
    vis = a["cos_sims"] >= 0.7
    assert (a["anchors"][vis] - b["anchors"][vis]).abs().max().item() <= 1e-3


@pytest.mark.parametrize("kind", ["sharp", "well"])
@pytest.mark.parametrize("geo,T,C", [(Geometry(H=98, W=126), 5, 32), (Geometry(), 6, 128), (Geometry(), 9, 256)])
def test_int8_pass_matches_fp16_pass_and_full_map(geo, T, C, kind):
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=7 + T, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=T)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=14.0, jitter_seed=T)
    mi = _tracker(feats, head, geo)
    s8, st8 = _infer(mi, q, 1, 1)
    f16, st16 = _infer(mi, q, 1, 0)
    full, st0 = _infer(mi, q, 0, -1)
    auto, sta = _infer(mi, q, -1, -1)
    print(f"[{geo.h}x{geo.w} T={T} C={C} {kind}] int8 {st8} | fp16 {st16}")
    assert st8["pipeline"] == "exact-window" and st8["coarse"] == "int8" and st16["coarse"] == "fp16"
    assert st0["pipeline"] == "full-map"
    assert 0 < st8["coarse_rho_f"] <= 0.03 and sta["coarse"] == "int8"
    _same(s8, f16)
    _same(s8, full)
    _same(s8, auto)


def test_outlier_channels_select_fp16_pass():
    geo, T, C = Geometry(), 6, 256
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=31, noise=0.2, max_shift=2)
    feats = torch.from_numpy(_outliers(feats.numpy(), axis=1))
    head = synth.head_weights("well", seed=3)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=14.0, jitter_seed=3)
    mi = _tracker(feats, head, geo)
    auto, sta = _infer(mi, q, -1, -1)
    s8, st8 = _infer(mi, q, 1, 1)
    print(f"[outlier channels] auto {sta} | int8 forced {st8}")
    assert sta["pipeline"] == "exact-window" and sta["coarse"] == "fp16" and sta["coarse_rho_f"] > 0.03
    assert st8["coarse"] == "int8"
    _same(auto, s8)


def test_probe_queue_switches_to_fp16_pass():
    """Every token has a near-twin (its right-hand neighbour, cosine ~0.99) in the same 128-token tile: 0.01-0.02 apart,
    well inside the int8 pass's 2 eps and well outside the fp16 pass's.  The residuals pass the rho_F rule, so the
    automatic mode starts on int8, the probe chunk queues most of its maps, and chunks 1.. run the fp16 pass."""
    geo, T, C = Geometry(), 8, 256
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=41, noise=0.2, max_shift=2)
    f = feats.numpy()
    rs = np.random.RandomState(41)
    f[..., 1::2] = f[..., 0:-1:2] + 0.08 * rs.standard_normal(f[..., 1::2].shape).astype(np.float32)
    feats = torch.from_numpy(f)
    head = synth.head_weights("sharp", seed=5)
    q = synth.lattice_query_points(16, 12, geo.H, geo.W, t_q=[i % T for i in range(192)], margin=14.0, jitter_seed=5)
    mi = _tracker(feats, head, geo)
    auto, sta = _infer(mi, q, -1, -1)
    s8, st8 = _infer(mi, q, 1, 1)
    f16, st16 = _infer(mi, q, 1, 0)
    print(f"[twin tokens] auto {sta} | int8 forced {st8} | fp16 forced {st16}")
    assert sta["anchor_maps"] > 4096, "needs a probe chunk and at least one more"
    assert st8["coarse"] == "int8" and st8["full_map"] * 16 > st8["anchor_maps"]
    assert sta["pipeline"] == "exact-window" and sta["coarse_rho_f"] <= 0.03 and sta["coarse"] == "fp16"
    assert sta["full_map"] < st8["full_map"]          # chunks after the probe ran the fp16 pass's tighter plan
    _same(auto, s8)
    _same(auto, f16)

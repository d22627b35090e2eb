"""GPU: the int8 coarse pass above C = 1040 (ViT-g/14's C = 1536, and the cap C = 2048).

Above C = 1040 the int32 accumulator <q_d, q_x> is still exact (C 127^2 < 2^31), but its conversion to float rounds
(cvt.rn.f32.s32, <= 2^-24 relative), and the exact split path's 3 ceil(C / 16) truncating adds outgrow 2^-15: eps's slack
is 2^-15 + 3 ceil(C / 16) 2^-23 there (csrc/xwin.cuh, DESIGN 3.1), checked against the reported eps.
- Keys bit for bit against test_coarse_s8_keys_exact_gpu.py's reference: exact integer products in float64, rounded to
  float32 to nearest even as cvt.rn.f32.s32 does, then the pass's float32 roundings.  The features are made "flat"
  (every channel's magnitude within 3 % of the row maximum), so a token's product with its own multiple reaches
  C 127^2 > 2^24 and the conversion does round; the test checks that it did.  Shapes off the tile grid as there.
- `infer` at C = 1536 on three heads: the forced int8 and fp16 passes give byte-identical trajectories, occlusion and
  cosines, and both match the GPU fp32 oracle (|dxy| <= 1e-3 px, identical occlusion).
- infer_stats()['coarse'] is int8 in the automatic mode on Gaussian-like features.
- The training step's reverse pass at C = 1536 against float64 (test_train_backward_gpu.py's bound)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import inference as oi
from oracle import synth
from oracle.tracker import Geometry

import test_train_backward_gpu as tb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))


def _module(name):
    spec = importlib.util.spec_from_file_location(name + "_cases", os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _flat(x):
    """sign(x) (1 - 0.03 |sin(1000 x)|): every channel within 3 % of the row maximum, so q = rint(127 x / max|x|) is
    123..127.  Elementwise, so duplicated tokens stay duplicated."""
    return (np.sign(x) * (1 - 0.03 * np.abs(np.sin(x * 1e3)))).astype(np.float32)


KEY_CASES = {
    "rows_c1536": dict(seed=31, hw=(67, 121), T=3, C=1536, sizes=(1, 255, 256, 300), frames=(0, 2, 1, 2), first_row=7),
    "blocks_c1536": dict(seed=32, hw=(13, 25), T=4, C=1536, sizes=(129, 256, 1000, 3, 511), frames=(1, 0, 1, 3, 2),
                         first_row=3, gaps=True),
    "rows_c2048": dict(seed=33, hw=(3, 43), T=2, C=2048, sizes=(257, 64, 130), frames=(0, 1, 0), first_row=5),
}


@pytest.mark.parametrize("name", sorted(KEY_CASES))
def test_int8_keys_bit_exact_above_1040(name):
    ke = _module("test_coarse_s8_keys_exact_gpu")
    cs = ke.make_case(**KEY_CASES[name])
    cs["feats"] = _flat(cs["feats"])
    cs["desc"] = 2 * _flat(cs["desc"] / 2)     # a descriptor row 2 x a token stays 2 x that token
    r = ke._s8_module()._run_keys_i8(cs)
    n_rounded = 0
    for r0, m, f in zip(cs["row0"], cs["m"], cs["frame"]):
        ints = r["dq"][int(r0):int(r0 + m)].double() @ r["fq"][f].double().T
        n_rounded += int((ints.float().double() != ints).sum())
    assert n_rounded > 0, "no accumulator above 2^24 needed rounding"
    key1, max2 = r["key1"].view(np.uint64), r["max2"]
    val = ((key1 >> np.uint64(32)).astype(np.uint32).view(np.float32) + np.float32(0)).view(np.uint32)
    tok = 0x7FFFFFFF - (key1 & np.uint64(0xFFFFFFFF)).astype(np.int64)
    for sl, k1, kt, k2 in ke.reference_keys(r, cs):
        assert np.array_equal(val[sl], k1.view(np.uint32)), "tile maximum differs"
        assert np.array_equal(tok[sl], kt), "token of the tile maximum differs"
        assert np.array_equal((max2[sl] + np.float32(0)).view(np.uint32), k2.view(np.uint32)), "second value differs"
    print(f"[{name}] {n_rounded} accumulators rounded by the float conversion")
    _check_eps(ke, cs, r)


def _check_eps(ke, cs, r):
    """eps = rho_d + (1 + rho_d) rho_F + slack, rounded up: slack = 2^-15 up to C = 1040, 2^-15 + 3 ceil(C / 16) 2^-23
    (the exact split path's truncating adds, csrc/xwin.cuh) above.  Against float64 from the unrounded residuals: never
    below, and above by no more than the kernel's upward roundings."""
    C = cs["C"]
    qr = ke._s8_module()._quant_ref
    rho_d = qr(cs["desc"])[3]
    rho_f = qr(cs["feats"])[3].max(axis=1)
    slack = 2.0 ** -15 + (3 * -(-C // 16) * 2.0 ** -23 if C > 1040 else 0.0)
    for r0, m, f in zip(cs["row0"], cs["m"], cs["frame"]):
        rd = rho_d[int(r0):int(r0 + m)]
        want = rd + (1 + rd) * rho_f[f] + slack
        got = r["eps"][int(r0):int(r0 + m)].astype(np.float64)
        assert (got >= want).all() and (got <= want * (1 + 2.0 ** -20)).all(), C


@pytest.mark.parametrize("C", [1024, 1040])
def test_eps_slack_unchanged_up_to_1040(C):
    ke = _module("test_coarse_s8_keys_exact_gpu")
    cs = ke.make_case(seed=34, hw=(13, 25), T=2, C=C, sizes=(129, 40), frames=(1, 0), first_row=2)
    _check_eps(ke, cs, ke._s8_module()._run_keys_i8(cs))


@pytest.mark.parametrize("kind", ["sharp", "well", "mixed"])
def test_infer_c1536_int8_equals_fp16_and_oracle(kind):
    s8m = _module("test_coarse_s8_gpu")
    geo, T, C = Geometry(), 5, 1536
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=17, noise=0.2, max_shift=2)
    head = synth.head_weights(kind, seed=17)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=14.0, jitter_seed=17)
    mi = s8m._tracker(feats, head, geo)
    s8, st8 = s8m._infer(mi, q, 1, 1)
    f16, st16 = s8m._infer(mi, q, 1, 0)
    auto, sta = s8m._infer(mi, q, -1, -1)
    print(f"[C=1536 {kind}] int8 {st8} | fp16 {st16} | auto {sta}")
    assert st8["coarse"] == "int8" and st16["coarse"] == "fp16"
    assert 0 < sta["coarse_rho_f"] <= 0.03
    if kind != "mixed":   # mixed-sign refiner weights may send the automatic mode to the full-map pipeline after the probe
        assert sta["pipeline"] == "exact-window" and sta["coarse"] == "int8"
    for k in ("traj", "occ", "cos_sims"):
        assert torch.equal(s8[k], f16[k]), k
    oracle.use_exact_fp32()
    with torch.no_grad():
        t_ref, o_ref = oi.infer(feats.to(DEV), q.to(DEV), {k: v.to(DEV) for k, v in head.items()}, geo, 0.7, 0.6)
    for r in (s8, f16):
        assert (r["traj"][..., :2] - t_ref).abs().max().item() <= 1e-3
        assert torch.equal(r["occ"].cpu(), o_ref.cpu())


@pytest.mark.parametrize("kind", ["sharp", "well"])
def test_training_step_c1536_against_float64(kind):
    geo = Geometry(H=154, W=210)
    feats, _ = synth.shifted_field_features(4, 1536, geo.h, geo.w, seed=121, noise=0.2, max_shift=2)
    gen = tb._gen("c1536", kind)
    pts, tgt, gout = tb._batch(geo, 4, 256, gen)
    tb.run_production(f"C=1536 {kind}", geo, feats, synth.head_weights(kind, seed=121), "fp16x3", pts, tgt, gout)


def test_quantise_features_cap():
    from dino_tracker_b200 import _lib
    x = torch.randn(1, 6, 2048, device=DEV)
    assert _lib.quantise_features(x, x.norm(dim=-1).contiguous(), _lib.stream_ptr()) is not None
    x = torch.randn(1, 6, 2064, device=DEV)
    assert _lib.quantise_features(x, x.norm(dim=-1).contiguous(), _lib.stream_ptr()) is None

"""GPU: the int8 coarse pass's keys (key1, max2 of dinotrk_xw_coarse_keys_i8) bit for bit.  They must equal the same
statistics formed from the exact integer products with the pass's float32 roundings: u = float(q_d . q_x) * fac_x per
token; the maximum of u per 128-token tile, the first token holding it and the second value; those two values times
fac_d, clamped at zero.  (test_coarse_s8_gpu.py checks the same keys against a float64 reference within a tolerance.)

The cases are shapes off the GEMM's tile grid:
- group row counts off the 128 / 256 grid next to full ones;
- groups that start at arbitrary rows of one descriptor table, back to back;
- launches with few row blocks next to one with about 200;
- C = 1040, where the last K block is almost all zero fill, and C = 64 / 128 / 256 (one or two K blocks);
- P off the 128 grid, down to a last tile of one token;
- maxima tied between the two 128-token key tiles of one 256-token GEMM tile."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 128
HERE = os.path.dirname(os.path.abspath(__file__))


def _s8_module():
    spec = importlib.util.spec_from_file_location("coarse_s8_cases", os.path.join(HERE, "test_coarse_s8_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_case(seed, hw, T, C, sizes, frames, first_row=0, gaps=False):
    """Groups of `sizes` rows against `frames`, laid out from `first_row` of one descriptor table (with gaps of 3 rows
    when `gaps`, else back to back).  In every frame, each tile holds an exact duplicate token (b > a), and each pair of
    tiles (2j, 2j + 1) holds a token of tile 2j copied into tile 2j + 1; every 4th descriptor row is 2 x one of those
    duplicated tokens, so that the tied tokens hold their tiles' maxima."""
    rng = np.random.default_rng(seed)
    h, w = hw
    P = h * w
    n_tiles = -(-P // TILE)
    feats = rng.standard_normal((T, P, C), dtype=np.float32)
    dups = [[] for _ in range(T)]
    for f in range(T):
        for t in range(n_tiles):
            lo, hi = t * TILE, min(P, (t + 1) * TILE)
            if hi - lo >= 2:
                a, b = np.sort(rng.choice(np.arange(lo, hi), size=2, replace=False))
                feats[f, b] = feats[f, a]
                dups[f].append(a)
        for t in range(0, n_tiles - 1, 2):
            hi = min(P, (t + 2) * TILE)
            a, b = rng.integers(t * TILE, (t + 1) * TILE), rng.integers((t + 1) * TILE, hi)
            feats[f, b] = feats[f, a]
            dups[f].append(a)
    row0 = []
    r = first_row
    for m in sizes:
        row0.append(r)
        r += m + (3 if gaps else 0)
    desc = rng.standard_normal((r + 5, C), dtype=np.float32)
    for g, (m, f) in enumerate(zip(sizes, frames)):
        for j in range(0, m, 4):
            desc[row0[g] + j] = 2.0 * feats[f, dups[f][rng.integers(len(dups[f]))]]
    return dict(feats=feats, desc=desc, hw=hw, T=T, C=C, P=P, n_tiles=n_tiles, row0=np.array(row0, np.int32),
                m=np.array(sizes, np.int32), frame=np.array(frames, np.int32))


def reference_keys(r, cs):
    """key1 / max2 rows of every group from the exact integer products, with the kernel's float32 roundings."""
    P, nt = cs["P"], cs["n_tiles"]
    fq, dq, ffac, dfac = r["fq"], r["dq"], r["ffac"], r["dfac"]
    out = []
    for r0, m, f in zip(cs["row0"], cs["m"], cs["frame"]):
        sl = slice(int(r0), int(r0 + m))
        ints = dq[sl].double() @ fq[f].double().T                 # exact: |sum| <= C 127^2 < 2^24
        u = ints.float() * ffac[f][None, :]
        u = torch.cat([u, torch.full((m, nt * TILE - P), -np.inf, device=DEV)], 1).view(m, nt, TILE)
        top = u.topk(2, dim=2).values
        tok = u.argmax(dim=2) + torch.arange(nt, device=DEV)[None, :] * TILE   # the first token holding the maximum
        d = dfac[sl, None]
        k1 = torch.fmax(top[..., 0] * d, torch.zeros((), device=DEV)) + 0.0
        k2 = torch.fmax(top[..., 1] * d, torch.zeros((), device=DEV)) + 0.0
        out.append((sl, k1.cpu().numpy(), tok.cpu().numpy(), k2.cpu().numpy()))
    return out


CASES = {   # name: make_case arguments
    # 5 row blocks; C = 1040: 9 K blocks, the last one 16 channels wide
    "rows_c1040": dict(seed=3, hw=(67, 121), T=3, C=1040, sizes=(1, 255, 256, 300), frames=(0, 2, 1, 2), first_row=7),
    # adjacent groups from an odd row
    "rows_c1024": dict(seed=4, hw=(67, 121), T=2, C=1024, sizes=(512, 700), frames=(1, 0), first_row=1),
    # ~200 row blocks, more than one per CTA pair; two K blocks
    "blocks_c256": dict(seed=5, hw=(13, 25), T=4, C=256, sizes=tuple(int(x) for x in
                       np.random.default_rng(9).integers(1, 1300, size=60)), frames=tuple(i % 4 for i in range(60)),
                       first_row=11, gaps=True),
    # one K block
    "kb1_c64": dict(seed=6, hw=(13, 25), T=2, C=64, sizes=(129, 256, 1000, 3), frames=(1, 0, 1, 0), first_row=0),
    # P = 129: the last key tile holds a single token
    "p129_c128": dict(seed=7, hw=(3, 43), T=2, C=128, sizes=(257, 64), frames=(0, 1), first_row=5),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_int8_keys_bit_exact(name):
    cs = make_case(**CASES[name])
    assert cs["P"] % TILE != 0
    r = _s8_module()._run_keys_i8(cs)
    key1, max2 = r["key1"].view(np.uint64), r["max2"]
    val = ((key1 >> np.uint64(32)).astype(np.uint32).view(np.float32) + np.float32(0)).view(np.uint32)
    tok = 0x7FFFFFFF - (key1 & np.uint64(0xFFFFFFFF)).astype(np.int64)
    n_cross = 0
    for sl, k1, kt, k2 in reference_keys(r, cs):
        assert np.array_equal(val[sl], k1.view(np.uint32)), "tile maximum differs"
        assert np.array_equal(tok[sl], kt), "token of the tile maximum differs"
        assert np.array_equal((max2[sl] + np.float32(0)).view(np.uint32), k2.view(np.uint32)), "second value differs"
        # maxima tied between the two key tiles of a 256-token GEMM tile: each tile names its own token
        n_cross += int(((k1[:, 0:-1:2] == k1[:, 1::2]) & (k1[:, 0:-1:2] > 0.5)).sum())
    assert n_cross > 0 or cs["n_tiles"] < 2

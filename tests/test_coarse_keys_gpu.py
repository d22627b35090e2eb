"""GPU: the coarse pass's tile keys (csrc/xwin.cu, dinotrk_xw_coarse_keys) against float64 and a stored capture.

No result of the tracker depends on a coarse value, so a wrong key -- a lost maximum, a wrong tie, an under-reported
second value that hides an ambiguity -- shows up elsewhere only as extra full-map work or, at a near-tie, as a wrong
candidate set.  Here the keys are checked directly: per (descriptor row, 128-token tile) the maximum, the first token
holding it and the second largest value of relu(hi(d) . hi(F) / (|d| |F|)), against the same expression in float64 on
the fp16-rounded operands, and bit for bit against keys captured from an earlier build of the kernel.

Rewrite the capture (only when the kernel's arithmetic is meant to change):  python tests/test_coarse_keys_gpu.py
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coarse_keys.npz")
TILE = 128
CANARY_KEY = 0x5A5A5A5A5A5A5A5A
CANARY_MAX2 = -7.25

# name: (seed, token grid h x w, T, C, group sizes, group frames)
CASES = {
    "wide_c1024": (11, (67, 121), 3, 1024, (1, 255, 256, 257, 655), (0, 1, 2, 1, 0)),
    "wide_c64": (12, (67, 121), 3, 64, (1, 255, 256, 257, 655), (2, 0, 1, 1, 0)),
    "odd_tiles_c1024": (13, (13, 25), 4, 1024, (655, 1, 257, 256, 255), (3, 0, 1, 2, 3)),
    "odd_tiles_c64": (14, (13, 25), 4, 64, (257, 255, 1, 655, 256), (1, 2, 3, 0, 2)),
}
GOLDEN_CASES = {   # small enough to store their keys
    "golden_wide": (21, (67, 121), 2, 128, (1, 257, 40), (0, 1, 0)),
    "golden_odd": (22, (13, 25), 3, 64, (655, 256), (2, 0)),
}
GAP = 3   # descriptor rows between groups (and before the first): their key slots must keep the canary


def make_case(seed, hw, T, C, sizes, frames):
    """Seeded inputs (numpy PCG64: the same on every machine).  Every tile of every frame holds one exact duplicate token
    (b > a, same features); every 5th descriptor row of a group is 2 x token a of some tile of its frame, so that the
    duplicated pair holds the tile's maximum and the key must name a, the first of them."""
    rng = np.random.default_rng(seed)
    h, w = hw
    P = h * w
    n_tiles = -(-P // TILE)
    feats = rng.standard_normal((T, P, C), dtype=np.float32)
    dup = np.zeros((T, n_tiles), dtype=np.int64)
    for f in range(T):
        for t in range(n_tiles):
            lo, hi = t * TILE, min(P, (t + 1) * TILE)
            a, b = np.sort(rng.choice(np.arange(lo, hi), size=2, replace=False))
            feats[f, b] = feats[f, a]
            dup[f, t] = a
    row0 = []
    r = GAP
    for m in sizes:
        row0.append(r)
        r += m + GAP
    desc = rng.standard_normal((r, C), dtype=np.float32)
    for g, (m, f) in enumerate(zip(sizes, frames)):
        for j in range(0, m, 5):
            desc[row0[g] + j] = 2.0 * feats[f, dup[f, rng.integers(n_tiles)]]
    norms = np.sqrt((feats.astype(np.float64) ** 2).sum(-1)).astype(np.float32)
    desc_norm = np.sqrt((desc.astype(np.float64) ** 2).sum(-1)).astype(np.float32)
    return dict(feats=feats, norms=norms, desc=desc, desc_norm=desc_norm, hw=hw, T=T, C=C, P=P, n_tiles=n_tiles,
                row0=np.array(row0, np.int32), m=np.array(sizes, np.int32), frame=np.array(frames, np.int32))


def run_keys(cs):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    h, w = cs["hw"]
    g = _lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
    assert (g.h, g.w) == (h, w)
    feats = torch.from_numpy(cs["feats"]).to(DEV)
    hi = feats.half().contiguous()
    norms = torch.from_numpy(cs["norms"]).to(DEV)
    fs = _lib.make_features(feats, norms, hi, hi)   # (the coarse pass reads the hi halves only)
    desc_hi = torch.from_numpy(cs["desc"]).to(DEV).half().contiguous()
    desc_norm = torch.from_numpy(cs["desc_norm"]).to(DEV)
    gf, gr, gm = (torch.from_numpy(cs[k]).to(DEV) for k in ("frame", "row0", "m"))
    rows, n_groups = desc_hi.shape[0], len(cs["m"])
    key1 = torch.full((rows, cs["n_tiles"]), CANARY_KEY, dtype=torch.int64, device=DEV)
    max2 = torch.full((rows, cs["n_tiles"]), CANARY_MAX2, dtype=torch.float32, device=DEV)
    nb = lib.dinotrk_xw_coarse_keys_workspace_bytes(cs["T"], n_groups, ctypes.byref(g))
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    _lib.check(lib.dinotrk_xw_coarse_keys(ctypes.byref(fs), ctypes.byref(g), _lib.ptr(desc_hi), rows, _lib.ptr(desc_norm),
                                          _lib.ptr(gf), _lib.ptr(gr), _lib.ptr(gm), n_groups, _lib.ptr(key1), _lib.ptr(max2),
                                          _lib.ptr(ws), nb, _lib.stream_ptr()), "xw_coarse_keys")
    torch.cuda.synchronize()
    return key1.cpu().numpy(), max2.cpu().numpy()


def group_rows(cs):
    return np.concatenate([np.arange(r, r + m) for r, m in zip(cs["row0"], cs["m"])])


def reference(cs):
    """float64 on the fp16-rounded operands: pre-ReLU values v[row][token] of the group rows (the kernel applies the ReLU to
    the two statistics, after the arg-max)."""
    P = cs["P"]
    hi = torch.from_numpy(cs["feats"]).to(DEV).half().double()
    dh = torch.from_numpy(cs["desc"]).to(DEV).half().double()
    rn = 1.0 / torch.from_numpy(cs["norms"]).to(DEV).double().clamp_min(1e-4)
    rd = 1.0 / torch.from_numpy(cs["desc_norm"]).to(DEV).double().clamp_min(1e-4)
    out = {}
    for r0, m, f in zip(cs["row0"], cs["m"], cs["frame"]):
        v = (dh[r0:r0 + m] @ hi[f].T) * rn[f][None, :] * rd[r0:r0 + m, None]
        pad = torch.full((m, cs["n_tiles"] * TILE - P), -np.inf, dtype=torch.float64, device=DEV)
        out[int(r0)] = torch.cat([v, pad], 1).view(m, cs["n_tiles"], TILE).cpu().numpy()
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_coarse_keys_match_float64(name):
    cs = make_case(*CASES[name])
    key1, max2 = run_keys(cs)
    C, P = cs["C"], cs["P"]
    tol = max(C, 64) * 2.0 ** -21          # fp32 accumulation of C exact fp16 products, in cosine units (plus the scalings)
    kmax = (key1.view(np.uint64) >> np.uint64(32)).astype(np.uint32).view(np.float32)
    ktok = 0x7FFFFFFF - (key1.view(np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)
    rows = group_rows(cs)
    outside = np.setdiff1d(np.arange(key1.shape[0]), rows)
    assert (key1[outside] == CANARY_KEY).all() and (max2[outside] == CANARY_MAX2).all(), "key slot outside every group written"
    ref = reference(cs)
    n_checked = n_dup = 0
    for r0, m in zip(cs["row0"], cs["m"]):
        v = ref[int(r0)]
        km, kt, k2 = kmax[r0:r0 + m], ktok[r0:r0 + m], max2[r0:r0 + m]
        tiles = np.arange(cs["n_tiles"])[None, :]
        assert ((kt >= tiles * TILE) & (kt < np.minimum((tiles + 1) * TILE, P))).all(), "token outside its tile / past P"
        srt = -np.sort(-v, axis=2)
        top1, top2 = srt[..., 0], srt[..., 1]
        assert np.abs(km - np.maximum(top1, 0.0)).max() <= tol, "tile maximum off"
        assert np.abs(k2 - np.maximum(top2, 0.0)).max() <= tol, "second value off"
        first = v.argmax(axis=2) + tiles * TILE
        sure = top1 - top2 > 2 * tol
        assert (kt[sure] == first[sure]).all(), "token is not the first arg-max of a clear tile maximum"
        # exact duplicates holding the maximum (the descriptor rows built from token a): the first token, max2 == max
        tie = (top1 == top2) & (top1 > 0.5)
        tok_v = np.take_along_axis(v, (kt - tiles * TILE)[..., None], axis=2)[..., 0]
        assert (kt[tie] == first[tie]).all() and (k2[tie] == km[tie]).all(), "exact tie not resolved to the first token"
        assert (tok_v[tie] == top1[tie]).all()
        n_checked += int(sure.sum())
        n_dup += int(tie.sum())
    assert n_dup >= len(cs["m"]) and n_checked > 0.75 * rows.size * cs["n_tiles"], (n_dup, n_checked)


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_coarse_keys_bit_identical_to_capture(name):
    g = np.load(GOLDEN)
    cs = make_case(*GOLDEN_CASES[name])
    assert np.isclose(float(np.abs(cs["feats"]).astype(np.float64).sum()), float(g[name + ".feat_abs_sum"]), rtol=1e-12), \
        "seeded inputs drifted from the capture"
    key1, max2 = run_keys(cs)
    assert np.array_equal(key1, g[name + ".key1"]), "key1 differs from the capture"
    assert np.array_equal(max2.view(np.uint32), g[name + ".max2"].view(np.uint32)), "max2 differs from the capture"


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    arrays = {}
    for name, cfg in GOLDEN_CASES.items():
        cs = make_case(*cfg)
        k1, m2 = run_keys(cs)
        arrays[name + ".key1"], arrays[name + ".max2"] = k1, m2
        arrays[name + ".feat_abs_sum"] = np.array(np.abs(cs["feats"]).astype(np.float64).sum())
    out = sys.argv[1] if len(sys.argv) > 1 else GOLDEN
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})

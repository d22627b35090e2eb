"""GPU: the exact box GEMM of the exact-window pipeline (csrc/xwin.cu, dinotrk_xw_box_gemm) on its own.

Per cell (up to 128 descriptor rows correlating with one frame) the kernel writes the raw split-precision accumulators of
the 21 x 21 token box, xbox[row][by * 21 + bx].  Everything the exact-window head decides is formed from these values as
relu(acc / max(|d| |F|, 1e-8)), the full-map epilogue's expression, so they are checked
  - bit for bit against the full-map GEMM (dinotrk_corr_maps on groups wide enough for the tensor GEMM): the same split
    products in the same order, descriptors on the wgmma M side there;
  - against float64 on the same fp16 operands, within the split's error bound plus the tensor cores' accumulation;
  - for exact zeros on box tokens outside the token grid (zero fill), and for untouched canaries in columns 441..447, in
    the rows of a skipped cell and between cells.
Cell sizes 1, 50, 64 (every cell of the call fits one 64-row tile) and 65, 100, 128 (two 64-row halves), C = 64 and 1024,
boxes inside the grid and hanging over each of its sides.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BOX, COLS = 21, 448
CANARY = -12345.5
SKIP = -(2 ** 31)
GAP = 3   # descriptor rows before and between cells: never written

# name: (seed, token grid h x w, frames, C, cell sizes)
CASES = {
    "t50_c1024": (41, (67, 121), 3, 1024, (50, 1, 64, 50, 50, 50, 50, 50, 50)),
    "t50_c64": (42, (67, 121), 3, 64, (50, 1, 64, 50, 50, 50, 50, 50, 50)),
    "t100_c1024": (43, (67, 121), 3, 1024, (100, 1, 50, 64, 65, 128, 100, 100, 100)),
    "t100_c64": (44, (67, 121), 3, 64, (128, 65, 1, 50, 64, 100, 100, 128, 100)),
}


def origins(h, w):
    """Box origins (first row, first column), one per cell in turn: inside, over every side and corner, and a skipped cell."""
    return [(30, 50), (-6, -9), (h - 15, w - 12), (-20, 60), (20, -20), (10, w - 1), (h - 1, 3), (25, SKIP), (h - 21, w - 21)]


def make_case(seed, hw, T, C, sizes):
    rng = np.random.default_rng(seed)
    h, w = hw
    feats = rng.standard_normal((T, h * w, C), dtype=np.float32)
    row0, r = [], GAP
    for m in sizes:
        row0.append(r)
        r += m + GAP
    desc = rng.standard_normal((r, C), dtype=np.float32)
    org = origins(h, w)
    assert len(org) >= len(sizes)
    return dict(feats=feats, desc=desc, hw=hw, T=T, C=C, row0=np.array(row0, np.int32), m=np.array(sizes, np.int32),
                frame=np.array([k % T for k in range(len(sizes))], np.int32), org=np.array(org[:len(sizes)], np.int32))


def box_tokens(cs, k):
    """(token index clamped into the grid, inside-the-grid mask) of cell k's 441 box positions, row-major."""
    h, w = cs["hw"]
    oy, ox = cs["org"][k]
    by, bx = np.meshgrid(np.arange(BOX), np.arange(BOX), indexing="ij")
    r, c = (oy + by).ravel(), (ox + bx).ravel()
    inside = (r >= 0) & (r < h) & (c >= 0) & (c < w)
    return np.where(inside, r * w + c, 0), inside


class Inputs:
    def __init__(self, cs):
        from dino_tracker_b200 import _lib
        self.lib, self._lib = _lib.load(), _lib
        h, w = cs["hw"]
        self.geom = _lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
        assert (self.geom.h, self.geom.w) == (h, w)
        st = _lib.stream_ptr()
        self.feats = torch.from_numpy(cs["feats"]).to(DEV)
        self.norms = self.feats.norm(dim=2).contiguous()
        self.f_hi, self.f_lo = _lib.split_fp16(self.feats, st)
        self.fs = _lib.make_features(self.feats, self.norms, self.f_hi, self.f_lo)
        self.desc = torch.from_numpy(cs["desc"]).to(DEV)
        self.dn = self.desc.norm(dim=1).contiguous()
        self.d_hi, self.d_lo = _lib.split_fp16(self.desc, st)
        torch.cuda.synchronize()


def run_box(cs, x):
    _lib, lib = x._lib, x.lib
    rows = cs["desc"].shape[0]
    xbox = torch.full((rows, COLS), CANARY, dtype=torch.float32, device=DEV)
    row0, m, frame = (torch.from_numpy(cs[k]).to(DEV) for k in ("row0", "m", "frame"))
    org = torch.from_numpy(cs["org"]).to(DEV).contiguous()
    _lib.check(lib.dinotrk_xw_box_gemm(ctypes.byref(x.fs), ctypes.byref(x.geom), _lib.ptr(x.d_hi), _lib.ptr(x.d_lo), rows,
                                       _lib.ptr(row0), _lib.ptr(m), _lib.ptr(frame), _lib.ptr(org), len(cs["m"]),
                                       int(cs["m"].max()), _lib.ptr(xbox), _lib.stream_ptr()), "xw_box_gemm")
    torch.cuda.synchronize()
    return xbox.cpu().numpy()


def run_full_maps(cs, x, f):
    """Full-map split-precision GEMM of every descriptor row against frame f (one group: the tensor GEMM)."""
    _lib, lib = x._lib, x.lib
    rows, C = cs["desc"].shape
    grp = torch.tensor([[f], [0], [rows], [0]], dtype=torch.int32, device=DEV)
    maps = torch.zeros(rows, lib.dinotrk_map_stride(ctypes.byref(x.geom)), device=DEV)
    nb = lib.dinotrk_corr_maps_workspace_bytes(rows, 1, C)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    _lib.check(lib.dinotrk_corr_maps(ctypes.byref(x.fs), ctypes.byref(x.geom), _lib.ptr(x.desc), _lib.ptr(x.dn), _lib.ptr(grp[0]),
                                     _lib.ptr(grp[1]), _lib.ptr(grp[2]), _lib.ptr(grp[3]), 1, rows, rows, _lib.ptr(maps),
                                     _lib.ptr(ws), nb, _lib.stream_ptr()), "corr_maps")
    torch.cuda.synchronize()
    return maps.cpu().numpy()


@pytest.fixture(scope="module", params=sorted(CASES))
def case(request):
    cs = make_case(*CASES[request.param])
    x = Inputs(cs)
    return cs, x, run_box(cs, x)


def test_untouched_and_zero_fill(case):
    cs, _, xbox = case
    written = np.zeros(xbox.shape[0], bool)
    for k, (r0, m) in enumerate(zip(cs["row0"], cs["m"])):
        if cs["org"][k][1] != SKIP:
            written[r0:r0 + m] = True
    assert (xbox[~written] == CANARY).all(), "a row outside every computed cell was written"
    assert (xbox[written][:, BOX * BOX:] == CANARY).all(), "a padding column (441..447) was written"
    for k, (r0, m) in enumerate(zip(cs["row0"], cs["m"])):
        if cs["org"][k][1] == SKIP:
            continue
        _, inside = box_tokens(cs, k)
        assert (xbox[r0:r0 + m, :BOX * BOX][:, ~inside] == 0.0).all(), f"cell {k}: box token outside the grid is not zero"
        assert np.isfinite(xbox[r0:r0 + m, :BOX * BOX]).all()


def test_bit_identical_to_full_map_gemm(case):
    cs, x, xbox = case
    fn = x.norms.cpu().numpy()
    dn = x.dn.cpu().numpy()
    n_pos = 0
    for f in sorted(set(cs["frame"].tolist())):
        maps = run_full_maps(cs, x, f)
        for k, (r0, m) in enumerate(zip(cs["row0"], cs["m"])):
            if cs["frame"][k] != f or cs["org"][k][1] == SKIP:
                continue
            tok, inside = box_tokens(cs, k)
            acc = xbox[r0:r0 + m, :BOX * BOX][:, inside]
            # the exact-window head's expression (xw_window_kernel): __fmul_rn, fmaxf, __fdiv_rn, ReLU -- all float32
            den = np.maximum(dn[r0:r0 + m, None] * fn[f][tok[inside]][None, :], np.float32(1e-8))
            v = np.maximum(acc / den, np.float32(0.0))
            ref = maps[r0:r0 + m][:, tok[inside]]
            bad = v != ref
            assert not bad.any(), (f"cell {k} (m = {m}): {int(bad.sum())} box values differ from the full-map GEMM, "
                                   f"max |diff| = {np.abs(v - ref).max():.3g}")
            n_pos += int((v > 0).sum())
    assert n_pos > 0


def test_matches_float64(case):
    cs, x, xbox = case
    C = cs["C"]
    d64 = (x.d_hi.double() + x.d_lo.double()).cpu().numpy()
    f_hi, f_lo = x.f_hi.cpu().numpy(), x.f_lo.cpu().numpy()
    dnorm = np.linalg.norm(cs["desc"].astype(np.float64), axis=1)
    fnorm = np.linalg.norm(cs["feats"].astype(np.float64), axis=2)
    # split bound (DESIGN 3.1) + the tensor cores' truncating accumulation, <= 2^-22 of the running magnitude per wgmma
    rel = 2.0 ** -21 + 3 * (C // 16) * 2.0 ** -22
    worst = 0.0
    for k, (r0, m) in enumerate(zip(cs["row0"], cs["m"])):
        if cs["org"][k][1] == SKIP:
            continue
        f = cs["frame"][k]
        tok, inside = box_tokens(cs, k)
        ft = f_hi[f][tok].astype(np.float64) + f_lo[f][tok].astype(np.float64)
        ref = (d64[r0:r0 + m] @ ft.T) * inside[None, :]
        scale = dnorm[r0:r0 + m, None] * fnorm[f][tok][None, :]
        err = np.abs(xbox[r0:r0 + m, :BOX * BOX].astype(np.float64) - ref)
        assert (err <= rel * scale).all(), f"cell {k}: max error {(err / scale).max():.3g} of |d||F| (bound {rel:.3g})"
        worst = max(worst, float((err / scale).max()))
    assert worst < rel

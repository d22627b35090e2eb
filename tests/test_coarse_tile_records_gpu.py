"""GPU: the coarse pass's per-tile records (tcgemm.cuh, fragment epilogues).  The producer decodes every tile once and hands
the consumers a record in shared memory -- group, first row, first column, frame, first descriptor row and row count --
next to the tile's first K block; the epilogue takes the group's first map and the row factor from it.  The int8 keys
must stay bit for bit the statistics of the exact integer products (test_coarse_s8_keys_exact_gpu.py's reference) where
that hand-over has edges:
- a CTA whose consecutive tiles belong to different groups (many groups, each of one or two row blocks);
- groups of one row block, down to one row;
- more CTA pairs than tiles (the grid is sized from a bound on the row blocks), so some CTAs get no tile;
- a last key tile of one token (P = 129) and K of one block (C = 64), where the producer runs furthest ahead."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _module(name):
    spec = importlib.util.spec_from_file_location(name[:-3], os.path.join(HERE, name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CASES = {   # name: make_case arguments of test_coarse_s8_keys_exact_gpu
    # 90 groups of 1..300 rows over 4 frames, back to back: every CTA pair changes group from one tile to the next
    "group_changes_c128": dict(seed=21, hw=(13, 25), T=4, C=128, sizes=tuple(int(x) for x in
                               np.random.default_rng(22).integers(1, 300, size=90)), frames=tuple((7 * i) % 4 for i in range(90)),
                               first_row=3),
    # one-row and one-block groups; P = 129: one GEMM N tile whose second key tile holds one token; one K block
    "one_block_p129_c64": dict(seed=23, hw=(3, 43), T=3, C=64, sizes=(1, 1, 256, 2, 255, 1, 129), frames=(2, 0, 1, 1, 0, 2, 0),
                               first_row=0, gaps=True),
    # 10 groups of 200 rows: 10 row blocks against a grid bound of 17 pairs, so 7 pairs find no tile
    "idle_ctas_c1040": dict(seed=24, hw=(3, 43), T=2, C=1040, sizes=(200,) * 10, frames=tuple(i % 2 for i in range(10)),
                            first_row=5),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_int8_keys_with_tile_records(name):
    exact = _module("test_coarse_s8_keys_exact_gpu.py")
    cs = exact.make_case(**CASES[name])
    r = exact._s8_module()._run_keys_i8(cs)
    key1, max2 = r["key1"].view(np.uint64), r["max2"]
    val = ((key1 >> np.uint64(32)).astype(np.uint32).view(np.float32) + np.float32(0)).view(np.uint32)
    tok = 0x7FFFFFFF - (key1 & np.uint64(0xFFFFFFFF)).astype(np.int64)
    for sl, k1, kt, k2 in exact.reference_keys(r, cs):
        assert np.array_equal(val[sl], k1.view(np.uint32)), "tile maximum differs"
        assert np.array_equal(tok[sl], kt), "token of the tile maximum differs"
        assert np.array_equal((max2[sl] + np.float32(0)).view(np.uint32), k2.view(np.uint32)), "second value differs"

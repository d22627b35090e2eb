"""Anchor-phase planner of the exact-window pipeline without a GPU (dinotrk_infer_plan_anchors): which descriptor rows the
GEMMs read in place from the unique (query, source frame) table and which are gathered into the chunk's own rows.  For
random anchor lists -- full, a few holes, alternating queries, empty frames, flagged queries, T not dividing 256 -- every
(slot, i, a) item appears exactly once and in order, an in-place group's rows are qlist * T + i, flagged queries are never
read in place, the padding rule holds both ways, and the group and chunk tables stay inside their bounds."""
import ctypes

import numpy as np
import pytest

from dino_tracker_b200 import _lib

RING, TILE, PAD_DIV, PROBE_MAPS = 4, 256, 16, 4096


def make_lists(kind, T, N, rs):
    """-> cnt [T], qlist [T][N] (ascending queries per frame), flag [N]"""
    keep = np.ones((T, N), dtype=bool)
    flag = np.zeros(N, dtype=np.uint8)
    if kind == "holes":
        keep = rs.rand(T, N) > 0.03
    elif kind == "alternating":
        keep[:, 1::2] = False
    elif kind == "ragged":
        keep = rs.rand(T, N) > 0.5
    elif kind == "empty_frames":
        keep[rs.randint(0, T, size=max(1, T // 3))] = False
    elif kind == "flagged":
        flag[rs.randint(0, N, size=max(1, N // 20))] = 1
    elif kind == "mixed":
        keep = rs.rand(T, N) > 0.02
        keep[:, N // 2:] &= (np.arange(N - N // 2) % 3 != 0)[None]
        flag[rs.randint(0, N, size=2)] = 1
    cnt = keep.sum(1).astype(np.int32)
    qlist = np.full((T, N), -1, dtype=np.int32)
    for a in range(T):
        qlist[a, :cnt[a]] = np.nonzero(keep[a])[0]
    return cnt, qlist, flag


def plan(T, N, cnt, qlist, flag, chunk, probe):
    lib = _lib.load()
    gcap = int(lib.dinotrk_infer_anchor_gcap(T, chunk))
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    n = ctypes.c_int(-1)
    assert lib.dinotrk_infer_plan_anchors(T, N, p(cnt), p(qlist), p(flag), chunk, probe, None, None, 0, ctypes.byref(n)) == 0
    groups = np.zeros((max(n.value, 1), 5, gcap), dtype=np.int32)
    meta = np.zeros((max(n.value, 1), 5), dtype=np.int32)
    n2 = ctypes.c_int(-1)
    assert lib.dinotrk_infer_plan_anchors(T, N, p(cnt), p(qlist), p(flag), chunk, probe, p(groups), p(meta), n.value,
                                          ctypes.byref(n2)) == 0
    assert n2.value == n.value
    return groups[:n.value], meta[:n.value], gcap


def run_lengths(qs, flag):
    """lengths of the maximal runs of consecutive unflagged queries covering each position of qs"""
    out = np.zeros(len(qs), dtype=np.int64)
    s = 0
    while s < len(qs):
        e = s + 1
        if not flag[qs[s]]:
            while e < len(qs) and qs[e] == qs[e - 1] + 1 and not flag[qs[e]]:
                e += 1
        out[s:e] = e - s
        s = e
    return out


KINDS = ["full", "holes", "alternating", "ragged", "empty_frames", "flagged", "mixed"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(3))
def test_anchor_rows_plan(kind, seed):
    rs = np.random.RandomState(1000 * KINDS.index(kind) + seed)
    T = int(rs.choice([7, 16, 30, 50, 64]))
    N = int(rs.choice([40, 97, 256]))
    chunk = int(rs.choice([T, 1000, 4096, 32768]))
    probe = int(seed % 2)
    cnt, qlist, flag = make_lists(kind, T, N, rs)
    groups, meta, gcap = plan(T, N, cnt, qlist, flag, chunk, probe)
    ch = max(chunk, T)
    cap = (ch // T) * T
    total = int(cnt.sum()) * T
    assert gcap <= T + 4 + 2 * (ch // 241)                                        # what sizes the workspace's group tables
    assert groups.shape[0] <= -(-N * T * T // cap) + 2
    seen, n_in, n_ga = [], 0, 0
    for k in range(groups.shape[0]):
        used, maxm, ng, no_thin, gathered = (int(x) for x in meta[k])
        f, r, m, map0, item = (groups[k, j, :ng].astype(np.int64) for j in range(5))
        assert 0 < used <= cap and 1 <= ng <= gcap and used % T == 0
        assert int(m.sum()) == used and int(m.max()) == maxm and (m > 0).all() and (m % T == 0).all()
        assert np.array_equal(map0, np.concatenate([[0], np.cumsum(m)[:-1]]))      # maps numbered consecutively
        if k + 1 < groups.shape[0]:
            first_cap = min(cap, max(T, PROBE_MAPS // T * T)) if (probe and k == 0) else cap
            assert used == first_cap                                               # only the last chunk may be partial
        chunk_row0 = N * T + (k % RING) * ch
        g_here = 0
        for j in range(ng):
            a = int(f[j])
            assert item[j] % T == 0
            slots = np.arange(item[j] // T, (item[j] + m[j]) // T)
            assert slots[-1] < cnt[a]
            qs = qlist[a, slots]
            seen += [(a, int(u)) for u in range(item[j], item[j] + m[j])]
            if r[j] < N * T:                                                        # read in place
                assert r[j] == qs[0] * T and np.array_equal(qs, qs[0] + np.arange(len(qs)))   # rows = qlist * T + i
                assert not flag[qs].any()
                pad = -(-m[j] // TILE) * TILE - m[j]
                assert pad * PAD_DIV <= m[j]
                n_in += int(m[j])
            else:                                                                   # gathered: the chunk's own rows
                assert r[j] == chunk_row0 + map0[j] and r[j] + m[j] <= chunk_row0 + ch
                if j > 0 and f[j - 1] == a:
                    assert r[j - 1] < N * T                                         # adjacent gathered runs are one group
                # no run inside a gathered group would have qualified (runs are cut at the group's / span's ends)
                span = [jj for jj in range(ng) if f[jj] == a]
                s_lo, s_hi = item[span[0]] // T, (item[span[-1]] + m[span[-1]]) // T
                rl = run_lengths(qlist[a, s_lo:s_hi], flag)[slots - s_lo] * T
                ok = (-(-rl // TILE) * TILE - rl) * PAD_DIV <= rl
                assert not (ok & (flag[qs] == 0)).any()
                g_here += int(m[j])
                n_ga += int(m[j])
        assert g_here == gathered
    assert seen == [(a, u) for a in range(T) for u in range(int(cnt[a]) * T)]       # every (anchor frame, item) once, in order
    assert n_in + n_ga == total
    if kind == "alternating" and T < 241:
        assert n_in == 0


def test_flagship_lists_are_read_in_place():
    """T = 50, 256 queries all anchored everywhere, 32 768-map chunks: every frame is one run, only a few spans cut short by
    a chunk boundary are gathered, and every chunk has few groups."""
    T, N = 50, 256
    cnt = np.full(T, N, dtype=np.int32)
    qlist = np.tile(np.arange(N, dtype=np.int32), (T, 1))
    groups, meta, _ = plan(T, N, cnt, qlist, np.zeros(N, dtype=np.uint8), 32768, 1)
    assert int(meta[:, 0].sum()) == N * T * T and int(meta[:, 4].sum()) * 50 <= N * T * T
    assert int(meta[:, 2].max()) <= 4
    same, _, _ = plan(T, N, cnt, qlist, np.zeros(N, dtype=np.uint8), 32768, 0)
    assert int(same[:, 2].sum()) > 0 and int(same.shape[0]) == 20


def test_rejects_lists_out_of_range():
    lib = _lib.load()
    T, N = 4, 5
    cnt = np.array([6, 0, 0, 0], dtype=np.int32)
    qlist = np.zeros((T, N), dtype=np.int32)
    flag = np.zeros(N, dtype=np.uint8)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    n = ctypes.c_int(0)
    assert lib.dinotrk_infer_plan_anchors(T, N, p(cnt), p(qlist), p(flag), 64, 0, None, None, 0, ctypes.byref(n)) != 0
    cnt[0] = 2
    qlist[0, 1] = 5
    assert lib.dinotrk_infer_plan_anchors(T, N, p(cnt), p(qlist), p(flag), 64, 0, None, None, 0, ctypes.byref(n)) != 0

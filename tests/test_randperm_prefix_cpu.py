"""CPU suite: ``dinotrk_randperm_prefix`` (the cycle-consistency term's pixel draws) against torch.randperm on the host
generator -- the prefix, the generator state afterwards and the draws that follow, from fresh and pre-advanced states
(offsets around the mt19937 624-word twist) and at the bench's mask sizes."""
import pytest
import torch

SIZES = [0, 1, 2, 623, 624, 625, 84_000, 322_504, 406_504]


def _ks(n):
    return sorted({0, 1, 77, 179, n, n + 5})


def _pair(seed, offset):
    a, b = torch.Generator().manual_seed(seed), torch.Generator().manual_seed(seed)
    if offset:
        torch.randperm(offset + 1, generator=a)          # exactly `offset` draws
        torch.randperm(offset + 1, generator=b)
    return a, b


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("seed,offset", [(0, 0), (1, 1), (2, 622), (3, 623), (4, 624), (5, 1247), (6, 1248)])
def test_prefix_and_state_match_torch_randperm(n, seed, offset):
    from dino_tracker_b200 import cycle
    for k in _ks(n):
        a, b = _pair(seed, offset)
        want = torch.randperm(n, generator=a)[:k]
        got = cycle._prefix_raw(b, n, k)
        assert got.dtype == torch.int64 and torch.equal(got, want), (n, k)
        assert torch.equal(a.get_state(), b.get_state()), (n, k)
        assert torch.equal(torch.randint(0, 1 << 30, (700,), generator=a), torch.randint(0, 1 << 30, (700,), generator=b))
        assert torch.equal(torch.rand(50, generator=a), torch.rand(50, generator=b))


def test_default_generator_draws_match_torch_randperm():
    """The entry the trainer calls: the default CPU generator, as ``torch.randperm(n)`` uses it."""
    from dino_tracker_b200 import cycle
    torch.manual_seed(11)
    want = [torch.randperm(n)[:k] for n, k in ((84_000, 179), (322_504, 77), (623, 179))]
    after = torch.rand(5)
    torch.manual_seed(11)
    got = [cycle.randperm_prefix(n, k) for n, k in ((84_000, 179), (322_504, 77), (623, 179))]
    assert cycle._prefix_checked is True
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert torch.equal(torch.rand(5), after)


def test_refuses_what_it_cannot_reproduce():
    import ctypes
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    state = torch.Generator().manual_seed(3).get_state()
    out = torch.empty(4, dtype=torch.int64)
    short = state[:-8].clone()
    assert lib.dinotrk_randperm_prefix(ctypes.c_void_p(short.data_ptr()), short.numel(), 10, 4,
                                       ctypes.c_void_p(out.data_ptr())) != 0
    assert lib.dinotrk_randperm_prefix(ctypes.c_void_p(state.data_ptr()), state.numel(), 2 ** 32 // 20, 4,
                                       ctypes.c_void_p(out.data_ptr())) != 0
    assert torch.equal(state, torch.Generator().manual_seed(3).get_state())     # refused calls leave the state alone

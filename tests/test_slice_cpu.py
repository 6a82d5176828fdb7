"""The host restatement of the slice sampler's random stream (tests/helpers.py `PhiloxDraws`): the Philox4x32-10
block function against Random123's known-answer vectors, and the cuRAND stream conventions built on it.
tests/test_slice_gpu.py then pins the stream to the kernel's own draws."""
import pytest

from tests.helpers import PhiloxDraws, philox4x32_10


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert philox4x32_10(ctr, key) == want


def test_stream_layout_follows_curand_init():
    """Key = the seed's two words, subsequence in the counter's high 64 bits, four words per block in order, then
    the counter's low 64 bits step by one (carrying into the high half)."""
    seed, sub = (7 << 32) | 0x1234, (3 << 32) | 5
    d = PhiloxDraws(seed, sub)
    key = (0x1234, 7)
    words = [d.word() for _ in range(12)]
    assert words[:4] == list(philox4x32_10((0, 0, 5, 3), key))
    assert words[4:8] == list(philox4x32_10((1, 0, 5, 3), key))
    assert words[8:] == list(philox4x32_10((2, 0, 5, 3), key))
    assert d.n_words == 12
    d.ctr = [0xffffffff, 0xffffffff, 0xffffffff, 0]
    d._next = 4
    assert d.word() == philox4x32_10((0, 0, 0, 1), key)[0]


def test_rand_and_shuffle_conventions():
    """rand() = 1 - (x * 2^-32 + 2^-32), exact in float64 and in [0, 1); shuffle is Fisher-Yates from the last
    position down with j = int(rand() * (i + 1)), one word per swap."""
    a, b = PhiloxDraws(11, 2), PhiloxDraws(11, 2)
    for _ in range(64):
        x = b.word()
        r = a.rand()
        assert r == 1.0 - (x + 1) / 2.0 ** 32 and 0.0 <= r < 1.0
    order = list(range(6))
    a.shuffle(order)
    want = list(range(6))
    for i in range(5, 0, -1):
        j = int((1.0 - (b.word() + 1) / 2.0 ** 32) * (i + 1))
        want[i], want[j] = want[j], want[i]
    assert order == want and sorted(order) == list(range(6))
    assert a.n_words == b.n_words == 64 + 5

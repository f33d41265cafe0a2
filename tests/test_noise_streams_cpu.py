"""The seeded noise streams without a GPU: the numpy Philox4x32-10 of cases_noise against the Random123 known answers,
and every stream's properties: a draw depends on (seed, stream, word 2, element) alone, and no two streams or word-2
values of one seed share a value.  The GPU tests compare each kernel's noise with `cases_noise.normals`."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases_noise as CN  # noqa: E402

SEEDS = (0, 7, 2 ** 63 + 1, 2 ** 64 - 1)
WORDS = (0, 1, 981)  # word 2: a step index / image index / timestep


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123's known-answer vectors for Philox4x32-10."""
    got = CN.philox4x32([np.uint32(c) for c in ctr], [np.uint32(k) for k in key])
    assert [int(v) for v in got.reshape(-1)] == list(want)


@pytest.mark.parametrize("name", list(CN.STREAMS))
def test_stream(name):
    s = CN.STREAMS[name]
    z = CN.normals(123, s, 7, 4099)
    assert np.array_equal(z[:10], CN.normals(123, s, 7, 10))  # a prefix does not depend on the length
    assert not np.array_equal(z[:16], CN.normals(124, s, 7, 16))
    assert not np.array_equal(z[:16], CN.normals(123, s, 6, 16))  # word 2 changes the draw
    for high, low in ((2 ** 40 + 5, 5), (2 ** 64 - 1, 2 ** 32 - 1)):  # both seed words enter the key
        big = CN.normals(high, s, 3, 1 << 16)
        assert not np.array_equal(big[:16], CN.normals(low, s, 3, 16))
        assert abs(big.mean()) < 5 / 256 and abs(big.var() - 1) < 0.02
    z = CN.normals(123, s, 500, 200000)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01

    n = 4 * 4096 + 3
    for seed in SEEDS:
        draws = {(t, w): CN.normals(seed, t, w, n) for t in CN.STREAMS.values() for w in WORDS}
        for w in WORDS:
            mine = draws[(s, w)]
            assert np.array_equal(CN.normals(seed, s, w, 10), mine[:10])
            # disjoint from every other stream of the seed, and from this stream at another word 2
            others = np.concatenate([v for k, v in draws.items() if k != (s, w)])
            assert not np.isin(mine, others).any()
        # the first groups are Box-Muller on the Philox words at counter (c, 0, word 2, stream)
        for w in (0, 21):
            c = np.arange(3, dtype=np.uint64)
            words = CN.philox4x32([c, np.zeros(3, np.uint32), np.full(3, w, np.uint32), np.full(3, s, np.uint32)],
                                  [np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32)])
            u = (words.astype(np.float64) + 0.5) * 2.0 ** -32
            r01, r23 = np.sqrt(-2 * np.log(u[0])), np.sqrt(-2 * np.log(u[2]))
            want = np.stack([r01 * np.cos(2 * np.pi * u[1]), r01 * np.sin(2 * np.pi * u[1]),
                             r23 * np.cos(2 * np.pi * u[3]), r23 * np.sin(2 * np.pi * u[3])], 1).reshape(-1)
            assert np.allclose(CN.normals(seed, s, w, 12), want, rtol=0, atol=1e-12)

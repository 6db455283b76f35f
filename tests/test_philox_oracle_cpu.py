"""CPU suite: the Philox4x32-10 oracle of the rollout's in-kernel generator (oracle/philox_oracle.py).  The block function against the
published known-answer vectors, the two fp32 uniform mappings over every one of their 2^24 codes, the distributions of the draws built on
them at 2^20 samples, the independence of neighbouring rows, groups, calls and streams, and the edge draws the GPU tests replay."""
import numpy as np
import pytest
from scipy import stats

import philox_oracle as P

N20 = 1 << 20

# Draws whose top 24 bits are all ones, so that the (0, 1] mapping gives exactly 1.0.  12345 is the agent's seed word at seed 0, rank 0.
# (seed, call, stream, group, word, row): the Bernoulli draw of policy_sample_rng(stream_id=0) at row 909 of 1024, and the task uniforms
# of stream 0 (reset mode of ase_task_resample) at env 1420 (reach height, u[2]) and env 3612 (location / reach offset, u[0]) of 4096.
EDGE_BERNOULLI = dict(seed=12345, call=3636, sid=1, group=P.GROUP_BERNOULLI, word=0, row=909, rows=1024)
EDGE_REACH_HEIGHT = dict(seed=12345, call=1086, sid=0, group=0, word=2, row=1420, rows=4096)
EDGE_OFFSET = dict(seed=12345, call=103, sid=0, group=0, word=0, row=3612, rows=4096)


def _hex(ws):
    return [f'{int(w):08x}' for w in ws]


@pytest.mark.parametrize('ctr,key,want', [
    ((0, 0, 0, 0), (0, 0), '6627e8d5 e169c58d bc57ac4c 9b00dbd8'),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, '408f276d 41c83b0e a20bc7c6 6d5451fd'),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), 'd16cfe09 94fdcceb 5001e420 24126ea1'),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    assert _hex(P.philox4x32_10(ctr, key)) == want.split()
    # vectorised: the same block at every position of an array
    out = P.philox4x32_10(tuple(np.full(5, c, dtype=np.uint64) for c in ctr), key)
    assert all(_hex(w) == [x] * 5 for w, x in zip(out, want.split()))


def test_addressing_reads_int64_as_uint64():
    assert P.key_of(-1, 0) == (0xFFFFFFFF, 0xFFFFFFFF)
    assert P.key_of(-2 ** 63, 0) == (0, 0x80000000)
    assert P.key_of(0x123456789, 3) == (0x23456789, 0x1 ^ ((3 * 0x9E3779B1) & 0xFFFFFFFF))
    # call >= 2^32 fills counter words 2 and 3; a negative call wraps like the seed
    rows = np.arange(7)
    for call in (2 ** 32 + 5, -3):
        c = call % 2 ** 64
        want = P.philox4x32_10((rows, 9, c & 0xFFFFFFFF, c >> 32), P.key_of(-77, 2))
        got = P.words(-77, call, 2, rows, 9)
        assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_u01_closed_and_open_over_all_codes():
    codes = np.arange(1 << 24, dtype=np.uint64)
    for low in (0, 0xFF):                          # the low 8 bits of a word do not matter
        x = (codes << np.uint64(8)) | np.uint64(low)
        c, o = P.u01_closed(x), P.u01_open(x)
        assert c.dtype == np.float32 and o.dtype == np.float32
        # (0, 1]: smallest 2^-25, largest exactly 1.0, reached by the top code alone
        assert c.min() == np.float32(2.0 ** -25) and c.max() == np.float32(1.0)
        assert np.nonzero(c == 1.0)[0].tolist() == [0xFFFFFF]
        assert np.all(np.diff(c) >= 0)
        # below 2^23 the +0.5 is exact; above, it rounds half to even
        k = codes.astype(np.float64)
        exact = (k + 0.5) / 2 ** 24
        assert np.array_equal(c[: 1 << 23].astype(np.float64), exact[: 1 << 23])
        hi = codes[1 << 23:]
        assert np.array_equal(c[1 << 23:].astype(np.float64), (hi + (hi & np.uint64(1))).astype(np.float64) / 2 ** 24)
        # (0, 1): the same values except the top code, which becomes the largest float32 below 1
        assert o.min() == np.float32(2.0 ** -25) and o.max() == np.float32(1.0 - 2.0 ** -24) and np.all(o < 1.0)
        assert np.array_equal(o[:-1], c[:-1]) and o[-1] == np.nextafter(np.float32(1), np.float32(0))


def test_normals_distribution():
    z = P.normals(seed=2024, call=7, sid=0, n=N20 // 16, cols=16).ravel()
    assert z.size == N20 and np.all(np.isfinite(z))
    assert stats.kstest(z, 'norm').pvalue > 1e-3
    n = z.size
    assert abs(z.mean()) < 5 / np.sqrt(n)
    assert abs(z.var() - 1.0) < 5 * np.sqrt(2.0 / n)
    assert abs(stats.skew(z)) < 5 * np.sqrt(6.0 / n)
    assert abs(stats.kurtosis(z)) < 5 * np.sqrt(24.0 / n)
    # the largest radius the mapping can give: u = 2^-25
    assert np.abs(z).max() <= np.sqrt(-2.0 * np.log(2.0 ** -25)) + 1e-12


def test_normals_column_layout():
    """Column j of a row comes from group j // 4: a ragged width is the prefix of the next multiple of 4, and the pairs share a radius."""
    z7, z8 = P.normals(5, 11, 1, 33, 7), P.normals(5, 11, 1, 33, 8)
    assert np.array_equal(z7, z8[:, :7])
    r = np.hypot(z8[:, 0::2], z8[:, 1::2])
    x, _, zz, _ = P.words(5, 11, 1, np.arange(33), 1)
    assert np.allclose(r[:, 2], np.sqrt(-2 * np.log(P.u01_closed(x).astype(np.float64))), rtol=1e-14)
    assert np.allclose(r[:, 3], np.sqrt(-2 * np.log(P.u01_closed(zz).astype(np.float64))), rtol=1e-14)


def _exact_bernoulli_probability(p):
    """P(u_open < p) over the 2^24 equally likely codes."""
    u = P.u01_open(np.arange(1 << 24, dtype=np.uint64) << np.uint64(8))
    return float(np.count_nonzero(u < np.float32(p))) / (1 << 24)


@pytest.mark.parametrize('p', [0.0, 0.3, 1.0 - np.exp(-10.0), 1.0])
def test_bernoulli_frequencies(p):
    m = P.bernoulli(seed=99, call=3, sid=0, p=np.full(N20, p, dtype=np.float32))
    assert set(np.unique(m).tolist()) <= {0.0, 1.0}
    q = _exact_bernoulli_probability(p)
    if p in (0.0, 1.0):
        assert q == p and np.all(m == p)
        return
    assert abs(q - np.float32(p)) <= 2 ** -23        # above 1/2 two codes share each value
    k = m.sum()
    assert abs(k - N20 * q) < 5 * np.sqrt(N20 * q * (1 - q)) + 1, (k, N20 * q)


def test_randint_chi_square_and_width_one():
    x = P.randint(seed=31, call=2 ** 33 + 1, sid=2, n=N20, lo=1, hi=150)
    assert x.min() == 1 and x.max() == 149
    counts = np.bincount(x - 1, minlength=149)
    assert stats.chisquare(counts).pvalue > 1e-3
    for lo, hi in ((5, 6), (5, 5)):               # width 1, and an empty range, give lo
        assert np.all(P.randint(31, 0, 2, 4096, lo, hi) == lo)


def test_latents_uniform_on_the_sphere():
    zdim, n = 64, N20 // 64
    v = P.latents(seed=8, call=12, sid=2, n=n, dim=zdim)
    assert np.allclose(np.linalg.norm(v, axis=-1), 1.0, rtol=0, atol=1e-12)
    assert np.abs(v.mean(0)).max() < 5 / np.sqrt(zdim * n)
    cov = v.T @ v / n
    assert np.abs(cov - np.eye(zdim) / zdim).max() < 6 / (zdim * np.sqrt(n))


def _corr(a, b):
    return float(np.corrcoef(P.u01_closed(a).astype(np.float64), P.u01_closed(b).astype(np.float64))[0, 1])


def test_neighbouring_rows_groups_calls_and_streams_are_uncorrelated():
    rows = np.arange(N20)
    bound = 5 / np.sqrt(N20)
    base = P.words(4, 10, 0, rows, 0)
    neighbours = {'row': P.words(4, 10, 0, rows + 1, 0), 'group': P.words(4, 10, 0, rows, 1), 'call': P.words(4, 11, 0, rows, 0),
                  'stream': P.words(4, 10, 1, rows, 0), 'seed': P.words(5, 10, 0, rows, 0), 'call_hi': P.words(4, 10 + 2 ** 32, 0, rows, 0)}
    for name, other in neighbours.items():
        for w in range(4):
            assert abs(_corr(base[w], other[w])) < bound, (name, w)
    for w in range(1, 4):                          # the words of one block
        assert abs(_corr(base[0], base[w])) < bound, w


@pytest.mark.parametrize('edge', [EDGE_BERNOULLI, EDGE_REACH_HEIGHT, EDGE_OFFSET], ids=['bernoulli', 'reach_height', 'offset'])
def test_edge_draws_hit_the_top_code(edge):
    """The GPU edge tests replay these draws: each is the only top-code word of its launch, the (0, 1] mapping gives 1.0 and the (0, 1)
    mapping does not."""
    w = P.words(edge['seed'], edge['call'], edge['sid'], np.arange(edge['rows']), edge['group'])[edge['word']]
    assert np.nonzero((w >> np.uint64(8)) == 0xFFFFFF)[0].tolist() == [edge['row']]
    assert P.u01_closed(w[edge['row']]) == 1.0 and P.u01_open(w[edge['row']]) < 1.0
    if edge is EDGE_BERNOULLI:
        assert np.all(P.bernoulli(edge['seed'], edge['call'], edge['sid'] - 1, np.ones(edge['rows'])) == 1.0)
    else:
        u = P.uniforms(edge['seed'], edge['call'], edge['sid'], edge['rows'])
        assert u.max() < 1.0 and u[edge['row'], edge['word']] == np.float32(1.0 - 2.0 ** -24)


def test_latent_update_semantics():
    n, zdim = 6, 5
    lat = np.full((n, zdim), 7.0)
    steps = np.array([3, 3, 10, 2 ** 31 - 1, 5, 0])
    prog = np.array([0, 3, 9, 2 ** 31 + 5, 4, 0])
    done = np.array([1, 0, 0, 0, 0, 1])
    new, s, touched = P.latent_update(lat, steps, prog, done, 1, 150, seed=3, call=4, sid=2)
    r = P.randint(3, 4, 2, n, 1, 150)
    assert touched.tolist() == [True, True, False, True, False, True]
    assert s.tolist() == [r[0], 3 + r[1], 10, 2 ** 31 - 1 + r[3], 5, r[5]]
    assert np.all(new[~touched] == 7.0)
    assert np.allclose(new[touched], P.latents(3, 4, 2, n, zdim)[touched], rtol=0, atol=0)

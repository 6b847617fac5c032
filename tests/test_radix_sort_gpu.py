"""The device radix sort on its own (radix_sort_kernel, csrc/radix_sort.cu, through lb200_radix_sort_device), held to its contract: a stable
sort of (u64 key, u64 value) pairs by key.  The reference is np.argsort(kind="stable"), and for up to a few thousand pairs also the oracle's
restatement of the reference's own PipelineImpl::radixSort; the device result must equal it element for element.  Values are mostly the
input positions, so that any pair of equal keys that changes order shows.

G is the grid an unconstrained sort launches and T = G * 8192 the largest n the register path takes (512 threads x 16 keys per block).
Cases cover both paths, the sizes where the keys per thread or the path change, grids from 1 block to G, digit windows that the data
places (none, bit 0, bit 63, one window across a byte border, eight windows), the count read on the device below and above the capacity,
and sorts enqueued back to back on the shared scratch."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import sortkeys

pytestmark = pytest.mark.gpu

THREADS, REG_ITEMS, TILE = 512, 16, 2048
SENT_KEY, SENT_VALUE = np.uint64(0xA5A5_5A5A_DEAD_BEEF), np.uint64(0x0123_4567_89AB_CDEF)
ORACLE_MAX = 4096  # up to here the oracle's restatement of the reference sort is compared too
U64_MAX = np.iinfo(np.uint64).max


@pytest.fixture(scope="module")
def G(ctx):
    """Blocks of an unconstrained sort: the capacity (ceil(cap / 2048) blocks at most) is large enough not to limit it."""
    cap = 1 << 20
    _, _, g = lb.radix_sort(ctx, np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), count=0)
    assert 64 < g < cap // TILE, "the grid cases below assume more than 64 co-resident blocks"
    return g


def _rand64(rng, n):
    return rng.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)


def _expected(keys, values, oracle):
    o = np.argsort(keys, kind="stable")
    ek, ev = keys[o], values[o]
    if oracle is not None and len(keys) <= ORACLE_MAX:
        ok, ov = oracle.radix_sort(keys, values)
        assert np.array_equal(ok, ek) and np.array_equal(ov, ev), "the oracle's sort disagrees with a stable argsort"
    return ek, ev


def _sort(ctx, keys, values, room=0, max_blocks=0, tiled=False):
    """Device sort of the n = len(keys) pairs in a buffer of cap = n + room whose tail holds sentinels (the count word is n).
    -> (sorted keys, sorted values, grid); the tail is checked to be untouched."""
    n = len(keys)
    k = np.full(n + room, SENT_KEY, np.uint64)
    v = np.full(n + room, SENT_VALUE, np.uint64)
    k[:n], v[:n] = keys, values
    gk, gv, grid = lb.radix_sort(ctx, k, v, count=n, max_blocks=max_blocks, tiled=tiled)
    assert np.all(gk[n:] == SENT_KEY) and np.all(gv[n:] == SENT_VALUE), "entries past the count were written"
    return gk[:n], gv[:n], grid


def _path(n, grid, tiled):
    return "tiled" if tiled or n > grid * THREADS * REG_ITEMS else "register"


def _check(ctx, oracle, keys, values, room=0, max_blocks=0, tiled=False):
    """Sorts on the device and compares with the stable reference exactly.  -> (keys, values, grid, path)."""
    gk, gv, grid = _sort(ctx, keys, values, room, max_blocks, tiled)
    path = _path(len(keys), grid, tiled)
    ek, ev = _expected(keys, values, oracle)
    assert np.array_equal(gk, ek), f"keys differ from a stable sort (n={len(keys)}, grid={grid}, {path} path)"
    assert np.array_equal(gv, ev), f"values differ from a stable sort (n={len(keys)}, grid={grid}, {path} path): order among equal keys"
    return gk, gv, grid, path


def _both_paths(ctx, oracle, keys, values, room=0, max_blocks=0):
    """The automatic choice and the forced tiled path: each equal to the reference, and to each other.  -> (grid, automatic path)."""
    ak, av, grid, path = _check(ctx, oracle, keys, values, room, max_blocks, tiled=False)
    tk, tv, tgrid, _ = _check(ctx, oracle, keys, values, room, max_blocks, tiled=True)
    assert tgrid == grid
    assert np.array_equal(tk, ak) and np.array_equal(tv, av), "the tiled path disagrees with the register path"
    return grid, path


def _keys_with_ties(rng, n):
    """Random 64-bit keys (every digit window in play) drawn from about n / 8 distinct values: long enough runs of equal keys."""
    pool = _rand64(rng, max(2, n // 8))
    return pool[rng.integers(0, len(pool), n)]


# (id, n as a function of G, the path the automatic choice must take, or None where n alone does not fix it)
SIZES = [(str(n), (lambda n: lambda G: n)(n), None) for n in (0, 1, 2, 3, 31, 32, 33, 511, 512, 513, 2047, 2048, 2049)] + [
    ("G*512-1", lambda G: G * 512 - 1, "register"),    # 1 key per thread
    ("G*512", lambda G: G * 512, "register"),
    ("G*512+1", lambda G: G * 512 + 1, "register"),    # 2 keys per thread
    ("15*G*512+1", lambda G: 15 * G * 512 + 1, "register"),  # 16 keys per thread
    ("T-1", lambda G: G * 8192 - 1, "register"),
    ("T", lambda G: G * 8192, "register"),
    ("T+1", lambda G: G * 8192 + 1, "tiled"),
    ("3T+12345", lambda G: 3 * G * 8192 + 12345, "tiled"),  # several tiles per block, partial last tile
]


@pytest.mark.parametrize("size,auto_path", [(s[1], s[2]) for s in SIZES], ids=[s[0] for s in SIZES])
def test_sizes(ctx, oracle, G, size, auto_path):
    """Sizes at the early return (n < 2), warp / block / tile borders, where the keys per thread go from 1 to 2 and reach 16, and where the
    path switches.  In a roomy buffer (sentinel tail) the grid is G; below G * 2048 pairs the sort also runs with cap = n, where the
    capacity limits the grid to ceil(n / 2048) blocks."""
    n = size(G)
    rng = np.random.default_rng(n + 1)
    keys, values = _keys_with_ties(rng, n), np.arange(n, dtype=np.uint64)
    grid, path = _both_paths(ctx, oracle, keys, values, room=max(0, G * TILE - n) + 777)
    assert grid == G
    if auto_path is not None:
        assert path == auto_path, f"n = {n} on a grid of {grid} took the {path} path"
    if n < G * TILE:
        grid, _ = _both_paths(ctx, oracle, keys, values)
        assert grid == max(1, -(-n // TILE))


GRIDS = [("1", lambda G: 1), ("2", lambda G: 2), ("3", lambda G: 3), ("7", lambda G: 7), ("64", lambda G: 64), ("G-1", lambda G: G - 1), ("G", lambda G: G)]


@pytest.mark.parametrize("blocks", [g[1] for g in GRIDS], ids=[g[0] for g in GRIDS])
def test_grids(ctx, oracle, G, blocks):
    """max_blocks from 1 to G, each at a few sizes and on both paths: 5000 pairs (on the tiled path at G most blocks own no tile), 2 keys
    per thread, the largest register-path size g * 8192 and one more (at g = 1: one block on the tiled path with 5 tiles)."""
    g = blocks(G)
    rng = np.random.default_rng(g)
    for n in (5000, g * 512 + 1, g * 8192, g * 8192 + 1):
        keys = _keys_with_ties(rng, n)
        room = max(0, g * TILE - n) + 100  # the capacity does not limit the grid
        grid, path = _both_paths(ctx, oracle, keys, np.arange(n, dtype=np.uint64), room=room, max_blocks=g)
        assert grid == g
        assert path == ("tiled" if n > g * 8192 else "register")


def test_tiled_with_blocks_that_own_no_tile(ctx, oracle, G):
    """3 tiles dealt to G blocks: G - 3 blocks count nothing, scatter nothing and still take part in every grid barrier."""
    rng = np.random.default_rng(5)
    n = 5000
    keys = _keys_with_ties(rng, n)
    _, _, grid, path = _check(ctx, oracle, keys, np.arange(n, dtype=np.uint64), room=G * TILE, tiled=True)
    assert grid == G and path == "tiled"


def test_one_block_tiled(ctx, oracle):
    """max_blocks = 1, n = 8193: one block walks 5 tiles, the last with one key."""
    rng = np.random.default_rng(6)
    n = 8193
    keys = _keys_with_ties(rng, n)
    _, _, grid, path = _check(ctx, oracle, keys, np.arange(n, dtype=np.uint64), max_blocks=1)
    assert grid == 1 and path == "tiled"


def _pattern(name, rng, n):
    """-> (keys, values) of a key pattern; values are the positions unless the pattern says otherwise."""
    pos = np.arange(n, dtype=np.uint64)
    base = np.uint64(0x5A00_0000_0000_0000)
    bit = lambda b: rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(b)  # noqa: E731
    if name == "all_equal":  # no bit varies: no pass runs and the pairs stay in input order
        return np.full(n, np.uint64(0x0123_4567_89AB_CDEF), np.uint64), pos
    if name == "bit0":
        return base | bit(0), pos
    if name == "bit63":
        return (base >> np.uint64(1)) | bit(63), pos
    if name == "bits7_8":  # one digit window over bits 7..14, across the byte border
        return base | bit(7) | bit(8), pos
    if name == "create_sort_keys":  # bucket << 56 | 20-bit key, the shape createSortKeys emits; random 64-bit values
        bucket = rng.integers(0, 4, n, dtype=np.uint64)
        return (bucket << np.uint64(56)) | rng.integers(0, 1 << 20, n, dtype=np.uint64), _rand64(rng, n)
    if name == "random64":  # eight passes; random 64-bit values
        return _rand64(rng, n), _rand64(rng, n)
    if name == "few_runs":  # a few distinct keys in long runs
        distinct = _rand64(rng, 5)
        return np.repeat(distinct[rng.integers(0, 5, 64)], -(-n // 64))[:n].copy(), pos
    if name == "sorted":
        return np.sort(_keys_with_ties(rng, n)), pos
    if name == "reverse_sorted":
        return np.sort(_keys_with_ties(rng, n))[::-1].copy(), pos
    if name == "zero_and_ones":
        return np.where(rng.random(n) < 0.5, np.uint64(0), np.uint64(U64_MAX)).astype(np.uint64), pos
    raise ValueError(name)


PATTERNS = ["all_equal", "bit0", "bit63", "bits7_8", "create_sort_keys", "random64", "few_runs", "sorted", "reverse_sorted", "zero_and_ones"]


@pytest.mark.parametrize("large", [False, True], ids=["n=3000", "n=T-1000"])
@pytest.mark.parametrize("pattern", PATTERNS)
def test_key_patterns(ctx, oracle, G, pattern, large):
    """Each key pattern at a small size and at T - 1000 (16 keys per thread), on the register path and on the tiled path."""
    n = G * 8192 - 1000 if large else 3000
    keys, values = _pattern(pattern, np.random.default_rng([PATTERNS.index(pattern), n]), n)
    room = max(0, G * TILE - n) + 100
    grid, path = _both_paths(ctx, oracle, keys, values, room=room)
    assert grid == G and path == "register"


@pytest.mark.parametrize("n_fn", [lambda G: 100_000, lambda G: G * 8192 + 5], ids=["100000", "T+5"])
def test_count_below_cap(ctx, oracle, G, n_fn):
    """*dev_count < cap: the first count pairs are sorted, the sentinels behind them come back unchanged."""
    n = n_fn(G)
    rng = np.random.default_rng(n)
    keys = _keys_with_ties(rng, n)
    _both_paths(ctx, oracle, keys, np.arange(n, dtype=np.uint64), room=54_321)


@pytest.mark.parametrize("over", [1, 5000, 1 << 31])
@pytest.mark.parametrize("cap_fn", [lambda G: 50_000, lambda G: G * 8192 + 100], ids=["50000", "T+100"])
@pytest.mark.parametrize("tiled", [False, True], ids=["auto", "tiled"])
def test_count_above_cap(ctx, oracle, G, cap_fn, over, tiled):
    """*dev_count > cap: exactly cap pairs are sorted."""
    cap = cap_fn(G)
    rng = np.random.default_rng(cap + over)
    keys = _keys_with_ties(rng, cap)
    values = np.arange(cap, dtype=np.uint64)
    gk, gv, grid = lb.radix_sort(ctx, keys, values, count=min(cap + over, 0xffffffff), tiled=tiled)
    ek, ev = _expected(keys, values, oracle)
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev)
    assert grid == min(G, -(-cap // TILE))


def test_back_to_back(ctx, oracle, G):
    """Four sorts on different buffers enqueued with nothing waiting between them: each launch resets the shared sort state and block
    histograms on the stream.  The largest capacity goes first, so that the context's scratch is grown (which waits) before the first."""
    rng = np.random.default_rng(77)
    T = G * 8192
    cases = [  # (n, cap, max_blocks, tiled)
        (3 * T + 7, 3 * T + 7, 0, False),   # tiled, 8 passes
        (T - 5, T - 5, 0, False),           # register path, 16 keys per thread
        (40_000, G * TILE, 0, True),        # tiled, most blocks own no tile
        (1000, 3 * TILE, 3, False),         # 3 blocks
    ]
    inputs, dev = [], []
    for n, cap, max_blocks, tiled in cases:
        k = np.full(cap, SENT_KEY, np.uint64)
        v = np.full(cap, SENT_VALUE, np.uint64)
        k[:n], v[:n] = _keys_with_ties(rng, n), np.arange(n, dtype=np.uint64)
        inputs.append((k[:n].copy(), v[:n].copy()))
        dev.append([ctx.to_device(k), ctx.to_device(v), ctx.to_device(np.array([n], np.uint32))])
    try:
        grids = [sortkeys.radix_sort_device(ctx, d[0], d[1], d[2], cap, max_blocks, tiled) for d, (_, cap, max_blocks, tiled) in zip(dev, cases)]
        assert grids == [G, G, G, 3]
        for (n, cap, _, _), d, (k, v) in zip(cases, dev, inputs):
            gk, gv = ctx.copy_to_host(d[0], cap, np.uint64), ctx.copy_to_host(d[1], cap, np.uint64)
            ek, ev = _expected(k, v, oracle)
            assert np.array_equal(gk[:n], ek) and np.array_equal(gv[:n], ev), f"sort of {n} pairs enqueued back to back"
            assert np.all(gk[n:] == SENT_KEY) and np.all(gv[n:] == SENT_VALUE)
    finally:
        for d in dev:
            for p in d:
                ctx.free_device(p)

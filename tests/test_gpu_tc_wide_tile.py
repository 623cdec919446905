"""The similarity kernel with 128-row corpus tiles (wgmma m64n128) against the same index searched with 64-row tiles.
Every search is held to the fp64 oracle, and the two widths must return identical ids and scores: the final scores are
the exact re-rank's fp64 re-scores of the same rows, so once the candidates agree the scores agree bit for bit.  The
shapes are where the wide tile differs from the narrow one: a last 128-row tile that is partial (with the best row of
some queries at the very last row), fewer rows than one tile, CTAs with odd and even tile counts in one launch, one and
twelve k-blocks, partial query blocks, the k at which the 128-row layout stops fitting, tenant-scope bit masks, id
subsets and tombstones."""

from __future__ import annotations

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index
from oracle import cosine_topk as O
from tests.gpu_exact import check_exact, dev_search
from tests.test_gpu_tc_pipeline import tile_sets
from tests.test_tc_tile_rule import NARROW, WIDE, auto_tile, largest_wide_k

pytestmark = pytest.mark.gpu
KSLACK = 8


def _sm_count() -> int:
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def _data(n, d, nq, seed, last_row_queries=0):
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    for i in range(nq):   # a few close rows per query, spread over the tiles
        for r in rng.choice(n, min(3, n), replace=False):
            C[r] = Q[i] + 0.3 * rng.standard_normal(d).astype(np.float32)
    for i in range(min(last_row_queries, nq)):   # the best row of these queries is the corpus's last row
        Q[i] = C[n - 1] + 0.05 * rng.standard_normal(d).astype(np.float32)
    return O.round_to_bf16(C), O.round_to_bf16(Q)


def _search(ix, Q, k, tile, **kw):
    N.check(ix._lib.aur_set_option(ix._h, b"tc_tile", tile))
    got = dev_search(ix, Q, k, **kw)
    assert ix.stats()["last_tile_n"] == tile
    return got


def _both_widths(ix, Q, C, k, kernels=(N.KERNEL_TC1, N.KERNEL_TC2), oracle_kw=None, **kw):
    """Searches with 128- and 64-row tiles under each kernel; every result is held to the oracle and to the others."""
    oracle_kw = oracle_kw or {}
    want = O.cosine_topk(Q, C, k, return_f64=True, **oracle_kw)
    runs = []
    for kern in kernels:
        ix.set_kernel(kern)
        for tile in (WIDE, NARROW):
            got = _search(ix, Q, k, tile, **kw)
            assert ix.stats()["last_kernel"] == kern
            check_exact(got, Q, C, k, want=want)
            runs.append(got)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert np.array_equal(a, b), "the 128-row and 64-row tiles (or TC1 and TC2) differ"
    return want


@pytest.mark.parametrize("rem", [1, 63, 64, 65, 127])
def test_partial_last_tile_with_best_row_last(rem):
    """n = 128 m + rem: the last tile's missing rows come in as TMA's zero fill and are masked by the row-count guard on
    the inverse norms; queries 0..3 find their best row at the corpus's very last row."""
    d, nq, k = 64, 65, 32
    n = 128 * 40 + rem
    C, Q = _data(n, d, nq, seed=rem, last_row_queries=4)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        want = _both_widths(ix, Q, C, k)
    assert (want[0][:4, 0] == n - 1).all()


@pytest.mark.parametrize("n", [1, 37, 100, 127])
def test_fewer_rows_than_one_tile(n):
    d, nq, k = 576, 64, 10
    C, Q = _data(n, d, nq, seed=n, last_row_queries=2)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_widths(ix, Q, C, k)


# (kernel whose geometry sets the corpus size, dim, nq, k, 128-row tiles per CTA or pair); the corpus holds
# tile_sets * tiles + tile_sets // 2 wide tiles, so half the CTAs take one tile more than the other half
@pytest.mark.parametrize("kernel,d,nq,k,tiles", [
    (N.KERNEL_TC1, 64, 1, 1, 3),        # one k-block per tile, one query
    (N.KERNEL_TC1, 576, 128, 32, 4),
    (N.KERNEL_TC2, 64, 257, 32, 4),     # a partial third CTA pair
    (N.KERNEL_TC2, 576, 512, 32, 5),    # four query super-blocks sharing every tile
    (N.KERNEL_TC2, 768, 256, 32, 6),    # the benchmark's shape
])
def test_tile_counts_and_query_blocks(kernel, d, nq, k, tiles):
    ts = tile_sets(kernel, nq, k + KSLACK, _sm_count())
    n = (ts * tiles + ts // 2) * WIDE
    C, Q = _data(n, d, nq, seed=d + nq + tiles)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_widths(ix, Q, C, k, kernels=(kernel,))


@pytest.mark.parametrize("nq", [1, 64, 65, 128, 256, 257, 512])
def test_query_counts(nq):
    d, k, n = 768, 32, 30_000
    C, Q = _data(n, d, nq, seed=nq)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_widths(ix, Q, C, k)


def test_auto_width_follows_the_rule_at_its_edge():
    """Auto takes 128-row tiles up to the largest k whose layout keeps four ring stages and 64-row tiles above it; a
    forced 128 where not even two stages fit is refused."""
    d, nq, n = 768, 256, 20_000
    kmax = largest_wide_k(d)
    C, Q = _data(n, d, nq, seed=3)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        for k in (1, kmax, kmax + 1):
            _both_widths(ix, Q, C, k)
            N.check(ix._lib.aur_set_option(ix._h, b"tc_tile", 0))
            got = dev_search(ix, Q, k)
            assert ix.stats()["last_tile_n"] == auto_tile(d, k + KSLACK)
            check_exact(got, Q, C, k)
        assert auto_tile(d, kmax + KSLACK) == WIDE and auto_tile(d, kmax + 1 + KSLACK) == NARROW
        N.check(ix._lib.aur_set_option(ix._h, b"tc_tile", WIDE))
        q = ix._rows_buffer(Q[:8])
        dq, ds, di = DeviceBuffer(q.nbytes).upload(q), DeviceBuffer(8 * 128 * 4), DeviceBuffer(8 * 128 * 8)
        assert ix._lib.aur_search_dev(ix._h, dq.ptr, 8, 128, None, None, ds.ptr, di.ptr, None, None) == N.AUR_ERR_UNSUPPORTED
        assert ix._lib.aur_set_option(ix._h, b"tc_tile", 96) == N.AUR_ERR_INVALID


def test_scopes_subsets_and_tombstones():
    """Up to 32 tenant scopes in one batch (row bit masks, the kMask kernels), an id subset and tombstones."""
    d, nq, k, n = 768, 200, 16, 128 * 150 + 77
    C, Q = _data(n, d, nq, seed=11)
    rng = np.random.default_rng(12)
    ru = rng.integers(0, 40, n).astype(np.int32)
    ro = rng.integers(-1, 6, n).astype(np.int32)
    live = np.ones(n, dtype=bool)
    qu = rng.integers(0, 20, nq).astype(np.int32)
    qo = (qu % 7 - 1).astype(np.int32)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), ru, ro)
        gone = np.concatenate([rng.choice(n, 300, replace=False), [n - 1]]).astype(np.int64)
        ix.remove(gone)
        live[gone] = False
        _both_widths(ix, Q, C, k, oracle_kw=dict(live=live))
        allow = np.sort(rng.choice(n, n // 3, replace=False)).astype(np.int64)
        sub = np.zeros(n, dtype=bool)
        sub[allow] = True
        # the host entry points: the scoped batch's distinct scopes are gathered there (the kMask kernels)
        for search, oracle_kw in ((lambda: ix.search(Q, k, qu, qo), dict(live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo)),
                                  (lambda: ix.search_subset(Q, k, allow), dict(live=live & sub))):
            want = O.cosine_topk(Q, C, k, **oracle_kw)
            res = []
            for kern in (N.KERNEL_TC1, N.KERNEL_TC2):
                ix.set_kernel(kern)
                for tile in (WIDE, NARROW):
                    N.check(ix._lib.aur_set_option(ix._h, b"tc_tile", tile))
                    ids, sc = search()
                    assert ix.stats()["last_kernel"] == kern and ix.stats()["last_tile_n"] == tile
                    assert np.array_equal(ids, want[0]), f"{int((ids != want[0]).sum())} id mismatches"
                    res.append((ids, sc))
            for ids, sc in res[1:]:
                assert np.array_equal(ids, res[0][0]) and np.array_equal(sc, res[0][1])

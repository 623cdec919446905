"""The similarity kernel with its first query k-blocks in the MMA warpgroup's registers (wgmma with a register A operand,
csrc/simtopk_tc.cu) against the same index searched with the whole query block in shared memory.  The register operand
carries the same values into the same MMAs in the same order, so every search is held to the fp64 oracle and the two
placements must return bit-identical ids, float32 scores and fp64 scores.  The shapes are where the placements differ:
partial query blocks (zero rows of the fragment), a dim that leaves no query tile in shared memory and the dims around
it, a ring capped to two and three stages so that it wraps inside the unrolled register k-blocks, and the launches the
register path must leave alone (64-row tiles)."""

from __future__ import annotations

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index
from oracle import cosine_topk as O
from tests.gpu_exact import check_exact, dev_search
from tests.test_gpu_tc_wide_tile import _data
from tests.test_tc_qregs_rule import QREGS, pick_qregs
from tests.test_tc_tile_rule import NARROW, WIDE, auto_tile

pytestmark = pytest.mark.gpu
KSLACK = 8
KERNELS = (N.KERNEL_TC1, N.KERNEL_TC2)


def _opt(ix, key, value):
    N.check(ix._lib.aur_set_option(ix._h, key, value))


def _both_placements(ix, Q, C, k, kernels=KERNELS, caps=(0,), oracle_kw=None, want_tile=WIDE):
    """Searches with the query k-blocks in registers (auto) and all in shared memory (tc_qregs 0), under each kernel and
    ring cap: every result is held to the oracle, and all of them to the first, bit for bit."""
    want = O.cosine_topk(Q, C, k, return_f64=True, **(oracle_kw or {}))
    runs = []
    for kern in kernels:
        ix.set_kernel(kern)
        for cap in caps:
            _opt(ix, b"tc_stages", cap)
            for qregs in (-1, 0):
                _opt(ix, b"tc_qregs", qregs)
                got = dev_search(ix, Q, k)
                st = ix.stats()
                assert st["last_kernel"] == kern and st["last_tile_n"] == want_tile
                check_exact(got, Q, C, k, want=want)
                runs.append(got)
    _opt(ix, b"tc_stages", 0)
    _opt(ix, b"tc_qregs", -1)
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert np.array_equal(a, b), "register and shared-memory query operands (or TC1 and TC2) differ"
    return want


@pytest.mark.parametrize("nq", [1, 63, 64, 65, 128, 129, 256, 300, 512])
def test_query_counts(nq):
    d, k, n = 768, 32, 30_000
    assert pick_qregs(d, auto_tile(d, k + KSLACK)) == QREGS
    C, Q = _data(n, d, nq, seed=100 + nq)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_placements(ix, Q, C, k)


@pytest.mark.parametrize("kbs", [QREGS - 1, QREGS, QREGS + 1])
def test_dims_around_the_register_depth(kbs):
    """dim = 64 * QREGS leaves no query tile in shared memory; one k-block less and the launch keeps them all there."""
    d, nq, k, n = 64 * kbs, 130, 32, 128 * 300 + 5
    assert pick_qregs(d, auto_tile(d, k + KSLACK)) == (QREGS if kbs >= QREGS else 0)
    C, Q = _data(n, d, nq, seed=kbs)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_placements(ix, Q, C, k)
        want = N.AUR_OK if kbs >= QREGS else N.AUR_ERR_INVALID   # forcing the depth needs that many k-blocks
        assert ix._lib.aur_set_option(ix._h, b"tc_qregs", QREGS) == want
        assert ix._lib.aur_set_option(ix._h, b"tc_qregs", QREGS + 1) == N.AUR_ERR_INVALID
        assert ix._lib.aur_set_option(ix._h, b"tc_stages", 1) == N.AUR_ERR_INVALID
        assert ix._lib.aur_set_option(ix._h, b"tc_stages", 13) == N.AUR_ERR_INVALID


@pytest.mark.parametrize("cap", [2, 3])
def test_ring_wraps_inside_the_register_kblocks(cap):
    """With two or three stages the ring's stage index and phase wrap inside the unrolled k-blocks of every tile."""
    d, nq, k, n = 768, 200, 32, 128 * 500 + 77
    C, Q = _data(n, d, nq, seed=cap, last_row_queries=3)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        want = _both_placements(ix, Q, C, k, caps=(cap, 0))
    assert (want[0][:3, 0] == n - 1).all()


@pytest.mark.parametrize("n", [37, 127, 128 * 40 + 1, 128 * 40 + 127])
def test_short_corpus_and_partial_last_tile(n):
    """Fewer rows than one tile, and a partial last tile whose last row is the best row of queries 0..3."""
    d, nq, k = 768, 65, 32
    C, Q = _data(n, d, nq, seed=n, last_row_queries=4)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        want = _both_placements(ix, Q, C, k)
    assert (want[0][:4, 0] == n - 1).all()


def test_tombstones_subset_and_uniform_scope():
    d, nq, k, n = 768, 200, 16, 128 * 150 + 77
    C, Q = _data(n, d, nq, seed=21)
    rng = np.random.default_rng(22)
    ru = rng.integers(0, 4, n).astype(np.int32)
    ro = rng.integers(-1, 3, n).astype(np.int32)
    live = np.ones(n, dtype=bool)
    qu, qo = np.full(nq, 2, np.int32), np.full(nq, 1, np.int32)   # one tenant scope for the whole batch
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), ru, ro)
        gone = np.concatenate([rng.choice(n, 300, replace=False), [n - 1]]).astype(np.int64)
        ix.remove(gone)
        live[gone] = False
        _both_placements(ix, Q, C, k, oracle_kw=dict(live=live))
        allow = np.sort(rng.choice(n, n // 3, replace=False)).astype(np.int64)
        sub = np.zeros(n, dtype=bool)
        sub[allow] = True
        for search, oracle_kw in ((lambda: ix.search(Q, k, qu, qo), dict(live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo)),
                                  (lambda: ix.search_subset(Q, k, allow), dict(live=live & sub))):
            want = O.cosine_topk(Q, C, k, **oracle_kw)
            res = []
            for kern in KERNELS:
                ix.set_kernel(kern)
                for qregs in (-1, 0):
                    _opt(ix, b"tc_qregs", qregs)
                    ids, sc = search()
                    assert ix.stats()["last_kernel"] == kern and ix.stats()["last_tile_n"] == WIDE
                    assert np.array_equal(ids, want[0]), f"{int((ids != want[0]).sum())} id mismatches"
                    res.append((ids, sc))
            for ids, sc in res[1:]:
                assert np.array_equal(ids, res[0][0]) and np.array_equal(sc, res[0][1])


@pytest.mark.parametrize("d,k", [(1024, 32), (768, 34)])
def test_narrow_launches_are_left_alone(d, k):
    """dim 1024 and top-34 at dim 768 stay on 64-row tiles whatever tc_qregs says, with unchanged answers."""
    nq, n = 130, 20_000
    assert auto_tile(d, k + KSLACK) == NARROW
    C, Q = _data(n, d, nq, seed=d + k)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        _both_placements(ix, Q, C, k, want_tile=NARROW)
        _opt(ix, b"tc_qregs", QREGS)   # a forced depth applies to 128-row launches only
        ix.set_kernel(N.KERNEL_TC2)
        got = dev_search(ix, Q, k)
        assert ix.stats()["last_tile_n"] == NARROW
        check_exact(got, Q, C, k)

"""oracle.cosine_topk(return_f64=True): the fp64 scores the float32 ones are rounded from, and nothing else changes.
The GPU tests hold the engine's fp64 re-rank (aur_search_dev's scores64) to these."""

import numpy as np
import pytest

from oracle import cosine_topk as O


@pytest.mark.parametrize("case", ["plain", "filtered", "padded", "ties", "empty"])
def test_return_f64_changes_nothing_else(case):
    rng = np.random.default_rng(11)
    n, d, nq, k = 700, 48, 6, 9
    C = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    Q = O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))
    kw = {}
    if case == "filtered":
        kw = dict(live=rng.random(n) > 0.2, row_user=rng.integers(0, 4, n), row_org=rng.integers(-1, 3, n),
                  q_user=rng.integers(0, 4, nq), q_org=rng.integers(-1, 3, nq))
    elif case == "padded":
        live = np.zeros(n, dtype=bool)
        live[[3, 500, 699]] = True                              # 3 visible rows, k = 9
        kw = dict(live=live)
    elif case == "ties":
        C[100:160] = O.round_to_bf16(Q[0] * 0.5)
        kw = dict(ids=rng.permutation(10 * n)[:n].astype(np.int64))
    elif case == "empty":
        C = C[:0]
    ids, sc = O.cosine_topk(Q, C, k, **kw)
    ids2, sc2, s64 = O.cosine_topk(Q, C, k, return_f64=True, **kw)
    np.testing.assert_array_equal(ids2, ids)
    np.testing.assert_array_equal(sc2, sc)
    assert s64.dtype == np.float64 and s64.shape == (nq, k)
    np.testing.assert_array_equal(s64.astype(np.float32), sc)
    np.testing.assert_array_equal(np.isfinite(s64), ids >= 0)
    assert (s64[ids < 0] == -np.inf).all()
    if case == "padded":
        assert (ids[:, :3] >= 0).all() and (ids[:, 3:] == -1).all()


def test_f64_scores_are_the_exact_cosines_of_the_returned_rows():
    rng = np.random.default_rng(5)
    n, d, nq, k = 2000, 100, 4, 12
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    ids, _, s64 = O.cosine_topk(Q, C, k, return_f64=True)
    for i in range(nq):
        np.testing.assert_array_equal(s64[i], O.exact_cosine(Q[i], C[ids[i]]))
        assert np.all(np.diff(s64[i]) <= 0)

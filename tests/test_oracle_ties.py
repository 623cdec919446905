"""oracle.cosine_topk is exact at ties: a group of bit-identical rows larger than the k + slack candidates the fp64
selection keeps must still come out in id order, as a full position-independent ranking of every row gives it."""

import numpy as np
import pytest

from oracle import cosine_topk as O


def _full_ranking(Q, C, k, ids, live=None):
    out = []
    for q in Q:
        ex = O.exact_cosine(q, C)
        if live is not None:
            ex = np.where(live, ex, -np.inf)
        out.append(ids[np.lexsort((ids, -ex))[:k]])
    return np.stack(out)


@pytest.mark.parametrize("group,k", [(60, 10), (27, 10), (26, 10), (200, 64)])
def test_tie_group_larger_than_the_candidates_comes_out_by_id(group, k):
    n, d = 3000, 128
    rng = np.random.default_rng(0)
    C = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    Q = O.round_to_bf16(rng.standard_normal((2, d)).astype(np.float32))
    C[500:500 + group] = O.round_to_bf16(Q[0] * 0.5)          # bit-identical rows, every query's best matches
    ids = rng.permutation(10 * n)[:n].astype(np.int64)         # ids not in row order
    got, _ = O.cosine_topk(Q, C, k, ids=ids)
    np.testing.assert_array_equal(got, _full_ranking(Q, C, k, ids))


def test_tie_group_cut_with_tombstones_and_small_chunks():
    n, d, k = 2000, 64, 5
    rng = np.random.default_rng(3)
    C = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    Q = O.round_to_bf16(rng.standard_normal((1, d)).astype(np.float32))
    C[::50] = O.round_to_bf16(Q[0] * 2.0)                       # 40 tied rows spread over every chunk
    ids = rng.permutation(n).astype(np.int64)
    live = np.ones(n, dtype=bool)
    live[np.argsort(ids)[:3]] = False                           # the three lowest ids are deleted
    got, _ = O.cosine_topk(Q, C, k, ids=ids, live=live, chunk=256)
    np.testing.assert_array_equal(got, _full_ranking(Q, C, k, ids, live))

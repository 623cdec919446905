"""Hybrid fusion without a GPU: bm25.relative_score_fusion on hand-computed cases, the query facade's fusion_type over
the CPU doubles (OracleIndex + BM25Index, fused on the host), and aur_hybrid_search's argument checks that run before any
device is touched."""

import ctypes as C

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200 import retriever as R
from aurora_b200.filters import HybridFusion
from tests.doubles import HashEmbedder, OracleIndex


# ----------------------------------------------------------------------------- relative_score_fusion
def test_relative_score_hand_computed_overlap():
    dense = [(1, 0.9), (2, 0.5), (3, 0.1)]                 # lo 0.1, hi 0.9
    sparse = [(3, 8.0), (4, 4.0), (1, 2.0)]                # lo 2.0, hi 8.0
    got = bm25.relative_score_fusion([(0.5, dense), (0.5, sparse)], 10)
    want = {
        1: 0.0 + 0.5 * ((0.9 - 0.1) / (0.9 - 0.1)) + 0.5 * ((2.0 - 2.0) / (8.0 - 2.0)),
        2: 0.0 + 0.5 * ((0.5 - 0.1) / (0.9 - 0.1)),
        3: 0.0 + 0.5 * ((0.1 - 0.1) / (0.9 - 0.1)) + 0.5 * ((8.0 - 2.0) / (8.0 - 2.0)),
        4: 0.0 + 0.5 * ((4.0 - 2.0) / (8.0 - 2.0)),
    }
    assert got == sorted(want.items(), key=lambda kv: (-kv[1], kv[0]))
    assert [d for d, _ in got] == [1, 3, 2, 4]            # 1 and 3 tie at 0.5: the lower id first
    assert got[0][1] == got[1][1] == 0.5


def test_relative_score_disjoint_legs_and_limit():
    got = bm25.relative_score_fusion([(0.3, [(10, 1.0), (11, 0.0)]), (0.7, [(20, 5.0), (21, 3.0)])], 3)
    assert got == [(20, 0.7), (10, 0.3), (11, 0.0)]


def test_relative_score_equal_scores_give_the_weight():
    """hi == lo (one entry, or a list of equal scores): every entry of the leg contributes its weight."""
    assert bm25.relative_score_fusion([(0.25, [(5, 0.4)])], 5) == [(5, 0.25)]
    got = bm25.relative_score_fusion([(0.6, [(7, 2.0), (3, 2.0), (9, 2.0)]), (0.4, [(9, 1.0), (1, 0.5)])], 10)
    assert got == [(9, 0.6 + 0.4), (3, 0.6), (7, 0.6), (1, 0.0)]


def test_relative_score_empty_leg_and_zero_weight():
    assert bm25.relative_score_fusion([(0.5, []), (0.5, [(1, 3.0), (2, 1.0)])], 5) == [(1, 0.5), (2, 0.0)]
    # weight 0 (alpha = 0): the leg's documents do not appear at all, as in ranked_fusion
    assert bm25.relative_score_fusion([(0.0, [(8, 0.9)]), (1.0, [(1, 3.0), (2, 1.0)])], 5) == [(1, 1.0), (2, 0.0)]
    assert bm25.ranked_fusion([(0.0, [8]), (1.0, [1, 2])], 5) == [(1, 1.0 / 60.0), (2, 1.0 / 61.0)]
    assert bm25.relative_score_fusion([(-1.0, [(8, 0.9)]), (0.0, [(1, 3.0)])], 5) == []


# ----------------------------------------------------------------------------- the facade over the CPU doubles
def _kb():
    emb = HashEmbedder(64)
    kb = R.KnowledgeBase(emb, capacity=1024, index_factory=lambda d, c: OracleIndex(d, c))
    texts = ["disk full on node-7 after log rotation", "cpu spike on api pods oom killer", "database latency timeout",
             "disk pressure evictions node-7", "timeout to the payment gateway", "oom kill loop memory limit"]
    for rep in range(12):
        for j, t in enumerate(texts):
            kb.insert(f"u{j % 3}", f"doc{j}", "f.md", [{"content": f"{t} #{rep % 5}", "chunk_index": rep}])
    return kb, emb


def _legs(kb, emb, q):
    ids, scores = kb.index.search(emb.encode([q]), 128)
    dense = [(int(d), float(s)) for d, s in zip(ids[0], scores[0]) if d >= 0]
    return dense, kb.sparse.search(q, 128)


@pytest.mark.parametrize("alpha", [0.0, 0.3, 0.5, 0.999])
def test_facade_relative_score_equals_manual_fusion(alpha):
    kb, emb = _kb()
    hybrid = R._QueryFacade(kb).hybrid
    for q in ("disk node-7", "oom memory", "timeout", "no such words"):
        dense, sparse = _legs(kb, emb, q)
        want = bm25.relative_score_fusion([(alpha, dense), (1.0 - alpha, sparse)], 10)
        got = hybrid(q, limit=10, alpha=alpha, fusion_type=HybridFusion.RELATIVE_SCORE).objects
        cos = dict(dense) if alpha > 0 else {}
        assert [(o.uuid, o.metadata.score) for o in got] == [(kb._id2key[d], s) for d, s in want]
        assert [o.metadata.distance for o in got] == [None if d not in cos else 1.0 - cos[d] for d, _ in want]


def test_facade_ranked_and_none_are_unchanged():
    kb, emb = _kb()
    hybrid = R._QueryFacade(kb).hybrid
    for q in ("disk node-7", "timeout"):
        dense, sparse = _legs(kb, emb, q)
        want = bm25.ranked_fusion([(0.5, [d for d, _ in dense]), (0.5, [d for d, _ in sparse])], 7)
        for ft in (None, HybridFusion.RANKED):
            got = hybrid(q, limit=7, alpha=0.5, fusion_type=ft).objects
            assert [(o.uuid, o.metadata.score) for o in got] == [(kb._id2key[d], s) for d, s in want]
        assert [o.uuid for o in kb.query(q, 7, alpha=0.5)] == [kb._id2key[d] for d, _ in want]


def test_unknown_fusion_still_raises():
    kb, _ = _kb()
    with pytest.raises(NotImplementedError):
        R._QueryFacade(kb).hybrid("disk", fusion_type="FUSION_TYPE_SOMETHING_ELSE")
    with pytest.raises(NotImplementedError):
        kb.query("disk", 5, alpha=0.5, fusion="FUSION_TYPE_SOMETHING_ELSE")


# ----------------------------------------------------------------------------- C ABI, no device needed
@pytest.fixture(scope="module")
def lib():
    from aurora_b200.build import build_native

    build_native()
    return N.load()


def test_hybrid_search_null_handles_are_invalid_without_a_device(lib):
    q = np.zeros((1, 64), np.uint16)
    off = np.array([0, 0], np.int64)
    w = np.array([0.5], np.float64)
    s, i, c = np.empty(2, np.float64), np.empty(2, np.int64), np.empty(2, np.float32)
    snaps = (C.c_int64 * 2)()
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    for ix, kw in ((None, None), (None, C.c_void_p(1)), (C.c_void_p(1), None)):
        rc = lib.aur_hybrid_search(ix, kw, p(q), 1, 1, None, p(off), None, None, p(w), p(w), N.FUSION_RANKED, 2,
                                   p(s), p(i), p(c), snaps)
        assert rc == N.AUR_ERR_INVALID
        assert b"null" in lib.aur_last_error()

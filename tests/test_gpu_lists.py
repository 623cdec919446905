"""aur_search_lists: every query searches only the rows its own id list names.  Each answer is held to the fp64 oracle
over exactly the allowed, live rows (ids bit-exact, padding exact, float32 scores within one rounding)."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index, MultiIndex, _ptr, lists_csr
from oracle import cosine_topk as O
from tests.gpu_exact import check_host_exact

pytestmark = pytest.mark.gpu


def _corpus(n, d, seed):
    rng = np.random.default_rng(seed)
    C_ = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    ext = rng.permutation(n).astype(np.int64) * 5 + 11          # ids unrelated to rows, every residue mod 3
    return rng, C_, ext


def _queries(rng, nq, d):
    return O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))


def _check_lists(got, Q, C_, ext, live, lists, q_list, k):
    ids, sc = got
    q_list = np.asarray(q_list)
    for l in np.unique(q_list):
        qs = np.nonzero(q_list == l)[0]
        allow = np.isin(ext, np.asarray(lists[l], dtype=np.int64)) & live
        check_host_exact((ids[qs], sc[qs]), Q[qs], C_, k, ids=ext, live=allow)


def _index(C_, ext, d, extra=0):
    ix = Index(d, C_.shape[0] + extra + 64)
    ix.add(C_, ext)
    return ix


@pytest.fixture(scope="module")
def big():
    n, d = 210_000, 64
    rng, C_, ext = _corpus(n, d, 7)
    ix = _index(C_, ext, d)
    yield rng, C_, ext, ix
    ix.close()


SIZES = [0, 1, None, None, None, 2047, 2048, 2049, 40_000, 150_000]   # None: k - 1, k, k + 8


@pytest.mark.parametrize("k", [1, 10, 32, 100, 128])
def test_list_sizes_and_k(big, k):
    rng, C_, ext, ix = big
    sizes = [s for s in SIZES if s is not None] + [max(k - 1, 0), k, k + 8]
    lists = [rng.choice(ext, size=s, replace=False) for s in sizes]
    q_list = np.repeat(np.arange(len(lists), dtype=np.int32), 3)
    rng.shuffle(q_list)
    Q = _queries(rng, len(q_list), C_.shape[1])
    got = ix.search_lists(Q, k, lists, q_list)
    _check_lists(got, Q, C_, ext, np.ones(len(ext), bool), lists, q_list, k)
    assert ix.stats()["last_kernel"] == N.KERNEL_LIST == 4


def test_a_200k_list_beside_one_row_lists(big):
    rng, C_, ext, ix = big
    lists = [rng.choice(ext, size=200_000, replace=False)] + [ext[i:i + 1] for i in range(0, 70, 7)]
    q_list = np.array([0, 1, 2, 0, 3, 4, 5, 6, 7, 8, 9, 10, 0], dtype=np.int32)
    Q = _queries(rng, len(q_list), C_.shape[1])
    got = ix.search_lists(Q, 20, lists, q_list)
    _check_lists(got, Q, C_, ext, np.ones(len(ext), bool), lists, q_list, 20)


@pytest.mark.parametrize("d", [8, 200, 384, 768, 1024, 1536])
def test_dims(d):
    rng, C_, ext = _corpus(6000, d, 100 + d)
    with _index(C_, ext, d) as ix:
        lists = [rng.choice(ext, size=s, replace=False) for s in (1, 130, 2100, 5000)]
        q_list = np.array([0, 1, 2, 3, 3, 2, 1], dtype=np.int32)
        Q = _queries(rng, len(q_list), d)
        for k in (1, 16, 128):
            _check_lists(ix.search_lists(Q, k, lists, q_list), Q, C_, ext, np.ones(len(ext), bool), lists, q_list, k)


def test_unknown_duplicate_tombstoned_and_upserted_ids():
    d = 128
    rng, C_, ext = _corpus(9000, d, 3)
    with _index(C_, ext, d, extra=100) as ix:
        dead = ext[100:600]
        assert ix.remove(dead) == len(dead)
        new_rows = O.round_to_bf16(rng.standard_normal((50, d)).astype(np.float32))
        up = ext[1000:1050]                                       # upsert: the id moves to a new row
        ix.add(new_rows, up)
        C2 = np.concatenate([C_, new_rows])
        ext2 = np.concatenate([ext, up])
        live = np.ones(len(ext2), bool)
        live[np.isin(ext2, dead)] = False
        live[1000:1050] = False                                   # the upserted ids' old rows
        base = ext[:3000]
        lst = np.concatenate([base, base[:500], [-5, 10**12, 7]])  # duplicates and unknown ids
        rng.shuffle(lst)
        lists = [lst, np.concatenate([up, up]), dead]
        q_list = np.array([0, 1, 2, 0, 1], dtype=np.int32)
        Q = _queries(rng, len(q_list), d)
        Q[1] = new_rows[7]                                        # the upserted vector must be found under its id
        ids, sc = ix.search_lists(Q, 10, lists, q_list)
        _check_lists((ids, sc), Q, C2, ext2, live, lists, q_list, 10)
        assert ids[1, 0] == up[7]
        assert (ids[2] == -1).all() and (sc[2] == -np.inf).all()  # a list of tombstones is padding


def test_ties_cross_segment_and_query_group_edges():
    d, n = 96, 6000
    rng, C_, ext = _corpus(n, d, 5)
    C_[1500:2600] = C_[1500]                                      # 1100 identical rows under different ids
    with _index(C_, ext, d) as ix:
        lst = ext[np.argsort(ext)]                                # every row; listed rows sorted by row, not id
        lists = [lst, ext[1500:2600]]
        q_list = np.array([0] * 70 + [1] * 66, dtype=np.int32)    # more queries per list than one group of 64
        Q = _queries(rng, len(q_list), d)
        Q[::3] = C_[1500]
        for k in (10, 128):
            ids, sc = ix.search_lists(Q, k, lists, q_list)
            _check_lists((ids, sc), Q, C_, ext, np.ones(n, bool), lists, q_list, k)
            tied = np.sort(ext[1500:2600])[:k]
            assert np.array_equal(ids[0], tied) and np.array_equal(ids[69], tied)


def test_concurrent_writer_and_readers():
    d, n0, step, steps = 64, 4000, 500, 12
    rng, C_, ext = _corpus(n0 + step * steps, d, 9)
    with Index(d, len(ext) + 64) as ix:
        ix.add(C_[:n0], ext[:n0])
        lists = [rng.choice(ext, size=s, replace=False) for s in (50, 1500, 6000)]
        q_list = np.array([0, 1, 2, 2], dtype=np.int32)
        Q = _queries(rng, len(q_list), d)
        results, errors = [], []

        def writer():
            for i in range(steps):
                a = n0 + i * step
                ix.add(C_[a:a + step], ext[a:a + step])

        def reader():
            try:
                for _ in range(10):
                    results.append(ix.search_lists_snapshot(Q, 16, lists, q_list))
            except Exception as e:          # noqa: BLE001 - surfaced below
                errors.append(e)

        ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errors, errors
        assert len({snap for _, _, snap in results}) >= 1
        for ids, sc, snap in results:
            assert n0 <= snap <= len(ext)
            _check_lists((ids, sc), Q, C_[:snap], ext[:snap], np.ones(snap, bool), lists, q_list, 16)


@pytest.mark.parametrize("size", [300, 5000, 60_000])
def test_one_shared_list_equals_search_subset(big, size):
    rng, C_, ext, ix = big
    lst = rng.choice(ext, size=size, replace=False)
    Q = _queries(rng, 40, C_.shape[1])
    for k in (10, 100):
        a_ids, a_sc = ix.search_lists(Q, k, [lst], np.zeros(len(Q), np.int32))
        b_ids, b_sc = ix.search_subset(Q, k, lst)
        assert np.array_equal(a_ids, b_ids) and np.array_equal(a_sc, b_sc)


def _raw(ix, Q, k, flat, offsets, n_lists, q_list):
    q = ix._rows_buffer(Q)
    nq = q.shape[0]
    scores = np.full((nq, max(k, 1)), 7.0, np.float32)
    ids = np.full((nq, max(k, 1)), 77, np.int64)
    snap = C.c_int64(-9)
    rc = ix._lib.aur_search_lists(ix._h, _ptr(q), nq, int(k), _ptr(flat), _ptr(offsets), int(n_lists), _ptr(q_list),
                                  _ptr(scores), _ptr(ids), C.byref(snap))
    return rc, scores, ids, snap.value


def test_rejections_leave_outputs_untouched():
    d = 64
    rng, C_, ext = _corpus(500, d, 2)
    Q = _queries(rng, 3, d)
    flat, off = lists_csr([ext[:10], ext[10:30]])
    ql = np.array([0, 1, 0], np.int32)

    def untouched(r):
        rc, s, i, snap = r
        assert (s == 7.0).all() and (i == 77).all() and snap == -9
        return rc

    with Index(d, 1000, dtype="f32") as f32:
        f32.add(C_, ext)
        assert untouched(_raw(f32, Q, 5, flat, off, 2, ql)) == N.AUR_ERR_UNSUPPORTED
    with _index(C_, ext, d) as ix:
        assert untouched(_raw(ix, Q, 5, flat, np.array([0, 30, 10], np.int64), 2, ql)) == N.AUR_ERR_INVALID
        assert untouched(_raw(ix, Q, 5, flat, np.array([1, 10, 30], np.int64), 2, ql)) == N.AUR_ERR_INVALID
        assert untouched(_raw(ix, Q, 5, flat, off, 2, np.array([0, 2, 0], np.int32))) == N.AUR_ERR_INVALID
        assert untouched(_raw(ix, Q, 5, flat, off, 2, np.array([0, -1, 0], np.int32))) == N.AUR_ERR_INVALID
        assert untouched(_raw(ix, Q, 129, flat, off, 2, ql)) == N.AUR_ERR_UNSUPPORTED
        assert untouched(_raw(ix, Q, 0, flat, off, 2, ql)) == N.AUR_ERR_INVALID
        assert ix._lib.aur_set_option(ix._h, b"kernel", N.KERNEL_LIST) == N.AUR_ERR_INVALID
        rc, s, i, snap = _raw(ix, Q, 5, flat, off, 2, ql)
        assert rc == N.AUR_OK and snap == 500 and ix.stats()["last_kernel"] == N.KERNEL_LIST


def test_multi_index_three_shards():
    d = 128
    rng, C_, ext = _corpus(12_000, d, 4)
    with MultiIndex(d, 20_000, devices=[0, 0, 0]) as mi:
        mi.add(C_, ext)
        lists = [rng.choice(ext, size=s, replace=False) for s in (0, 5, 900, 7000)]
        q_list = np.array([3, 2, 1, 0, 3, 2], dtype=np.int32)
        Q = _queries(rng, len(q_list), d)
        got = mi.search_lists(Q, 32, lists, q_list)
        _check_lists(got, Q, C_, ext, np.ones(len(ext), bool), lists, q_list, 32)


def _shape(objs):
    return [(o.uuid, round(o.metadata.score, 5)) for o in objs]


def test_retriever_filtered_query_and_many_scope_batch(monkeypatch):
    from aurora_b200 import retriever as R
    from aurora_b200.filters import Filter
    from tests.doubles import HashEmbedder, OracleIndex

    monkeypatch.setattr(R, "_LIST_MAX_FRACTION", 1.0)            # every filter below through the list kernel

    emb = HashEmbedder(64)
    dev = R.KnowledgeBase(emb, capacity=8192)
    host = R.KnowledgeBase(emb, capacity=8192, index_factory=lambda d, c: OracleIndex(d, c))
    words = ["disk", "oom", "pod", "latency", "timeout", "node", "memory", "cpu", "network", "failover", "kafka", "dns"]
    rng = np.random.default_rng(1)
    for kb in (dev, host):
        r = np.random.default_rng(1)
        for t in range(48):
            for doc in range(3):
                chunks = [{"chunk_index": c, "content": " ".join(r.choice(words, size=6))} for c in range(8)]
                docid = f"discovery:{t}:{doc}" if doc == 0 else f"doc{t}-{doc}"
                kb.insert(f"u{t}", docid, "f.md", chunks, org_id=f"o{t % 20}")
    for q in ("disk node", "oom memory pod", "kafka dns latency"):
        for o in ("o3", "o7"):
            flt = Filter.by_property("org_id").equal(o)
            assert _shape(dev.query(q, 10, filters=flt)) == _shape(host.query(q, 10, filters=flt))
            flt2 = Filter.by_property("org_id").equal(o) & Filter.by_property("document_id").like("discovery:*")
            assert _shape(dev.query(q, 10, filters=flt2)) == _shape(host.query(q, 10, filters=flt2))
            assert dev.index.stats()["last_kernel"] == N.KERNEL_LIST
    reqs = [(f"u{t}", " ".join(rng.choice(words, size=3)), 8, None, None if t % 3 else f"o{(t + 5) % 20}")
            for t in range(40)]
    got = dev.query_batch(reqs)
    assert dev.index.stats()["last_kernel"] == N.KERNEL_LIST
    assert [_shape(x) for x in got] == [_shape(x) for x in host.query_batch(reqs)]
    dev.index.close()

"""The keyword store's term-major index (aur_kw_reindex, aur_kw_set_option "kw_path", aur_kw_get_index_stats): every
answer, however the indexed prefix and the tail are scored, is bit for bit the fp64 oracle's (oracle/bm25_topk.py) and
the forward scan's."""

import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import KeywordIndex, MultiKeywordIndex
from tests.keyword_mirror import Mirror, assert_matches_oracle, zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

AUTO, FORWARD, INDEX = N.KW_PATH_AUTO_OPT, N.KW_PATH_FORWARD_OPT, N.KW_PATH_INDEX_OPT
ROUND = 32           # rows per round of the scoring and selection kernels (csrc/keyword.cu)
MAX_TERM_POS = 64    # term positions a query group takes through the index (kIxMaxTermPos)


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def all_paths(st, m, qt, qo, k, *a, **kw):
    """The search forced forward, forced to the index and on the cost rule: each equal to the oracle (sampled queries),
    all three bit-identical on every query.  Returns the index path's (ids, scores, snapshot) and its last_path."""
    out = {}
    for path in (FORWARD, INDEX, AUTO):
        st.set_path(path)
        out[path] = assert_matches_oracle(st, m, qt, qo, k, *a, **kw)
        if path == INDEX:
            forced = st.index_stats()["last_path"]
    st.set_path(AUTO)
    ids0, sc0, snap0 = out[FORWARD]
    for path in (INDEX, AUTO):
        ids, sc, snap = out[path]
        assert snap == snap0 and np.array_equal(ids, ids0), path
        assert np.array_equal(sc.view(np.int64), sc0.view(np.int64)), path
    return out[INDEX], forced


def _add(st, m, rng, n, id0, **kw):
    t, f, off = zipf_docs(rng, n, **kw)
    ids = id0 + rng.permutation(n).astype(np.int64) * 3
    st.add(ids, t, f, off)
    m.add(ids, t, f, off)
    return ids


def _prefix_store(n_indexed, tail, seed, capacity=None, **kw):
    """n_indexed documents indexed, then `tail` more left to the forward scan (few enough not to trigger a rebuild)."""
    rng = np.random.default_rng(seed)
    st, m = KeywordIndex(capacity or 2 * (n_indexed + tail) + 8), Mirror()
    if n_indexed:
        _add(st, m, rng, n_indexed, 1, **kw)
        st.reindex()
    if tail:
        _add(st, m, rng, tail, 10 ** 7, **kw)
    return st, m, rng


@pytest.mark.parametrize("tail", [0, 1, 31, 32, 33, 1000])
def test_partial_prefix_and_round_edges_of_the_tail(tail):
    st, m, rng = _prefix_store(20_000, tail, seed=tail)
    ix = st.index_stats()
    assert ix["indexed_rows"] == 20_000 and ix["builds"] >= 1
    assert ix["index_postings"] == int(m.offsets[20_000]) and ix["index_bytes"] >= 8 * ix["index_postings"]
    qt, qo = zipf_queries(rng, 24)
    _, path = all_paths(st, m, qt, qo, 16)
    assert path == (N.KW_PATH_INDEX | N.KW_PATH_FORWARD if tail else N.KW_PATH_INDEX)
    st.set_path(FORWARD)
    st.search(qt, qo, 16)
    assert st.index_stats()["last_path"] == N.KW_PATH_FORWARD
    assert st.index_stats()["last_postings"] == m.offsets[-1]       # every posting of every row


def test_tail_across_block_edges():
    """Tails of 2 * SMs rounds -1 / +0 / +1 rows: the forward part's last block gets a short or a one-row range."""
    edge = 2 * _sms() * ROUND
    for tail in (edge - 1, edge, edge + 1):
        st, m, rng = _prefix_store(9 * edge + 64, tail, seed=tail, mean_len=10)
        assert st.index_stats()["indexed_rows"] == 9 * edge + 64
        qt, qo = zipf_queries(rng, 9)
        for k in (1, 128):
            all_paths(st, m, qt, qo, k)


def test_nothing_indexed_and_empty_stores():
    st, m = KeywordIndex(64), Mirror()
    ids, _, snap = st.search(np.array([1], np.int32), np.array([0, 1]), 4)
    assert snap == 0 and (ids == -1).all()
    st.reindex()                                                       # an empty index of nothing
    assert st.index_stats()["indexed_rows"] == 0
    ids0 = np.arange(5, dtype=np.int64)
    st.add(ids0, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(6, np.int64))   # zero-token documents only
    m.add(ids0, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(6, np.int64))
    st.set_path(INDEX)
    ids, _, snap = st.search(np.array([1], np.int32), np.array([0, 1]), 4)
    assert snap == 5 and (ids == -1).all()


def test_every_row_indexed_after_growth_from_a_tiny_posting_array():
    """Postings grow mid-run (the forward array moves); the index built after them reads every row right."""
    rng = np.random.default_rng(4)
    st, m = KeywordIndex(30_000, postings_capacity=16), Mirror()
    for c in range(6):
        _add(st, m, rng, 4000, 1 + c)
    s = st.stats()
    assert s["postings_allocated"] > 16
    st.reindex()
    builds = st.index_stats()["builds"]
    _add(st, m, rng, 100, 99)                                           # growth after the build
    assert st.stats()["postings_allocated"] >= st.stats()["postings_used"]
    qt, qo = zipf_queries(rng, 33)
    all_paths(st, m, qt, qo, 50)
    assert st.index_stats()["builds"] == builds


def test_tombstones_upserts_and_compaction_with_rebuild():
    rng = np.random.default_rng(5)
    st, m = KeywordIndex(60_000), Mirror()
    ids = _add(st, m, rng, 20_000, 1)
    st.reindex()
    qt, qo = zipf_queries(rng, 40)
    gone = rng.choice(ids, 3000, replace=False)
    assert st.remove(gone) == 3000
    m.remove(gone)
    again = rng.choice(np.setdiff1d(ids, gone), 500, replace=False)     # upserts of indexed rows: their new rows are tail
    t, f, off = zipf_docs(rng, len(again))
    st.add(again, t, f, off)
    m.add(again, t, f, off)
    all_paths(st, m, qt, qo, 64)
    builds = st.index_stats()["builds"]
    assert st.compact() == 3500
    m.compact()
    ix = st.index_stats()
    assert ix["builds"] == builds + 1 and ix["indexed_rows"] == len(m.ids) == st.stats()["docs"]
    _, path = all_paths(st, m, qt, qo, 64)
    assert path == N.KW_PATH_INDEX


def test_capacity_edge_zero_token_docs_and_huge_tf():
    st, m = KeywordIndex(5), Mirror()
    ids = np.array([10, 11, 12, 13, 14], np.int64)
    terms = np.array([0, 1, 0, 2, 0], np.int32)
    tfs = np.array([70_000, 3, 65_536, 1, 1], np.int32)
    off = np.array([0, 2, 2, 4, 4, 5], np.int64)                         # docs 11 and 13 have no tokens
    st.add(ids, terms, tfs, off)
    m.add(ids, terms, tfs, off)
    st.reindex()
    assert st.index_stats()["indexed_rows"] == 5 == st.stats()["capacity"]
    _, path = all_paths(st, m, np.array([0, 1, 2, 0, 2], np.int32), np.array([0, 1, 3, 5]), 5)
    assert path == N.KW_PATH_INDEX


def _uniform_store(n_docs, vocab, words, seed):
    rng = np.random.default_rng(seed)
    terms, tfs, off = [], [], [0]
    for _ in range(n_docs):
        u, c = np.unique(rng.integers(0, vocab, words), return_counts=True)
        terms.append(u.astype(np.int32))
        tfs.append(c.astype(np.int32))
        off.append(off[-1] + len(u))
    args = (np.arange(n_docs, dtype=np.int64) * 7 + 3, np.concatenate(terms), np.concatenate(tfs), np.asarray(off, np.int64))
    st, m = KeywordIndex(n_docs), Mirror()
    st.add(*args)
    m.add(*args)
    st.reindex()
    return st, m, rng, np.unique(args[1])


@pytest.mark.parametrize("n_terms", [1, 2, 17, MAX_TERM_POS, MAX_TERM_POS + 1])
def test_query_lengths_repeats_unknown_terms_and_the_position_cap(n_terms):
    """Repeats and unknown ids are dropped before term positions are counted; a query of more than the cap's live terms
    is scanned forward even when the index is forced."""
    st, m, rng, live = _uniform_store(3000, 6000, 60, seed=n_terms)
    q = rng.permutation(live)[:n_terms].astype(np.int32)
    q = np.concatenate([q, q[: n_terms // 2], np.array([9000, 2 ** 27], np.int32)])
    short = np.array([q[0], 9001, q[0]], np.int32)
    qt = np.concatenate([q, short])
    qo = np.array([0, len(q), len(qt)])
    _, path = all_paths(st, m, qt, qo, 40)
    assert path == (N.KW_PATH_FORWARD if n_terms > MAX_TERM_POS else N.KW_PATH_INDEX)
    assert st.stats()["last_terms"] == n_terms


@pytest.mark.parametrize("k", [1, 128])
@pytest.mark.parametrize("where", ["index", "across"])
def test_tie_groups_cut_inside_the_index_and_across_the_tail(k, where):
    """5 000 bit-equal documents among 20 000 others, ids shuffled: all indexed, or half indexed and half in the tail."""
    rng = np.random.default_rng(k + len(where))
    n_tie, n_other = 5000, 20_000
    t, f, off = zipf_docs(rng, n_other, vocab=3000)
    st, m = KeywordIndex(2 * (n_tie + n_other)), Mirror()
    other_ids = rng.permutation(n_other).astype(np.int64) * 2 + 1
    tie_ids = rng.permutation(n_tie).astype(np.int64) * 2
    first = n_tie if where == "index" else n_tie // 2

    def ties(ids):
        n = len(ids)
        return ids, np.tile(np.array([7, 3001], np.int32), n), np.tile(np.array([2, 1], np.int32), n), 2 * np.arange(n + 1)

    for a in ((other_ids, t, f, off), ties(tie_ids[:first])):
        st.add(*a)
        m.add(*a)
    st.reindex()
    if first < n_tie:
        a = ties(tie_ids[first:])                                        # 2 500 postings x 2: under the rebuild fraction
        st.add(*a)
        m.add(*a)
        assert st.index_stats()["indexed_rows"] == n_other + first
    for q in (np.array([3001], np.int32), np.array([7, 3001], np.int32)):
        (ids, sc, _), _ = all_paths(st, m, q, np.array([0, len(q)]), k)
        if len(q) == 1:
            assert (sc[0] == sc[0][0]).all()


@pytest.mark.parametrize("nq", [1, 2, 255, 256, 257])
def test_query_blocks_and_k(nq):
    st, m, rng = _prefix_store(30_000, 2000, seed=nq)
    qt, qo = zipf_queries(rng, nq)
    sample = sorted({0, nq // 2, nq - 1, min(255, nq - 1)})
    for k in (1, 128):
        all_paths(st, m, qt, qo, k, sample=sample)


def test_tenant_scopes_and_allow_lists():
    n = 30_000
    rng = np.random.default_rng(9)
    t, f, off = zipf_docs(rng, n)
    ids = rng.permutation(n).astype(np.int64) * 3 + 1
    user = rng.integers(0, 40, n).astype(np.int32)
    org = np.where(rng.random(n) < 0.5, rng.integers(0, 8, n), -1).astype(np.int32)
    st, m = KeywordIndex(2 * n), Mirror()
    st.add(ids, t, f, off, user, org)
    m.add(ids, t, f, off, user, org)
    assert st.index_stats()["indexed_rows"] == n                        # the writer built it
    nq = 300
    qt, qo = zipf_queries(rng, nq)
    q_user = rng.integers(-2, 42, nq).astype(np.int32)                   # > 32 distinct scopes, unknown codes
    q_org = rng.integers(-1, 9, nq).astype(np.int32)
    all_paths(st, m, qt, qo, 20, q_user, q_org, sample=range(0, nq, 7))
    all_paths(st, m, qt, qo, 20, q_user, None, sample=range(3, nq, 11))
    allow = np.concatenate([rng.choice(ids, 3000, replace=False), [10 ** 12, 5]])
    all_paths(st, m, qt, qo[:7], 16, allow_ids=allow)
    all_paths(st, m, qt, qo[:7], 16, q_user[:6], q_org[:6], allow_ids=allow)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_filtered_hybrid_through_the_index(n):
    """aur_hybrid_search_filtered with every store forced to the index equals the separate calls' host fusion (and the
    oracles on a sampled query) and the forced-forward answer bit for bit."""
    from aurora_b200.engine import hybrid_search
    from tests.test_gpu_hybrid import FUSIONS, weights
    from tests.test_gpu_hybrid_filtered import _filled, _programs, _queries

    pr = _filled(n, 6000, seed=40 + n)
    pr.kw.reindex()
    nq = 64
    qv, qt, qo, rng = _queries(nq, seed=n)
    progs, allows, q_prog = _programs(pr, 33, nq, rng, False)
    wd, ws = weights(nq, shift=n)
    for fusion in FUSIONS:
        pr.kw.set_path(INDEX)
        got = pr.check(qv, qt, qo, 16, 32, progs, allows, q_prog, fusion, wd, ws, ctx=(n, fusion), sample=3)
        again = hybrid_search(pr.ix, pr.kw, qv, 16, qt, qo, wd, ws, fusion, 32, programs=progs, q_program=q_prog)
        assert np.array_equal(again[0], got[0])
        stores = pr.kw.stores if n > 1 else [pr.kw]
        assert all(s.index_stats()["last_path"] & N.KW_PATH_INDEX for s in stores)
        pr.kw.set_path(FORWARD)
        fwd = hybrid_search(pr.ix, pr.kw, qv, 16, qt, qo, wd, ws, fusion, 32, programs=progs, q_program=q_prog)
        assert np.array_equal(got[0], fwd[0]) and np.array_equal(got[1].view(np.int64), fwd[1].view(np.int64))
    pr.close()


@pytest.mark.parametrize("n", [1, 2, 3])
def test_hybrid_multi_stores_indexed_to_different_prefixes(n):
    from aurora_b200.engine import MultiIndex, hybrid_search
    from tests.test_gpu_hybrid import FUSIONS, weights

    rng = np.random.default_rng(70 + n)
    dim, n_docs = 128, 9000
    mi, mk = MultiIndex(dim, 4 * n_docs, devices=[0] * n), MultiKeywordIndex(4 * n_docs, devices=[0] * n)
    ids = rng.permutation(n_docs).astype(np.int64)
    vec = rng.standard_normal((n_docs, dim)).astype(np.float32)
    t, f, off = zipf_docs(rng, n_docs)
    mi.add(vec, ids)
    mk.add(ids, t, f, off)
    mk.reindex()
    for s in range(n):   # store s gets 100 * s more documents, under its rebuild fraction: different tails
        extra = (10 ** 6 + np.arange(100 * s, dtype=np.int64)) * n + s
        if len(extra):
            et, ef, eo = zipf_docs(rng, len(extra))
            mi.add(rng.standard_normal((len(extra), dim)).astype(np.float32), extra)
            mk.add(extra, et, ef, eo)
    rows = [st["indexed_rows"] for st in mk.index_stats()]
    docs = [s["docs"] for s in mk.stats()["stores"]]
    assert rows == [d - 100 * s for s, d in enumerate(docs)]
    nq = 40
    qv = rng.standard_normal((nq, dim)).astype(np.float32)
    qt, qo = zipf_queries(rng, nq)
    wd, ws = weights(nq, shift=n)
    for fusion in FUSIONS:
        outs = []
        for path in (FORWARD, INDEX, AUTO):
            mk.set_path(path)
            outs.append(hybrid_search(mi, mk, qv, 20, qt, qo, wd, ws, fusion, 30))
        for o in outs[1:]:
            assert np.array_equal(o[0], outs[0][0]) and np.array_equal(o[1].view(np.int64), outs[0][1].view(np.int64))
            assert o[3] == outs[0][3]
    mk.set_path(AUTO)
    mi.close()
    mk.close()


def test_the_path_rule():
    """The cost rule picks the index for one query of rare words and the forward scan for 256 queries of common ones."""
    rng = np.random.default_rng(12)
    n = 200_000
    t, f, off = zipf_docs(rng, n, mean_len=40)
    st, m = KeywordIndex(n), Mirror()
    st.add(np.arange(n, dtype=np.int64), t, f, off)
    m.add(np.arange(n, dtype=np.int64), t, f, off)
    assert st.index_stats()["indexed_rows"] == n
    df = np.bincount(t)
    live = np.nonzero(df)[0]
    rare = np.sort(live[np.argsort(df[live], kind="stable")[:3]]).astype(np.int32)
    assert_matches_oracle(st, m, rare, np.array([0, 3]), 10)
    ix = st.index_stats()
    assert ix["last_path"] == N.KW_PATH_INDEX and ix["last_postings"] == int(df[rare].sum())
    common = np.argsort(-df)[:40].astype(np.int32)
    qs = [rng.choice(common, 4, replace=False) for _ in range(256)]
    qt, qo = np.concatenate(qs).astype(np.int32), np.arange(0, 4 * 257, 4, dtype=np.int64)
    assert_matches_oracle(st, m, qt, qo, 10, sample=range(0, 256, 51))
    assert st.index_stats()["last_path"] == N.KW_PATH_FORWARD


def test_rebuilds_under_concurrent_readers():
    """The writer's appends trigger rebuilds while three readers search with the index forced; every answer equals the
    oracle over the prefix it reports."""
    from oracle.bm25_topk import bm25_topk

    rng = np.random.default_rng(11)
    n = 60_000
    t, f, off = zipf_docs(rng, n)
    st, m = KeywordIndex(n), Mirror()
    st.set_path(INDEX)
    qt, qo = zipf_queries(rng, 24)
    chunks = np.array_split(np.arange(n), 30)
    answers, errors = [], []
    done = threading.Event()

    def writer():
        try:
            for c in chunks:
                sl = slice(off[c[0]], off[c[-1] + 1])
                st.add(c.astype(np.int64), t[sl], f[sl], off[c[0]:c[-1] + 2] - off[c[0]])
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader():
        while not done.is_set():
            answers.append(st.search(qt, qo, 16))

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors
    assert st.index_stats()["builds"] >= 5
    m.add(np.arange(n, dtype=np.int64), t, f, off)
    assert len({a[2] for a in answers}) >= 2
    for ids, scores, snap in answers[:: max(1, len(answers) // 12)]:
        wi, ws = bm25_topk(m.corpus(n_rows=snap), qt, qo, 16)
        assert np.array_equal(ids, wi) and np.array_equal(scores.view(np.int64), ws.view(np.int64)), snap


DOCS = [
    ("disk full on node-7 after log rotation failed", "u1", None),
    ("cpu spike on api pods; oom killer fired twice", "u1", "o1"),
    ("database latency timeout during failover", "u2", "o1"),
    ("disk pressure evictions, node-7 cordoned", "u2", None),
    ("timeout talking to the payment gateway", "u3", "o2"),
    ("oom kill loop in worker pods, memory limit 512Mi", "u1", None),
]


def _fill(kb, n_rep=40):
    for rep in range(n_rep):
        for j, (text, u, o) in enumerate(DOCS):
            kb.insert(u, f"doc{j}", "f.md", [{"content": f"{text} #{rep % 7}", "chunk_index": rep}], org_id=o)


def _shape(objs):
    return [(o.uuid, o.metadata.score, None if o.metadata.distance is None else round(o.metadata.distance, 5)) for o in objs]


@pytest.mark.parametrize("kind", ["index", "multi_index"])
def test_knowledge_base_through_the_index_matches_the_host_bm25(kind, monkeypatch):
    from aurora_b200 import retriever as R
    from aurora_b200.engine import MultiIndex
    from tests.doubles import HashEmbedder, OracleIndex

    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    emb = HashEmbedder(64)
    factory = (lambda d, c: MultiIndex(d, c, devices=[0, 0, 0])) if kind == "multi_index" else None
    dev = R.KnowledgeBase(emb, capacity=4096, **({"index_factory": factory} if factory else {}))
    host = R.KnowledgeBase(emb, capacity=4096, index_factory=lambda d, c: OracleIndex(d, c))
    assert isinstance(dev.sparse, bm25.DeviceBM25) and isinstance(host.sparse, bm25.BM25Index)
    for kb in (dev, host):
        _fill(kb)
        kb.delete_where(lambda p: p.get("document_id") == "doc3" and p.get("chunk_index", 0) % 5 == 0)
    dev.sparse.store.reindex()
    dev.sparse.store.set_path(INDEX)
    queries = ["disk node-7", "oom pods memory", "timeout", "nothing matches this", "latency failover disk"]

    def compare():
        for q in queries:
            for alpha in (0.0, 0.5):
                for scope in (("u1", None), ("u2", "o1")):
                    a = dev.query(q, 10, user_id=scope[0], org_id=scope[1], alpha=alpha, scoped=True)
                    b = host.query(q, 10, user_id=scope[0], org_id=scope[1], alpha=alpha, scoped=True)
                    assert _shape(a) == _shape(b), (q, alpha, scope)
                assert _shape(dev.query(q, 10, alpha=alpha)) == _shape(host.query(q, 10, alpha=alpha))
        reqs = [("u1", q, 6, a_, None) for q in queries for a_ in (0.0, 0.5)] + [("u2", q, 4, 0.3, "o1") for q in queries]
        assert [_shape(x) for x in dev.query_batch(reqs)] == [_shape(x) for x in host.query_batch(reqs)]

    compare()
    stats = dev.sparse.store.index_stats()
    for s in (stats if isinstance(stats, list) else [stats]):
        assert s["last_path"] & N.KW_PATH_INDEX
    for kb in (dev, host):                                               # a tail behind the index
        kb.insert("u1", "late", "f.md", [{"content": "late disk oom entry", "chunk_index": 0}])
    compare()

"""GPU keyword store (aur_kw_*, engine.KeywordIndex, bm25.DeviceBM25, the retriever's keyword leg).  Every answer is held
to the fp64 oracle (oracle/bm25_topk.py): ids bit-exact, fp64 scores bit-identical."""

import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import KeywordIndex
from tests.keyword_mirror import Mirror, assert_matches_oracle, zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

# the kernel's geometry (csrc/keyword.cu): 32-row rounds, up to 2 * SMs blocks, 256 queries per launch,
# 256-entry candidate buffers flushed above 224, folds of 2048 // k lists
ROUND, QBLOCK = 32, 256


def _store(n, seed=0, capacity=None, **kw):
    rng = np.random.default_rng(seed)
    t, f, off = zipf_docs(rng, n, **kw)
    ids = rng.permutation(n).astype(np.int64) * 3 + 1          # shuffled, sparse ids
    st = KeywordIndex(capacity or max(n, 1) * 2)
    m = Mirror()
    if n:
        st.add(ids, t, f, off)
        m.add(ids, t, f, off)
    return st, m, rng


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049])
@pytest.mark.parametrize("k", [1, 128])
def test_small_corpora_and_round_edges(n, k):
    st, m, rng = _store(n, seed=n)
    qt, qo = zipf_queries(rng, 17)
    assert_matches_oracle(st, m, qt, qo, k)


def test_grid_saturation_edges():
    """Corpora around 2 * SMs * 32 rows: the last block gets a full, a short and a one-row range."""
    edge = 2 * _sms() * ROUND
    for n in (edge - 1, edge, edge + 1, 3 * edge + 1):
        st, m, rng = _store(n, seed=n)
        qt, qo = zipf_queries(rng, 9)
        for k in (1, 7, 128):
            assert_matches_oracle(st, m, qt, qo, k)


def test_large_corpus_sampled_queries():
    st, m, rng = _store(200_000, seed=5, mean_len=30)
    qt, qo = zipf_queries(rng, 64)
    assert_matches_oracle(st, m, qt, qo, 128, sample=range(0, 64, 4))
    assert_matches_oracle(st, m, qt, qo, 10, sample=range(1, 64, 4))
    s = st.stats()
    assert s["last_launches"] >= 2 and s["last_ms"] > 0


@pytest.mark.parametrize("nq", [1, QBLOCK - 1, QBLOCK, QBLOCK + 1, 1025])
def test_query_blocks(nq):
    st, m, rng = _store(20_000, seed=nq)
    qt, qo = zipf_queries(rng, nq)
    assert_matches_oracle(st, m, qt, qo, 32, sample=sorted({0, nq // 2, nq - 1, min(QBLOCK, nq - 1)}))


def test_k_limits_and_more_k_than_matches():
    st, m, rng = _store(500, seed=1)
    qt = np.array([4999], np.int32)          # a rare word: fewer matching docs than k
    ids, _, _ = assert_matches_oracle(st, m, qt, np.array([0, 1]), 128)
    assert (ids[0] == -1).any()
    with pytest.raises(N.AuroraError) as e:
        st.search(qt, np.array([0, 1]), 129)
    assert e.value.code == N.AUR_ERR_UNSUPPORTED
    with pytest.raises(N.AuroraError) as e:
        st.search(qt, np.array([0, 1]), 0)
    assert e.value.code == N.AUR_ERR_INVALID


def _spill_threshold(nq):
    """Distinct live terms above which a launch of nq queries keeps its per-warp contribution table in global memory:
    the kernel's shared memory is nq (16 B threshold + 4 B count) + 8 warps x 256 x 16 B of sort area, rounded to 16,
    plus 8 warps x 8 B per distinct term, against the device's opt-in limit (csrc/keyword.cu, kw_score_kernel)."""
    import torch

    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    fixed = (nq * 16 + 8 * 256 * 16 + 4 * nq + 15) // 16 * 16
    return (optin - fixed) // 64


def _uniform_store(n_docs, vocab, words_per_doc, seed):
    """Documents of uniformly drawn words, so nearly every vocabulary id has live postings."""
    rng = np.random.default_rng(seed)
    terms, tfs, off = [], [], [0]
    for _ in range(n_docs):
        u, c = np.unique(rng.integers(0, vocab, words_per_doc), return_counts=True)
        terms.append(u.astype(np.int32))
        tfs.append(c.astype(np.int32))
        off.append(off[-1] + len(u))
    args = (np.arange(n_docs, dtype=np.int64) * 7 + 3, np.concatenate(terms), np.concatenate(tfs), np.asarray(off, np.int64))
    st, m = KeywordIndex(n_docs), Mirror()
    st.add(*args)
    m.add(*args)
    live_terms = np.unique(args[1])
    return st, m, rng, live_terms


@pytest.mark.parametrize("n_terms", [1, 10, 1000, "spill"])
def test_long_queries_duplicates_and_unknown_terms(n_terms):
    """A pasted alert body: a query of up to 1 000 live terms keeps its contribution table in shared memory; one with more
    live terms than shared memory holds spills the table to global memory and answers the same way."""
    st, m, rng, live = _uniform_store(6000, 12_000, 80, seed=7)
    spill = n_terms == "spill"
    want = _spill_threshold(1) + 400 if spill else n_terms
    assert len(live) >= want
    q = rng.permutation(live)[:want].astype(np.int32)
    q = np.concatenate([q, q[: want // 3], np.array([20_000, 20_001], np.int32)])   # repeats and unknown ids are ignored
    assert_matches_oracle(st, m, q, np.array([0, len(q)]), 64)
    s = st.stats()
    assert s["last_terms"] == want
    assert s["last_spilled"] == (1 if spill else 0)
    unknown = np.array([20_000, 20_001, 2 ** 27], np.int32)
    ids, scores, _ = st.search(unknown, np.array([0, 3]), 5)
    assert (ids == -1).all() and np.isneginf(scores).all()
    ids, scores, _ = st.search(np.zeros(0, np.int32), np.array([0, 0, 0]), 3)     # empty queries: padding only
    assert (ids == -1).all()


def test_query_block_whose_term_union_spills():
    """256 short queries whose distinct terms together exceed shared memory: the whole block spills, each answer exact."""
    st, m, rng, live = _uniform_store(6000, 12_000, 80, seed=8)
    nq = QBLOCK
    per = _spill_threshold(nq) // nq + 8
    qs = [rng.choice(live, per, replace=False).astype(np.int32) for _ in range(nq)]
    qt, qo = np.concatenate(qs), np.concatenate([[0], np.cumsum([len(x) for x in qs])]).astype(np.int64)
    assert len(np.unique(qt)) > _spill_threshold(nq)
    assert_matches_oracle(st, m, qt, qo, 16, sample=range(0, nq, 17))
    s = st.stats()
    assert s["last_spilled"] == 1 and s["last_terms"] == len(np.unique(qt))


def test_huge_tf_and_zero_token_docs():
    st = KeywordIndex(64)
    m = Mirror()
    ids = np.array([10, 11, 12, 13, 14], np.int64)
    terms = np.array([0, 1, 0, 2, 0], np.int32)
    tfs = np.array([70_000, 3, 65_536, 1, 1], np.int32)
    off = np.array([0, 2, 2, 4, 4, 5], np.int64)                 # docs 11 and 13 have no tokens (they count in N)
    st.add(ids, terms, tfs, off)
    m.add(ids, terms, tfs, off)
    assert st.stats()["live"] == 5 and st.stats()["total_len"] == 70_000 + 3 + 65_536 + 1 + 1
    assert_matches_oracle(st, m, np.array([0, 1, 2], np.int32), np.array([0, 1, 3]), 4)


@pytest.mark.parametrize("k", [1, 100, 128])
def test_tie_groups_cut_inside_and_across_blocks(k):
    """5 000 identical documents (equal tf and length: bit-equal scores) among others, ids shuffled: the cut keeps the
    lowest ids of the group, wherever the rows sit."""
    rng = np.random.default_rng(k)
    n_tie, n_other = 5000, 20_000
    t, f, off = zipf_docs(rng, n_other, vocab=3000)
    tie_t = np.tile(np.array([7, 3001], np.int32), n_tie)
    tie_f = np.tile(np.array([2, 1], np.int32), n_tie)
    rows_t, rows_f, rows_o = [t], [f], [off]
    all_off = np.concatenate([off, off[-1] + 2 * np.arange(1, n_tie + 1)])
    terms, tfs = np.concatenate(rows_t + [tie_t]), np.concatenate(rows_f + [tie_f])
    order = rng.permutation(n_other + n_tie)                    # interleave the group with the rest
    lens = np.diff(all_off)
    new_t, new_f, new_o = [], [], [0]
    for r in order:
        new_t.append(terms[all_off[r]:all_off[r + 1]])
        new_f.append(tfs[all_off[r]:all_off[r + 1]])
        new_o.append(new_o[-1] + lens[r])
    ids = rng.permutation(n_other + n_tie).astype(np.int64)
    st, m = KeywordIndex(n_other + n_tie), Mirror()
    args = (ids, np.concatenate(new_t), np.concatenate(new_f), np.asarray(new_o, np.int64))
    st.add(*args)
    m.add(*args)
    for q in (np.array([3001], np.int32), np.array([7, 3001], np.int32)):
        ids_out, sc, _ = assert_matches_oracle(st, m, q, np.array([0, len(q)]), k)
        if len(q) == 1:
            assert (sc[0] == sc[0][0]).all()                    # the whole list is one tie group


def test_upserts_removes_compaction_and_growth():
    """Upserts and removes keep N / df / avgdl equal to BM25Index's, so every score stays bit-identical; compaction
    changes no answer and reports what it reclaimed; the posting array grows mid-run from a tiny start."""
    rng = np.random.default_rng(3)
    words = [f"w{i}" for i in range(300)]
    text = lambda: " ".join(rng.choice(words, size=int(rng.integers(0, 30)), p=None))   # noqa: E731
    dev = bm25.DeviceBM25(4096, postings_capacity=16)
    host = bm25.BM25Index()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        for step in range(6):
            ids = rng.integers(0, 400, size=120)
            texts = [text() for _ in ids]
            dev.add_many(ids, texts)
            for d, t in zip(ids, texts):
                host.add(int(d), t)
            gone = rng.integers(0, 400, size=30)
            dev.remove_many(gone)
            for d in gone:
                host.remove(int(d))
            queries = [text() for _ in range(20)] + ["w1 w2 w3", "nothing", ""]
            got = dev.search_batch(queries, 50)
            assert got == [host.search(q, 50) for q in queries], step
            assert dev.search(queries[0], 7) == host.search(queries[0], 7)
        s = dev.stats()
        assert s["postings_allocated"] > 16 and s["live"] == len(host)
        before = dev.search_batch(queries, 50)
        dead = s["docs"] - s["live"]
        assert dev.compact() == dead and dead > 0
        assert dev.stats()["docs"] == len(host)
        assert dev.search_batch(queries, 50) == before
        assert dev.compact() == 0


def test_scopes_and_allow_lists():
    n = 30_000
    st, m, rng = _store(n, seed=9)
    # re-add with tenant codes: 40 users, 8 orgs (the upsert path, exclusively)
    t, f, off = m.csr()
    user = rng.integers(0, 40, n).astype(np.int32)
    org = np.where(rng.random(n) < 0.5, rng.integers(0, 8, n), -1).astype(np.int32)
    ids = np.asarray(m.ids, np.int64)
    st.add(ids, t, f, off, user, org)
    m.add(ids, t, f, off, user, org)
    nq = 300
    qt, qo = zipf_queries(rng, nq)
    q_user = rng.integers(-2, 42, nq).astype(np.int32)           # > 32 distinct scopes, unknown codes
    q_org = rng.integers(-1, 9, nq).astype(np.int32)
    assert_matches_oracle(st, m, qt, qo, 20, q_user, q_org, sample=range(0, nq, 7))
    assert_matches_oracle(st, m, qt, qo, 20, q_user, None, sample=range(3, nq, 11))
    allow = rng.choice(ids, 3000, replace=False)
    allow = np.concatenate([allow, [10 ** 12, 5]])                # unknown ids are ignored
    assert_matches_oracle(st, m, qt, qo[:7], 16, allow_ids=allow)
    assert_matches_oracle(st, m, qt, qo[:7], 16, q_user[:6], q_org[:6], allow_ids=allow)
    ids_out, _, _ = st.search(qt, qo, 4, allow_ids=np.zeros(0, np.int64))
    assert (ids_out == -1).all()


def test_concurrent_writer_and_readers():
    rng = np.random.default_rng(11)
    t, f, off = zipf_docs(rng, 60_000)
    st, m = KeywordIndex(60_000), Mirror()
    qt, qo = zipf_queries(rng, 24)
    chunks = np.array_split(np.arange(60_000), 30)
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
    m.add(np.arange(60_000, dtype=np.int64), t, f, off)
    snaps = sorted({a[2] for a in answers})
    assert len(snaps) >= 2
    for ids, scores, snap in answers[:: max(1, len(answers) // 12)]:
        corpus = m.corpus(n_rows=snap)
        from oracle.bm25_topk import bm25_topk

        wi, ws = bm25_topk(corpus, qt, qo, 16)
        assert np.array_equal(ids, wi) and np.array_equal(scores.view(np.int64), ws.view(np.int64)), snap


# ----------------------------------------------------------------------------- retriever
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


def test_retriever_device_keyword_leg_matches_host_loop_path(tmp_path):
    from aurora_b200 import retriever as R
    from aurora_b200.filters import Filter
    from tests.doubles import HashEmbedder, OracleIndex

    emb = HashEmbedder(64)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        dev = R.KnowledgeBase(emb, capacity=4096)
        host = R.KnowledgeBase(emb, capacity=4096, index_factory=lambda d, c: OracleIndex(d, c))
        assert isinstance(dev.sparse, bm25.DeviceBM25) and isinstance(host.sparse, bm25.BM25Index)
        for kb in (dev, host):
            _fill(kb)
            kb.delete_where(lambda p: p.get("document_id") == "doc3" and p.get("chunk_index", 0) % 5 == 0)
        queries = ["disk node-7", "oom pods memory", "timeout", "nothing matches this", "latency failover disk"]
        flt = Filter.by_property("document_id").like("doc*") & Filter.by_property("user_id").equal("u1")

        def compare(a, b):
            for q in queries:
                for alpha in (0.0, 0.5, 1.0):
                    for scope in (("u1", None), ("u2", "o1"), ("zz", "o2")):
                        ra = a.query(q, 10, user_id=scope[0], org_id=scope[1], alpha=alpha, scoped=True)
                        rb = b.query(q, 10, user_id=scope[0], org_id=scope[1], alpha=alpha, scoped=True)
                        assert _shape(ra) == _shape(rb), (q, alpha, scope)
                    assert _shape(a.query(q, 10, filters=flt, alpha=alpha)) == _shape(b.query(q, 10, filters=flt, alpha=alpha))
                    assert _shape(a.query(q, 10, alpha=alpha)) == _shape(b.query(q, 10, alpha=alpha))
            reqs = [("u1", q, 6, a_, None) for q in queries for a_ in (0.0, 0.5, None)] + \
                   [("u2", q, 4, 0.3, "o1") for q in queries] + [(None, "disk", 3, 0.5, "o2")]
            assert [_shape(x) for x in a.query_batch(reqs)] == [_shape(x) for x in b.query_batch(reqs)]

        compare(dev, host)
        dev.save(str(tmp_path / "dev"))
        host.save(str(tmp_path / "host"))
        dev2 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=4096)
        host2 = R.KnowledgeBase.load(str(tmp_path / "host"), emb, capacity=4096,
                                     index_loader=lambda p, c: OracleIndex.load(p, c))
        compare(dev2, host2)
        # WAL replay: mutations after the snapshot come back on both
        for kb, d in ((dev2, "dev"), (host2, "host")):
            kb.attach_wal(str(tmp_path / f"{d}.wal"))
            kb.insert("u1", "late", "f.md", [{"content": "late disk oom entry", "chunk_index": 0}])
            kb.delete_where(lambda p: p.get("document_id") == "doc4")
        dev3 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=4096)
        dev3.attach_wal(str(tmp_path / "dev.wal"))
        host3 = R.KnowledgeBase.load(str(tmp_path / "host"), emb, capacity=4096,
                                     index_loader=lambda p, c: OracleIndex.load(p, c))
        host3.attach_wal(str(tmp_path / "host.wal"))
        compare(dev3, host3)


def test_default_hybrid_calls_never_use_the_host_index(monkeypatch):
    """search_knowledge_base(alpha=0.5) and the daemon's coalesced batches on a CUDA index stay on the device."""
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder

    def boom(*a, **k):
        raise AssertionError("BM25Index.search called on a CUDA knowledge base")

    R.configure(encoder=HashEmbedder(64), capacity=2048)
    try:
        kb = R._get_kb()
        _fill(kb, 5)
        monkeypatch.setattr(bm25.BM25Index, "search", boom)
        calls = []
        real = bm25.DeviceBM25.search_batch
        monkeypatch.setattr(bm25.DeviceBM25, "search_batch", lambda self, *a, **k: calls.append(1) or real(self, *a, **k))
        assert R.search_knowledge_base("u1", "disk node-7 oom", limit=5)
        assert len(calls) == 1
        res = R.search_knowledge_base_batch([("u1", "disk", 5, 0.5, 0.0, None), ("u2", "timeout", 5, 0.0, 0.0, "o1"),
                                             ("u3", "payment", 5, 0.7, 0.0, None)])
        assert all(res) and len(calls) == 2                    # one device search for the whole batch
    finally:
        R.configure(factory=lambda: (_ for _ in ()).throw(RuntimeError("unconfigured")))


def test_delete_between_batched_keyword_search_and_fusion(monkeypatch):
    """A document deleted after query_batch's one keyword search and before fusion (another handler thread's delete)
    drops out of the answer; the batch does not fail."""
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder

    kb = R.KnowledgeBase(HashEmbedder(64), capacity=1024)
    _fill(kb, 3)
    real = bm25.DeviceBM25.search_batch
    gone = []

    def search_then_delete(self, *a, **k):
        out = real(self, *a, **k)
        victim = next(d for lst in out for d, _ in lst)
        gone.append(kb._id2key[victim])
        kb._delete_keys([gone[-1]])
        return out

    monkeypatch.setattr(bm25.DeviceBM25, "search_batch", search_then_delete)
    res = kb.query_batch([("u1", "disk node-7", 5, 0.5, None), ("u1", "oom pods", 5, 0.0, None)])
    assert len(gone) == 1 and res[0] and res[1]
    assert all(o.uuid != gone[0] for objs in res for o in objs)


def test_add_rejects_falling_offsets_before_reading_postings():
    """offsets that rise and fall back to 0 with NULL term_ids / tfs: refused as invalid, the arrays are never read."""
    import ctypes as C

    st = KeywordIndex(16)
    lib = N.load()
    ids = np.array([1, 2], np.int64)
    off = np.array([0, 5, 0], np.int64)
    rc = lib.aur_kw_add(st._h, ids.ctypes.data_as(C.c_void_p), None, None, None, None, off.ctypes.data_as(C.c_void_p), 2)
    assert rc == N.AUR_ERR_INVALID and b"offsets" in lib.aur_last_error()
    off = np.array([0, 0, 3], np.int64)
    rc = lib.aur_kw_add(st._h, ids.ctypes.data_as(C.c_void_p), None, None, None, None, off.ctypes.data_as(C.c_void_p), 2)
    assert rc == N.AUR_ERR_INVALID and b"term_ids" in lib.aur_last_error()
    assert st.stats()["docs"] == 0

"""Keyword analysis on the GPU (aur_kw_vocab_*, aur_kw_add_text, csrc/kw_text.cu) held to bm25.build_csr: the device
vocabulary and the rows it writes equal build_csr's for the same texts, and a store fed text answers every search
exactly as a store fed build_csr's rows does."""

import sys
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import KeywordIndex, KeywordVocab, MultiKeywordIndex
from tests.keyword_mirror import Mirror, assert_matches_oracle

pytestmark = pytest.mark.gpu

WORDS = ["disk", "Node-7", "OOM", "pods", "memory", "timeout", "10.0.3.17", "0xdeadBEEF", "latency", "failover", "kafka",
         "dns", "İstanbul", "Kelvin", "café", "naïve", "Über", "x86_64", "HTTP/2", "disk-full"]


def _gpus():
    return N.load().aur_device_count()


def _zipf_texts(rng, n, mean_words=30, vocab=400):
    out = []
    for _ in range(n):
        k = int(rng.poisson(mean_words))
        ws = [WORDS[i] if i < len(WORDS) else f"w{i}" for i in (rng.zipf(1.3, k) - 1) % vocab]
        out.append(" ".join(ws))
    return out


def _rand_unicode(rng, n, length=60):
    pts = rng.integers(0, 0x2FFFF, size=(n, length))
    ok = lambda c: not (0xD800 <= c <= 0xDFFF)   # noqa: E731  (surrogates have no UTF-8)
    return ["".join(chr(int(c)) for c in row if ok(c)) for row in pts]


def _batches(rng):
    """The analyzer's inputs, in the order they grow one vocabulary."""
    yield []
    yield ["The quick brown fox"]
    yield _zipf_texts(rng, 255)
    yield _zipf_texts(rng, 256)
    yield _zipf_texts(rng, 257)
    yield ["", "   ", "!!--..", "\x00", "a\x00b\x00\x00c", "", "\t\n\r", "ABC abc AbC"]
    yield ["z" * (1 << 20), " ".join(["repeat"] * 70000), "Y" * (1 << 20) + "q"]
    yield ["".join(chr(int(c)) for c in rng.integers(32, 127, 200)) for _ in range(100)]
    yield _rand_unicode(rng, 100)
    # every Unicode scalar value between two ASCII letters
    cps = [c for c in range(sys.maxunicode + 1) if not (0xD800 <= c <= 0xDFFF)]
    yield [" ".join(f"x{chr(c)}y" for c in cps[i:i + 1000]) for i in range(0, len(cps), 1000)]
    # U+0130 and U+212A at the text's edges and inside words
    yield ["İ", "K", "İabc", "abcİ", "abİcd", "Kab", "abK", "aKb", "KK",
           "İİ", "KKk", "İKİ", "ẋy", "K1İ2", "lone\ud83dsurrogate", "\udc00x\ud800"]
    yield _zipf_texts(rng, 10000, mean_words=20)


def _rows_equal(store, row0, terms, tfs, offsets, ids):
    got_ids, got_off, got_t, got_f = store.read_rows(row0, len(ids))
    assert np.array_equal(got_ids, np.asarray(ids, np.int64))
    assert np.array_equal(got_off, offsets)
    assert np.array_equal(got_t, terms) and np.array_equal(got_f, tfs)


@pytest.mark.parametrize("hash_bits", [64, 4, 1])
def test_analyzer_equals_build_csr(hash_bits):
    rng = np.random.default_rng(5)
    vocab = KeywordVocab(0)
    vocab.set_option("hash_bits", hash_bits)
    store = KeywordIndex(40000, postings_capacity=1 << 22)
    ref = {}
    row = 0
    for texts in _batches(rng):
        terms, tfs, offsets = bm25.build_csr(ref, texts)
        ids = np.arange(row, row + len(texts), dtype=np.int64)
        store.add_text(vocab, ids, texts)
        assert vocab.size()[0] == len(ref)
        assert vocab.read() == list(ref)                 # dict order is id order
        _rows_equal(store, row, terms, tfs, offsets, ids)
        row += len(texts)
    assert vocab.size()[1] == sum(len(w) for w in ref)
    with pytest.raises(N.AuroraError):
        vocab.set_option("hash_bits", 64)                # only on an empty vocabulary
    store.close(); vocab.close()


def test_vocab_read_count_mode_and_argument_checks():
    import ctypes as C

    vocab = KeywordVocab(0)
    store = KeywordIndex(16)
    store.add_text(vocab, [0, 1], ["alpha beta", "gamma alpha delta"])
    lib, h = N.load(), vocab._h
    off = np.zeros(5, np.int64)
    assert lib.aur_kw_vocab_read(h, 0, 4, None, 0, off.ctypes.data_as(C.c_void_p)) == N.AUR_OK
    assert off.tolist() == [0, 5, 9, 14, 19]
    buf = C.create_string_buffer(19)
    off2 = np.full(5, -7, np.int64)
    assert lib.aur_kw_vocab_read(h, 0, 4, buf, 18, off2.ctypes.data_as(C.c_void_p)) == N.AUR_ERR_INVALID
    assert (off2 == -7).all() and buf.raw == b"\0" * 19    # nothing written
    assert lib.aur_kw_vocab_read(h, 3, 2, None, 0, off.ctypes.data_as(C.c_void_p)) == N.AUR_ERR_INVALID
    assert vocab.read(1, 2) == ["beta", "gamma"]
    for bad in (0, 65):
        with pytest.raises(N.AuroraError):
            KeywordVocab(0).set_option("hash_bits", bad)
    with pytest.raises(N.AuroraError):
        vocab.set_option("nope", 1)
    handles = (C.c_void_p * 2)(store._h.value, store._h.value)
    ids = np.array([5], np.int64)
    toff = np.array([0, 1], np.int64)
    args = lambda hs, n: (hs, n, h, ids.ctypes.data_as(C.c_void_p), None, None, b"x", toff.ctypes.data_as(C.c_void_p), 1)  # noqa: E731
    assert lib.aur_kw_add_text(*args(handles, 2)) == N.AUR_ERR_INVALID          # a store twice
    assert lib.aur_kw_add_text(*args(handles, 0)) == N.AUR_ERR_INVALID
    assert lib.aur_kw_add_text(*args(handles, 65)) == N.AUR_ERR_INVALID
    assert lib.aur_kw_add_text(*args((C.c_void_p * 1)(None), 1)) == N.AUR_ERR_INVALID
    toff[:] = [-1, 0]                                                            # reads before the buffer
    assert lib.aur_kw_add_text(*args((C.c_void_p * 1)(store._h.value), 1)) == N.AUR_ERR_INVALID
    toff[:] = [1, 2]
    assert lib.aur_kw_add_text(*args((C.c_void_p * 1)(store._h.value), 1)) == N.AUR_ERR_INVALID
    assert store.stats()["docs"] == 2 and len(vocab) == 4
    # count mode of aur_kw_read_rows
    total = C.c_int64(-1)
    o = np.zeros(3, np.int64)
    assert lib.aur_kw_read_rows(store._h, 0, 2, None, o.ctypes.data_as(C.c_void_p), None, None, 0, C.byref(total)) == N.AUR_OK
    assert total.value == 5 and o.tolist() == [0, 2, 5]
    assert lib.aur_kw_read_rows(store._h, 1, 2, None, o.ctypes.data_as(C.c_void_p), None, None, 0, C.byref(total)) == N.AUR_ERR_INVALID


# ------------------------------------------------------------------------------------------------ store parity
def _stats(st):
    return {k: v for k, v in st.items() if not k.startswith("last_")}


def _same_answers(a, b, rng, vocab_size, ids_pool):
    nq = 48
    qt, qo = [], [0]
    for _ in range(nq):
        m = int(rng.integers(1, 6))
        qt.extend(np.unique(rng.integers(0, max(vocab_size, 1), m)).tolist())
        qo.append(len(qt))
    qt, qo = np.asarray(qt, np.int32), np.asarray(qo, np.int64)
    qu = rng.integers(0, 3, nq).astype(np.int32)
    qg = rng.integers(-1, 2, nq).astype(np.int32)
    allow = rng.choice(ids_pool, size=min(len(ids_pool), 50), replace=False) if len(ids_pool) else np.zeros(0, np.int64)
    for path in (N.KW_PATH_FORWARD_OPT, N.KW_PATH_INDEX_OPT):
        a.set_path(path); b.set_path(path)
        for scope in ((None, None, None), (qu, None, None), (qu, qg, None), (None, None, allow)):
            ia, sa, _ = a.search(qt, qo, 10, *scope)
            ib, sb, _ = b.search(qt, qo, 10, *scope)
            assert np.array_equal(ia, ib) and np.array_equal(sa.view(np.int64), sb.view(np.int64)), (path, scope)


def _check_pair(a, b, ref, vocab, rng, ids_pool):
    sa, sb = a.stats(), b.stats()
    assert _stats(sa) == _stats(sb)
    n = sa["docs"]
    ra, rb = a.read_rows(0, n), b.read_rows(0, n)
    for x, y in zip(ra, rb):
        assert np.array_equal(x, y)
    assert vocab.read() == list(ref)
    _same_answers(a, b, rng, len(ref), ids_pool)


def test_store_fed_text_equals_store_fed_build_csr():
    rng = np.random.default_rng(11)
    vocab = KeywordVocab(0)
    cap = 3000
    a, b = KeywordIndex(cap), KeywordIndex(cap)
    ref = {}

    def both(ids, texts, user=None, org=None):
        a.add_text(vocab, ids, texts, user, org)
        t, f, o = bm25.build_csr(ref, texts)
        b.add(ids, t, f, o, user, org)

    pool = np.arange(0, 1200, dtype=np.int64)
    for step in range(6):
        n = 300
        ids = rng.choice(pool, size=n, replace=True)                   # upserts within the batch and across calls
        both(ids, _zipf_texts(rng, n), rng.integers(0, 3, n), rng.integers(-1, 2, n))
        if step == 2:
            a.reindex(); b.reindex()
        if step % 2:
            gone = rng.choice(pool, size=80, replace=False)
            assert a.remove(gone) == b.remove(gone)
        for st in (a, b):
            st.set_attrs(2, pool[:400], rng.integers(0, 5, 400))
        _check_pair(a, b, ref, vocab, rng, pool)
    assert a.compact() == b.compact()
    _check_pair(a, b, ref, vocab, rng, pool)
    # the capacity edge: a batch that does not fit leaves both stores and the vocabulary unchanged
    room = cap - a.stats()["docs"]
    before = (len(vocab), a.stats())
    with pytest.raises(N.AuroraError) as e:
        a.add_text(vocab, np.arange(room + 1) + 5000, ["brandnewword"] * (room + 1))
    assert e.value.code == N.AUR_ERR_NOMEM and (len(vocab), a.stats()) == before
    with pytest.raises(N.AuroraError):
        a.add_text(vocab, np.array([-1]), ["anothernewword"])     # a rejected id: nothing changes either
    assert (len(vocab), a.stats()) == before
    both(np.arange(room) + 5000, _zipf_texts(rng, room))            # exactly full
    _check_pair(a, b, ref, vocab, rng, pool)
    a.close(); b.close(); vocab.close()


@pytest.mark.parametrize("n", [1, 2, 3, 8, "all_gpus"])
def test_several_stores(n):
    if n == "all_gpus":
        if _gpus() < 2:
            pytest.skip("needs two or more GPUs")
        devices = [s % _gpus() for s in range(max(_gpus(), 3))]
    else:
        devices = [0] * n
    rng = np.random.default_rng(3)
    vocab = KeywordVocab(0)
    a = MultiKeywordIndex(4096 * len(devices), devices=devices)
    b = MultiKeywordIndex(4096 * len(devices), devices=devices)
    ref = {}
    for _ in range(3):
        ids = rng.choice(3000, size=700, replace=True).astype(np.int64)
        texts = _zipf_texts(rng, 700)
        u, o = rng.integers(0, 3, 700), rng.integers(-1, 2, 700)
        a.add_text(vocab, ids, texts, u, o)
        t, f, off = bm25.build_csr(ref, texts)
        b.add(ids, t, f, off, u, o)
    assert vocab.read() == list(ref)
    for s, (sa, sb) in enumerate(zip(a.stores, b.stores)):
        assert _stats(sa.stats()) == _stats(sb.stats())
        ra, rb = sa.read_rows(0, sa.stats()["docs"]), sb.read_rows(0, sb.stats()["docs"])
        for x, y in zip(ra, rb):
            assert np.array_equal(x, y)
        assert np.all(ra[0] % len(devices) == s)
    _same_answers(a, b, rng, len(ref), np.arange(3000))
    a.close(); b.close(); vocab.close()


def test_writer_adding_text_under_three_readers():
    rng = np.random.default_rng(8)
    vocab = KeywordVocab(0)
    store = KeywordIndex(20000)
    mirror, ref = Mirror(), {}
    batches = [(np.arange(i * 200, (i + 1) * 200, dtype=np.int64), _zipf_texts(rng, 200)) for i in range(30)]
    for ids, texts in batches:                      # the mirror knows every row the writer will publish
        mirror.add(ids, *bm25.build_csr(ref, texts))
    q = [" ".join(rng.choice(WORDS, 3)) for _ in range(16)]
    qt, qo = bm25.query_csr(ref, q)
    errors, done = [], threading.Event()

    def reader():
        try:
            while not done.is_set():
                assert_matches_oracle(store, mirror, qt, qo, 10, sample=range(0, 16, 5))
        except Exception as exc:   # noqa: BLE001
            errors.append(exc)

    threads = [threading.Thread(target=reader) for _ in range(3)]
    for t in threads:
        t.start()
    for ids, texts in batches:
        store.add_text(vocab, ids, texts)
    done.set()
    for t in threads:
        t.join()
    assert not errors, errors[0]
    assert vocab.read() == list(ref)
    assert_matches_oracle(store, mirror, qt, qo, 10)
    store.close(); vocab.close()


# ------------------------------------------------------------------------------------------------ knowledge base
@pytest.mark.parametrize("multi", [False, True])
def test_knowledge_base_analyses_text_on_the_device(multi, monkeypatch, tmp_path):
    from aurora_b200 import retriever as R
    from aurora_b200.engine import MultiIndex
    from aurora_b200.filters import Filter as F
    from aurora_b200.filters import HybridFusion
    from tests.doubles import HashEmbedder, OracleIndex

    emb = HashEmbedder(64)
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    factory = (lambda d, c: MultiIndex(d, c, devices=[0, 0, 0])) if multi else None
    host = R.KnowledgeBase(emb, capacity=8192, index_factory=lambda d, c: OracleIndex(d, c))

    def boom(*a, **k):
        raise AssertionError("build_csr on the device analysis path")

    real_build_csr = bm25.build_csr
    monkeypatch.setattr(bm25, "build_csr", boom)
    dev = R.KnowledgeBase(emb, capacity=8192, index_factory=factory)
    assert isinstance(dev.sparse, bm25.DeviceBM25) and dev._hybrid_device

    inserted = []

    def fill(kb, log=None):
        r = np.random.default_rng(1)
        for t in range(20):
            for doc in range(3):
                chunks = [{"chunk_index": c, "content": " ".join(r.choice(WORDS, size=8))} for c in range(6)]
                kb.insert(f"u{t}", f"discovery:{t}:{doc}" if doc == 0 else f"doc{t}-{doc}", "f.md", chunks, org_id=f"o{t % 5}")
                if log is not None:
                    log.extend(c["content"] for c in chunks)
        kb.delete_where(lambda p: p.get("document_id") == "doc3-1")

    fill(host)
    fill(dev, inserted)
    queries = ["disk node-7", "OOM pods memory", "İstanbul kelvin", "nothing matches", "10.0.3.17 0xdeadbeef"]
    flts = [F.by_property("org_id").equal("o3") & F.by_property("document_id").like("discovery:*"),
            F.by_property("document_id").like("doc*") & F.by_property("user_id").equal("u1")]

    def shape(objs):
        return [(o.uuid, o.metadata.score) for o in objs]

    def compare(a, b, texts):
        ref = {}
        real_build_csr(ref, texts)
        assert a.sparse.vocab == ref
        for q in queries:
            for alpha in (0.0, 0.5):
                assert shape(a.query(q, 10, alpha=alpha)) == shape(b.query(q, 10, alpha=alpha))
                assert shape(a.query(q, 10, user_id="u2", org_id="o2", alpha=alpha, scoped=True)) == \
                    shape(b.query(q, 10, user_id="u2", org_id="o2", alpha=alpha, scoped=True))
                for f in flts:
                    assert shape(a.query(q, 10, filters=f, alpha=alpha, fusion=HybridFusion.RANKED)) == \
                        shape(b.query(q, 10, filters=f, alpha=alpha, fusion=HybridFusion.RANKED))
        reqs = [("u1", q, 6, a_, None) for q in queries for a_ in (0.0, 0.5, None)] + [("u2", q, 4, 0.3, "o1") for q in queries]
        assert [shape(x) for x in a.query_batch(reqs)] == [shape(x) for x in b.query_batch(reqs)]

    compare(dev, host, inserted)
    if multi:
        return                                     # save / load goes through an engine.Index shard
    dev.save(str(tmp_path / "dev"))
    dev2 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=8192)
    compare(dev2, host, [dev2._props[r]["content"] for r in dev2._props])
    snap = [dev2._props[r]["content"] for r in dev2._props]
    late = ("u1", "late", "f.md", [{"content": "late disk oom entry brandnew", "chunk_index": 0}])
    dev2.attach_wal(str(tmp_path / "dev.wal"))
    dev2.insert(*late)
    host.insert(*late)
    dev3 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=8192)
    dev3.attach_wal(str(tmp_path / "dev.wal"))             # replays the late insert
    compare(dev3, host, snap + [late[3][0]["content"]])

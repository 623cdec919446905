"""Sharded GPU keyword store (aur_kw_search_multi, engine.MultiKeywordIndex, the retriever over a MultiIndex).  Every
answer is held to the fp64 oracle (oracle/bm25_topk.py) over the whole corpus and to a single KeywordIndex holding the
same documents: ids exact, fp64 scores bit-identical.  The stores share device 0; where the machine has several GPUs
the same cases also run with the stores spread over them."""

import ctypes as C
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import KeywordIndex, MultiKeywordIndex
from oracle.bm25_topk import Corpus, bm25_topk
from tests.keyword_mirror import Mirror, zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

QBLOCK = 256


def _gpus():
    return N.load().aur_device_count()


@pytest.fixture(params=["device0", "per_gpu"])
def layout(request):
    if request.param == "per_gpu" and _gpus() < 2:
        pytest.skip("one store per GPU needs two or more GPUs; this machine has fewer")
    return request.param


def _devices(n, layout):
    return [0] * n if layout == "device0" else [s % _gpus() for s in range(n)]


def _rows(t, f, off, sel):
    """CSR rows sel of (t, f, off), offsets rebased."""
    lens = off[sel + 1] - off[sel]
    sub = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    take = np.repeat(off[sel] - sub[:-1], lens) + np.arange(sub[-1], dtype=np.int64)
    return t[take], f[take], sub


class Sharded:
    """A MultiKeywordIndex beside a single KeywordIndex with the same documents, a mirror of the union and one per
    store (the rows each store appended, for the snapshot prefixes it reports)."""

    def __init__(self, n, layout, capacity=100_000, postings_capacity=0):
        self.n = n
        self.multi = MultiKeywordIndex(capacity, devices=_devices(n, layout), postings_capacity=postings_capacity)
        self.single = KeywordIndex(capacity * 2)
        self.mirror = Mirror()
        self.parts = [Mirror() for _ in range(n)]

    def add(self, ids, t, f, off, user=None, org=None):
        ids = np.asarray(ids, np.int64)
        self.multi.add(ids, t, f, off, user, org)
        self.single.add(ids, t, f, off, user, org)
        self.mirror.add(ids, t, f, off, user, org)
        self._add_parts(ids, t, f, off, user, org)

    def _add_parts(self, ids, t, f, off, user=None, org=None):
        for s in range(self.n):
            sel = np.nonzero(ids % self.n == s)[0]
            if len(sel):
                self.parts[s].add(ids[sel], *_rows(t, f, off, sel), None if user is None else user[sel],
                                  None if org is None else org[sel])

    def remove(self, ids):
        got = self.multi.remove(ids)
        assert got == self.single.remove(ids)
        self.mirror.remove(ids)
        for m in self.parts:
            m.remove(ids)
        return got

    def compact(self):
        got = self.multi.compact()
        assert got == self.single.compact()
        self.mirror.compact()
        for m in self.parts:
            m.compact()
        return got

    def check(self, qt, qo, k, q_user=None, q_org=None, allow_ids=None, sample=None):
        ids, sc, snaps = self.multi.search(qt, qo, k, q_user, q_org, allow_ids)
        assert snaps == [len(m.ids) for m in self.parts]
        si, ss, _ = self.single.search(qt, qo, k, q_user, q_org, allow_ids)
        assert np.array_equal(ids, si) and np.array_equal(sc.view(np.int64), ss.view(np.int64))
        assert_oracle(self.mirror.corpus(), ids, sc, qt, qo, k, q_user, q_org, allow_ids, sample)
        return ids, sc


def assert_oracle(corpus, ids, sc, qt, qo, k, q_user=None, q_org=None, allow_ids=None, sample=None):
    for q in range(len(qo) - 1) if sample is None else sample:
        wi, ws = bm25_topk(corpus, qt[qo[q]:qo[q + 1]], np.array([0, qo[q + 1] - qo[q]]), k,
                           None if q_user is None else q_user[q:q + 1], None if q_org is None else q_org[q:q + 1], allow_ids)
        assert np.array_equal(ids[q], wi[0]), (q, ids[q][:8], wi[0][:8])
        assert np.array_equal(sc[q].view(np.int64), ws[0].view(np.int64)), (q, sc[q][:4], ws[0][:4])


def union_corpus(parts, snaps):
    """The oracle's corpus of the union of every store's reported prefix."""
    ts, fs, offs, ids, live, base = [], [], [0], [], [], 0
    for m, r in zip(parts, snaps):
        t, f, off = m.csr()
        ts.append(t[:off[r]]); fs.append(f[:off[r]])
        offs.extend((base + off[1:r + 1]).tolist())
        base += int(off[r])
        ids += m.ids[:r]; live += m.live[:r]
    return Corpus(np.concatenate(ts), np.concatenate(fs), offs, ids, live)


def _filled(n, layout, n_docs, seed, **kw):
    rng = np.random.default_rng(seed)
    sh = Sharded(n, layout, capacity=max(n_docs, 1) * 2)
    if n_docs:
        t, f, off = zipf_docs(rng, n_docs, **kw)
        sh.add(rng.permutation(n_docs).astype(np.int64) * 5 + 2, t, f, off)      # shuffled, sparse ids
    return sh, rng


# ----------------------------------------------------------------------------- store counts, k, query shapes
@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("k", [1, 128])
@pytest.mark.parametrize("n_docs", [5, 6000])
def test_store_counts_and_k(n, k, n_docs, layout):
    """n_docs 5 over 8 stores: some stores stay empty and answer with padding only."""
    sh, rng = _filled(n, layout, n_docs, seed=n * 100 + k + n_docs)
    qt, qo = zipf_queries(rng, 17)
    sh.check(qt, qo, k)
    if n_docs < n:
        assert min(s["docs"] for s in sh.multi.stats()["stores"]) == 0


@pytest.mark.parametrize("nq", [1, QBLOCK - 1, QBLOCK, QBLOCK + 1, 1025])
def test_query_blocks(nq, layout):
    sh, rng = _filled(3, layout, 20_000, seed=nq)
    qt, qo = zipf_queries(rng, nq)
    sh.check(qt, qo, 32, sample=sorted({0, nq // 2, nq - 1, min(QBLOCK, nq - 1)}))


def _spill_threshold(nq):
    """Distinct live terms above which a launch of nq queries keeps its contribution table in global memory
    (csrc/keyword.cu, kw_score_kernel: nq x 20 B + 8 warps x 256 x 16 B, rounded to 16, plus 64 B per term)."""
    import torch

    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    return (optin - (nq * 16 + 8 * 256 * 16 + 4 * nq + 15) // 16 * 16) // 64


def _uniform(n, layout, n_docs, vocab, words, seed):
    rng = np.random.default_rng(seed)
    terms, tfs, off = [], [], [0]
    for _ in range(n_docs):
        u, c = np.unique(rng.integers(0, vocab, words), return_counts=True)
        terms.append(u.astype(np.int32)); tfs.append(c.astype(np.int32)); off.append(off[-1] + len(u))
    t = np.concatenate(terms)
    sh = Sharded(n, layout, capacity=n_docs)
    sh.add(np.arange(n_docs, dtype=np.int64) * 7 + 3, t, np.concatenate(tfs), np.asarray(off, np.int64))
    return sh, rng, np.unique(t)


def test_unknown_repeated_terms_and_spilled_blocks(layout):
    sh, rng, live = _uniform(3, layout, 6000, 12_000, 80, seed=7)
    q = rng.permutation(live)[:40].astype(np.int32)
    q = np.concatenate([q, q[:13], np.array([20_000, 20_001], np.int32)])       # repeats and unknown ids are ignored
    unknown = np.array([20_000, 20_001, 2 ** 27], np.int32)                       # a query with no known term
    qt = np.concatenate([q, unknown])
    sh.check(qt, np.array([0, len(q), len(qt), len(qt)]), 64)                   # ... and an empty one
    ids, sc, _ = sh.multi.search(unknown, np.array([0, 3]), 5)
    assert (ids == -1).all() and np.isneginf(sc).all()
    # a 256-query block whose distinct terms exceed shared memory: every store spills, every answer exact
    per = _spill_threshold(QBLOCK) // QBLOCK + 8
    qs = [rng.choice(live, per, replace=False).astype(np.int32) for _ in range(QBLOCK)]
    qt, qo = np.concatenate(qs), np.concatenate([[0], np.cumsum([len(x) for x in qs])]).astype(np.int64)
    assert len(np.unique(qt)) > _spill_threshold(QBLOCK)
    sh.check(qt, qo, 16, sample=range(0, QBLOCK, 17))
    st = sh.multi.stats()
    assert [s["last_spilled"] for s in st["stores"]] == [1, 1, 1]
    assert [s["last_terms"] for s in st["stores"]] == [len(np.unique(qt))] * 3


# ----------------------------------------------------------------------------- the statistics must be the corpus's
@pytest.mark.parametrize("n", [2, 3, 8])
def test_term_held_by_one_store_gets_the_corpus_idf(n, layout):
    """Term 9000 appears only in documents with ids = 0 mod n (all in store 0): its idf from store 0's own N and df
    would differ from the corpus's, and so would every score it contributes to."""
    rng = np.random.default_rng(n)
    n_docs = 4000
    t, f, off = zipf_docs(rng, n_docs, vocab=3000)
    ids = np.arange(n_docs, dtype=np.int64)
    rows_t, rows_f, new_off = [], [], [0]
    for i in range(n_docs):
        rt, rf = t[off[i]:off[i + 1]], f[off[i]:off[i + 1]]
        if i % n == 0 and rng.random() < 0.3:
            rt, rf = np.append(rt, 9000).astype(np.int32), np.append(rf, int(rng.integers(1, 4))).astype(np.int32)
        rows_t.append(rt); rows_f.append(rf); new_off.append(new_off[-1] + len(rt))
    sh = Sharded(n, layout, capacity=n_docs)
    sh.add(ids, np.concatenate(rows_t), np.concatenate(rows_f), np.asarray(new_off, np.int64))
    qt = np.array([9000, 0, 9000, 5, 9000, 17, 40], np.int32)
    ids_out, _ = sh.check(qt, np.array([0, 1, 3, 5, 7]), 128)
    assert (ids_out[0][ids_out[0] >= 0] % n == 0).all() and (ids_out[0] >= 0).sum() > 100


@pytest.mark.parametrize("n", [2, 3])
def test_stores_of_very_different_lengths_get_the_corpus_avgdl(n, layout):
    """Store 0 holds long documents, the others short ones: each store's own avgdl is far from the corpus's."""
    rng = np.random.default_rng(30 + n)
    n_docs = 6000
    ids = np.arange(n_docs, dtype=np.int64)
    long_t, long_f, long_o = zipf_docs(rng, n_docs, vocab=2000, mean_len=300)
    short_t, short_f, short_o = zipf_docs(rng, n_docs, vocab=2000, mean_len=6, min_len=1)
    rows_t, rows_f, off = [], [], [0]
    for i in range(n_docs):
        t, f, o = (long_t, long_f, long_o) if i % n == 0 else (short_t, short_f, short_o)
        rows_t.append(t[o[i]:o[i + 1]]); rows_f.append(f[o[i]:o[i + 1]]); off.append(off[-1] + o[i + 1] - o[i])
    sh = Sharded(n, layout, capacity=n_docs)
    sh.add(ids, np.concatenate(rows_t), np.concatenate(rows_f), np.asarray(off, np.int64))
    per = sh.multi.stats()["stores"]
    assert per[0]["total_len"] / per[0]["live"] > 20 * per[1]["total_len"] / per[1]["live"]
    qt, qo = zipf_queries(rng, 24, vocab=2000)
    sh.check(qt, qo, 50)


# ----------------------------------------------------------------------------- ties, scopes, allow-lists
@pytest.mark.parametrize("k", [1, 100, 128])
def test_tie_groups_spread_over_stores_are_cut_by_id(k, layout):
    """5 000 identical documents (bit-equal scores) among 20 000 others, ids shuffled over 3 stores: the cut keeps the
    lowest ids of the group whichever store holds them."""
    rng = np.random.default_rng(k)
    n_tie, n_other = 5000, 20_000
    t, f, off = zipf_docs(rng, n_other, vocab=3000)
    terms = np.concatenate([t, np.tile(np.array([7, 3001], np.int32), n_tie)])
    tfs = np.concatenate([f, np.tile(np.array([2, 1], np.int32), n_tie)])
    off = np.concatenate([off, off[-1] + 2 * np.arange(1, n_tie + 1)])
    sh = Sharded(3, layout, capacity=n_other + n_tie)
    sh.add(rng.permutation(n_other + n_tie).astype(np.int64), terms, tfs, off)
    for q in (np.array([3001], np.int32), np.array([7, 3001], np.int32)):
        ids, sc = sh.check(q, np.array([0, len(q)]), k)
        if len(q) == 1:
            assert (sc[0] == sc[0][0]).all()
            assert len({int(d) % 3 for d in ids[0]}) == min(3, k)


def test_scopes_allow_lists_and_a_store_of_tombstones(layout):
    n, n_docs = 4, 30_000
    rng = np.random.default_rng(9)
    t, f, off = zipf_docs(rng, n_docs)
    ids = rng.permutation(n_docs).astype(np.int64)
    user = rng.integers(0, 40, n_docs).astype(np.int32)
    org = np.where(rng.random(n_docs) < 0.5, rng.integers(0, 8, n_docs), -1).astype(np.int32)
    sh = Sharded(n, layout, capacity=n_docs)
    sh.add(ids, t, f, off, user, org)
    nq = 300
    qt, qo = zipf_queries(rng, nq)
    q_user = rng.integers(-2, 42, nq).astype(np.int32)                            # > 32 distinct scopes, unknown codes
    q_org = rng.integers(-1, 9, nq).astype(np.int32)
    sh.check(qt, qo, 20, q_user, q_org, sample=range(0, nq, 7))
    sh.check(qt, qo, 20, q_user, None, sample=range(3, nq, 11))
    allow = np.concatenate([rng.choice(ids, 3000, replace=False), [10 ** 12, 5]])  # ids in every store, unknown ones
    assert len({int(d) % n for d in allow}) == n
    sh.check(qt, qo[:8], 16, allow_ids=allow)
    sh.check(qt, qo[:8], 16, q_user[:7], q_org[:7], allow_ids=allow)
    assert (sh.multi.search(qt, qo, 4, allow_ids=np.zeros(0, np.int64))[0] == -1).all()
    # every document of store 1 tombstoned: it still counts nothing, scans its rows and matches none
    gone = ids[ids % n == 1]
    assert sh.remove(gone) == len(gone)
    st = sh.multi.stats()["stores"]
    assert st[1]["live"] == 0 and st[1]["docs"] == len(gone)
    ids_out, _ = sh.check(qt, qo, 20, sample=range(0, nq, 13))
    assert not (ids_out[ids_out >= 0] % n == 1).any()
    sh.check(qt, qo[:8], 16, allow_ids=allow)


# ----------------------------------------------------------------------------- mutations
def test_upserts_removes_compaction_and_growth_against_bm25index(layout):
    """DeviceBM25 over a MultiKeywordIndex against the host BM25Index, step by step; an upsert lands on the store of
    the old row; posting arrays grow from a tiny start; compaction changes no answer."""
    rng = np.random.default_rng(3)
    words = [f"w{i}" for i in range(300)]
    text = lambda: " ".join(rng.choice(words, size=int(rng.integers(0, 30))))   # noqa: E731
    n = 3
    store = MultiKeywordIndex(4096, devices=_devices(n, layout), postings_capacity=16)
    start = [p["postings_allocated"] for p in store.stats()["stores"]]
    dev, host = bm25.DeviceBM25(store=store), bm25.BM25Index()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        for step in range(6):
            ids = rng.integers(0, 400, size=120)
            texts = [text() for _ in ids]
            dev.add_many(ids, texts)
            for d, tx in zip(ids, texts):
                host.add(int(d), tx)
            gone = rng.integers(0, 400, size=30)
            dev.remove_many(gone)
            for d in gone:
                host.remove(int(d))
            queries = [text() for _ in range(20)] + ["w1 w2 w3", "nothing", ""]
            assert dev.search_batch(queries, 50) == [host.search(q, 50) for q in queries], step
            assert dev.search(queries[0], 7) == host.search(queries[0], 7)
        # upserts of existing ids = 1 mod 3 only: store 1 appends and tombstones, the others do not move
        before = [dict(s) for s in store.stats()["stores"]]
        up = np.array(sorted(d for d in host._doc_len if d % n == 1)[:25], np.int64)
        texts = [text() for _ in up]
        dev.add_many(up, texts)
        for d, tx in zip(up, texts):
            host.add(int(d), tx)
        after = store.stats()["stores"]
        assert after[1]["docs"] == before[1]["docs"] + len(up) and after[1]["live"] == before[1]["live"]
        assert [(a["docs"], a["live"]) for i, a in enumerate(after) if i != 1] == \
               [(b["docs"], b["live"]) for i, b in enumerate(before) if i != 1]
        assert dev.search_batch(queries, 50) == [host.search(q, 50) for q in queries]
        s = store.stats()
        assert all(p["postings_allocated"] > a for p, a in zip(s["stores"], start)) and s["live"] == len(host)
        before = dev.search_batch(queries, 50)
        dead = s["docs"] - s["live"]
        assert dev.compact() == dead and dead > 0
        assert store.stats()["docs"] == len(host)
        assert dev.search_batch(queries, 50) == before == [host.search(q, 50) for q in queries]


# ----------------------------------------------------------------------------- concurrency
def _run(threads, timeout=300):
    for th in threads:
        th.daemon = True
        th.start()
    for th in threads:
        th.join(timeout)
    assert not any(th.is_alive() for th in threads), "a search or writer did not finish: lock-order defect?"


def test_writer_appending_into_every_store_with_three_readers(layout):
    n, n_docs = 3, 60_000
    rng = np.random.default_rng(11)
    t, f, off = zipf_docs(rng, n_docs)
    ids = np.arange(n_docs, dtype=np.int64)
    sh = Sharded(n, layout, capacity=n_docs)
    qt, qo = zipf_queries(rng, 24)
    chunks = np.array_split(np.arange(n_docs), 30)
    answers, errors = [], []
    done = threading.Event()

    def writer():
        try:
            for c in chunks:
                sh.multi.add(ids[c], *_rows(t, f, off, c))
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader():
        try:
            while not done.is_set():
                answers.append(sh.multi.search(qt, qo, 16))
        except Exception as e:   # pragma: no cover
            errors.append(e)

    _run([threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)])
    assert not errors
    sh._add_parts(ids, t, f, off)
    assert len({tuple(a[2]) for a in answers}) >= 2
    for got_i, got_s, snaps in answers[:: max(1, len(answers) // 12)]:
        assert_oracle(union_corpus(sh.parts, snaps), got_i, got_s, qt, qo, 16)


def test_removing_writers_and_readers_passing_the_stores_in_different_orders(layout):
    """Writers tombstone (exclusive lock, one store at a time) while readers list the stores in different orders: no
    deadlock, and every answer is the oracle's for one state of the removal sequences."""
    n, n_docs = 3, 3000
    sh, rng = _filled(n, layout, n_docs, seed=21)
    qt, qo = zipf_queries(rng, 8)
    live_ids = np.asarray(sh.mirror.ids, np.int64)
    # writer A tombstones in store 0, writer B in stores 1 and 2 by turns: one store per call, so every search sees
    # a prefix of each writer's sequence
    seq_a = [(0, b) for b in np.array_split(rng.permutation(live_ids[live_ids % n == 0])[:300], 5)]
    b1, b2 = (np.array_split(rng.permutation(live_ids[live_ids % n == s])[:300], 4) for s in (1, 2))
    seq_b = [step for x1, x2 in zip(b1, b2) for step in ((1, x1), (2, x2))]
    lib = N.load()
    answers, errors = [], []
    done = [threading.Event(), threading.Event()]
    reading = threading.Event()

    def writer(seq, ev):
        try:
            reading.wait(60)                  # tombstone while the readers are searching
            for s, b in seq:
                sh.multi.stores[s].remove(b)
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            ev.set()

    def reader(order):
        try:
            handles = (C.c_void_p * n)(*[sh.multi.stores[s]._h.value for s in order])
            q_off = qo.astype(np.int64)
            while True:
                finished = all(e.is_set() for e in done)
                sc, ids = np.empty((8, 10)), np.empty((8, 10), np.int64)
                snaps = np.empty(n, np.int64)
                N.check(lib.aur_kw_search_multi(handles, n, qt.ctypes.data_as(C.c_void_p), q_off.ctypes.data_as(C.c_void_p),
                                                8, 10, None, None, None, 0, sc.ctypes.data_as(C.c_void_p),
                                                ids.ctypes.data_as(C.c_void_p), snaps.ctypes.data_as(C.c_void_p)))
                answers.append((ids, sc))
                reading.set()
                if finished:
                    break
        except Exception as e:   # pragma: no cover
            errors.append(e)

    _run([threading.Thread(target=writer, args=(seq_a, done[0])), threading.Thread(target=writer, args=(seq_b, done[1]))]
         + [threading.Thread(target=reader, args=(o,)) for o in ([0, 1, 2], [2, 1, 0], [1, 2, 0])])
    assert not errors and answers
    # the oracle of every (steps of A done, steps of B done) state
    want = {}
    t, f, off = sh.mirror.csr()
    for a in range(len(seq_a) + 1):
        for b in range(len(seq_b) + 1):
            m = Mirror()
            m.add(sh.mirror.ids, t, f, off)
            m.remove(np.concatenate([np.zeros(0, np.int64)] + [x for _, x in seq_a[:a] + seq_b[:b]]))
            want[(a, b)] = bm25_topk(m.corpus(), qt, qo, 10)
    for ids, sc in answers[:: max(1, len(answers) // 20)]:
        assert any(np.array_equal(ids, wi) and np.array_equal(sc.view(np.int64), ws.view(np.int64))
                   for wi, ws in want.values())
    final = sh.multi.search(qt, qo, 10)
    wi, ws = want[(len(seq_a), len(seq_b))]
    assert np.array_equal(final[0], wi) and np.array_equal(final[1].view(np.int64), ws.view(np.int64))


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


def _assert_placement(kb):
    store = kb.sparse.store
    assert isinstance(kb.sparse, bm25.DeviceBM25) and isinstance(store, MultiKeywordIndex)
    n = len(store.stores)
    vocab_ids = np.array(sorted(kb.sparse.vocab.values()), np.int32)
    for s, st in enumerate(store.stores):
        mine = sorted(d for d in kb._props if d % n == s)
        assert st.stats()["live"] == len(mine)
        ids, _, _ = st.search(vocab_ids, np.array([0, len(vocab_ids)]), 128)
        assert len(mine) <= 128 and sorted(int(d) for d in ids[0] if d >= 0) == mine


@pytest.mark.parametrize("spread", ["device0", "all_gpus"])
def test_retriever_over_a_multi_index_matches_the_host_index(spread, tmp_path):
    from aurora_b200 import retriever as R
    from aurora_b200.engine import MultiIndex
    from aurora_b200.filters import Filter
    from tests.doubles import HashEmbedder, OracleIndex

    if spread == "all_gpus" and _gpus() < 2:
        pytest.skip("a KnowledgeBase over all GPUs needs two or more GPUs; this machine has fewer")
    devices = [0, 0, 0] if spread == "device0" else list(range(_gpus()))
    emb = HashEmbedder(64)
    multi = lambda d, c: MultiIndex(d, c, devices=devices)                            # noqa: E731
    multi_load = lambda p, c: MultiIndex.load(p, capacity=c, devices=devices)         # noqa: E731
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        dev = R.KnowledgeBase(emb, capacity=4096, index_factory=multi)
        host = R.KnowledgeBase(emb, capacity=4096, index_factory=lambda d, c: OracleIndex(d, c))
        assert isinstance(host.sparse, bm25.BM25Index)
        assert [st.device for st in dev.sparse.store.stores] == devices
        for kb in (dev, host):
            _fill(kb, 20)
            kb.delete_where(lambda p: p.get("document_id") == "doc3" and p.get("chunk_index", 0) % 5 == 0)
        _assert_placement(dev)
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
        dev2 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=4096, index_loader=multi_load)
        host2 = R.KnowledgeBase.load(str(tmp_path / "host"), emb, capacity=4096,
                                     index_loader=lambda p, c: OracleIndex.load(p, c))
        _assert_placement(dev2)
        compare(dev2, host2)
        for kb, d in ((dev2, "dev"), (host2, "host")):
            kb.attach_wal(str(tmp_path / f"{d}.wal"))
            kb.insert("u1", "late", "f.md", [{"content": "late disk oom entry", "chunk_index": 0}])
            kb.delete_where(lambda p: p.get("document_id") == "doc4")
        dev3 = R.KnowledgeBase.load(str(tmp_path / "dev"), emb, capacity=4096, index_loader=multi_load)
        dev3.attach_wal(str(tmp_path / "dev.wal"))
        host3 = R.KnowledgeBase.load(str(tmp_path / "host"), emb, capacity=4096,
                                     index_loader=lambda p, c: OracleIndex.load(p, c))
        host3.attach_wal(str(tmp_path / "host.wal"))
        _assert_placement(dev3)
        compare(dev3, host3)

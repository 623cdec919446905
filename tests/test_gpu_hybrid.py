"""The hybrid query on the GPU (aur_hybrid_search, engine.hybrid_search, the retriever's fused path).  Every fused list
is held bit for bit to the host definitions (bm25.ranked_fusion / relative_score_fusion) applied to the separate
calls' answers -- aur_search_ex for the dense leg, aur_kw_search for the keyword leg -- over the same snapshot."""

import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import Index, KeywordIndex, hybrid_search, to_bf16_bits
from tests.keyword_mirror import zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu

DIM = 128
ALPHAS = (0.0, 0.3, 0.5, 0.999)
FUSIONS = (N.FUSION_RANKED, N.FUSION_RELATIVE_SCORE)


def host_fuse(d_ids, d_sc, s_ids, s_sc, wd, ws, fusion, k):
    """One query's expected (ids, fp64 scores, fp32 cosines) of length k, padded (-1, -inf, NaN)."""
    dense = [(int(i), float(s)) for i, s in zip(d_ids, d_sc) if i >= 0]
    sparse = [(int(i), float(s)) for i, s in zip(s_ids, s_sc) if i >= 0]
    if fusion == N.FUSION_RANKED:
        fused = bm25.ranked_fusion([(wd, [d for d, _ in dense]), (ws, [d for d, _ in sparse])], k)
    else:
        fused = bm25.relative_score_fusion([(wd, dense), (ws, sparse)], k)
    cos = dict(dense) if wd > 0.0 else {}
    ids = np.full(k, -1, np.int64)
    sc = np.full(k, -np.inf)
    cs = np.full(k, np.nan, np.float32)
    for j, (d, s) in enumerate(fused):
        ids[j], sc[j] = d, s
        if d in cos:
            cs[j] = cos[d]
    return ids, sc, cs


def assert_row(got, want, ctx):
    gi, gs, gc = got
    wi, ws, wc = want
    assert np.array_equal(gi, wi), (ctx, gi[:8], wi[:8])
    assert np.array_equal(gs.view(np.int64), ws.view(np.int64)), (ctx, gs[:4], ws[:4])
    assert np.array_equal(np.isnan(gc), np.isnan(wc)), ctx
    ok = ~np.isnan(wc)
    assert np.array_equal(gc[ok].view(np.int32), wc[ok].view(np.int32)), ctx


def c_hybrid_search(ix, kw, qv, fetch, qt, qo, wd, ws=None, fusion=N.FUSION_RANKED, k_out=None, q_user=None, q_org=None):
    """engine.hybrid_search's single-shard call made through aur_hybrid_search itself (engine.hybrid_search takes
    aur_hybrid_search_multi with n = 1); the same arguments and return shape."""
    import ctypes as C

    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)   # noqa: E731
    q = ix._rows_buffer(qv)
    nq = q.shape[0]
    k_out = 2 * int(fetch) if k_out is None else int(k_out)
    wd = np.ascontiguousarray(np.broadcast_to(np.asarray(wd, dtype=np.float64), (nq,)))
    ws = 1.0 - wd if ws is None else np.ascontiguousarray(np.broadcast_to(np.asarray(ws, dtype=np.float64), (nq,)))
    qt = np.ascontiguousarray(qt, dtype=np.int32) if len(qt) else np.zeros(1, np.int32)
    qo = np.ascontiguousarray(qo, dtype=np.int64)
    u = None if q_user is None else np.ascontiguousarray(q_user, dtype=np.int32)
    o = None if q_org is None else np.ascontiguousarray(q_org, dtype=np.int32)
    scores, ids = np.empty((nq, k_out), np.float64), np.empty((nq, k_out), np.int64)
    cosine, snaps = np.empty((nq, k_out), np.float32), np.full(2, -1, np.int64)
    N.check(N.load().aur_hybrid_search(ix._h, kw._h, p(q), nq, int(fetch), p(qt), p(qo), p(u), p(o), p(wd), p(ws),
                                       int(fusion), k_out, p(scores), p(ids), p(cosine), p(snaps)))
    return ids, scores, cosine, (int(snaps[0]), int(snaps[1]))


def assert_same(a, b):
    """Two hybrid answers identical bit for bit, snapshots included."""
    for x, y in zip(a[:3], b[:3]):
        assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
    assert a[3] == b[3]


def weights(nq, shift=0):
    wd = np.array([max(0.0, ALPHAS[(q + shift) % len(ALPHAS)]) for q in range(nq)])
    return wd, 1.0 - wd


class Corpus2:
    """A bf16 vector shard and a keyword store holding the same ids and tenant codes."""

    def __init__(self, n, seed, vecs=None, docs=None, user=None, org=None):
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.vecs = rng.standard_normal((n, DIM)).astype(np.float32) if vecs is None else vecs
        t, f, off = zipf_docs(rng, n, vocab=3000) if docs is None else docs
        self.ids = rng.permutation(n).astype(np.int64) * 5 + 2
        self.user = rng.integers(0, 40, n).astype(np.int32) if user is None else user
        self.org = np.where(rng.random(n) < 0.4, rng.integers(0, 6, n), -1).astype(np.int32) if org is None else org
        self.ix = Index(DIM, max(n, 1) * 2)
        self.kw = KeywordIndex(max(n, 1) * 2)
        if n:
            self.ix.add(self.vecs, self.ids, self.user, self.org)
            self.kw.add(self.ids, t, f, off, self.user, self.org)

    def legs(self, qv, qt, qo, fetch, q_user, q_org):
        d_ids, d_sc = self.ix.search(qv, fetch, q_user, q_org)
        s_ids, s_sc, _ = self.kw.search(qt, qo, fetch, q_user, q_org)
        return d_ids, d_sc, s_ids, s_sc

    def check(self, qv, qt, qo, fetch, k_out, q_user=None, q_org=None, fusion=N.FUSION_RANKED, wd=None, ws=None):
        nq = qv.shape[0]
        if wd is None:
            wd, ws = weights(nq)
        got = hybrid_search(self.ix, self.kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
        assert_same(c_hybrid_search(self.ix, self.kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org), got)
        d_ids, d_sc, s_ids, s_sc = self.legs(qv, qt, qo, fetch, q_user, q_org)
        for q in range(nq):
            want = host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], wd[q], ws[q], fusion, k_out)
            assert_row((got[0][q], got[1][q], got[2][q]), want, (q, fetch, k_out, fusion))
        return got


@pytest.fixture(scope="module")
def corpus():
    return Corpus2(30_000, seed=1)


def _queries(c, nq, seed):
    rng = np.random.default_rng(seed)
    qv = rng.standard_normal((nq, DIM)).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=3000)
    return qv, qt, qo, rng


def _scopes(mode, nq, rng):
    if mode == "none":
        return None, None
    if mode == "one":
        return np.full(nq, 7, np.int32), np.full(nq, 3, np.int32)
    return rng.integers(0, 8, nq).astype(np.int32), rng.integers(-1, 3, nq).astype(np.int32)    # <= 32 scopes


@pytest.mark.parametrize("scope", ["none", "one", "mixed"])
@pytest.mark.parametrize("fetch", [1, 5, 128])
@pytest.mark.parametrize("nq", [1, 2, 255, 256, 257, 1100])
def test_bit_exact_against_the_separate_calls(corpus, nq, fetch, scope):
    """Both fusions, k_out in {1, fetch, 2 fetch}, alpha cycling over {0, 0.3, 0.5, 0.999} across the queries: the fused
    lists equal host fusion of aur_search_ex + aur_kw_search, bit for bit; a shorter k_out is a prefix of the longest."""
    qv, qt, qo, rng = _queries(corpus, nq, seed=nq * 7 + fetch)
    q_user, q_org = _scopes(scope, nq, rng)
    if q_user is not None and scope == "mixed":
        assert len(set(zip(q_user.tolist(), q_org.tolist()))) <= 32
    wd, ws = weights(nq, shift=nq)
    for fusion in FUSIONS:
        full = corpus.check(qv, qt, qo, fetch, 2 * fetch, q_user, q_org, fusion, wd, ws)
        for k_out in sorted({1, fetch}):
            ids, sc, cs, snaps = hybrid_search(corpus.ix, corpus.kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
            assert np.array_equal(ids, full[0][:, :k_out])
            assert np.array_equal(sc.view(np.int64), full[1][:, :k_out].view(np.int64))
            assert np.array_equal(cs.view(np.int32), full[2][:, :k_out].view(np.int32))
            assert snaps == (corpus.ix.stats()["rows"], corpus.kw.stats()["docs"])


def test_stats_of_both_legs(corpus):
    qv, qt, qo, _ = _queries(corpus, 64, seed=3)
    hybrid_search(corpus.ix, corpus.kw, qv, 32, qt, qo, 0.5)
    s, k = corpus.ix.stats(), corpus.kw.stats()
    assert s["last_kernel"] in (N.KERNEL_TC1, N.KERNEL_TC2, N.KERNEL_SIMT) and s["last_launches"] >= 2
    assert k["last_launches"] >= 2 and k["last_ms"] > 0


def test_adversarial_ties_empty_tenant_no_match_equal_scores():
    """300 copies of one document (same vector, same text) among others: every leg's scores tie, fused scores tie and are
    cut by id; a tenant with no rows gives padding only; a query without keyword matches is the dense leg alone;
    alpha 0 lists no dense-only id and no cosine."""
    rng = np.random.default_rng(5)
    n_dup, n_other = 300, 2000
    vecs = rng.standard_normal((n_dup + n_other, DIM)).astype(np.float32)
    vecs[:n_dup] = vecs[0]
    t, f, off = zipf_docs(rng, n_other, vocab=3000)
    dup_t, dup_f = np.array([3001, 3002], np.int32), np.array([2, 1], np.int32)
    terms = np.concatenate([np.tile(dup_t, n_dup), t])
    tfs = np.concatenate([np.tile(dup_f, n_dup), f])
    offs = np.concatenate([np.arange(0, 2 * n_dup + 1, 2), 2 * n_dup + off[1:]]).astype(np.int64)
    user = np.zeros(n_dup + n_other, np.int32)
    c = Corpus2(n_dup + n_other, seed=6, vecs=vecs, docs=(terms, tfs, offs), user=user,
                org=np.full(n_dup + n_other, -1, np.int32))
    dup_ids = set(c.ids[:n_dup].tolist())
    qv = np.repeat(vecs[:1], 4, axis=0)
    qt = np.array([3001, 3002, 3001, 99_999, 3002], np.int32)
    qo = np.array([0, 2, 3, 4, 5], np.int64)               # query 2: an unknown word only -> no keyword match
    for fusion in FUSIONS:
        for alpha in ALPHAS:
            wd, ws = np.full(4, alpha), np.full(4, 1.0 - alpha)
            ids, sc, cs, _ = c.check(qv, qt, qo, 128, 256, fusion=fusion, wd=wd, ws=ws)
            top = ids[0][ids[0] >= 0]
            assert set(top[:128].tolist()) <= dup_ids
            assert (np.diff(top[:128]) > 0).all()          # one tie group, lowest ids first
            if alpha == 0.0:
                assert np.isnan(cs).all()
                assert set(ids[0][ids[0] >= 0].tolist()) <= dup_ids   # dense-only ids are absent
            if fusion == N.FUSION_RELATIVE_SCORE and alpha > 0:
                assert (sc[0][:128] == alpha + (1.0 - alpha)).all()   # both legs' lists are all-equal: weight each
            if alpha > 0:
                assert (ids[2] >= 0).sum() == 128 and not np.isnan(cs[2][:128]).any()
        # a tenant with no rows: padding only
        ids, sc, cs, _ = c.check(qv, qt, qo, 16, 32, np.full(4, 55, np.int32), None, fusion)
        assert (ids == -1).all() and np.isneginf(sc).all() and np.isnan(cs).all()


def test_argument_errors(corpus):
    qv, qt, qo, _ = _queries(corpus, 2, seed=9)

    def code(**kw):
        args = dict(fetch=8, w=np.array([0.5, 0.5]), fusion=N.FUSION_RANKED, k_out=16, ix=corpus.ix, kw=corpus.kw)
        args.update(kw)
        codes = []
        for search in (hybrid_search, c_hybrid_search):   # aur_hybrid_search_multi with n = 1, aur_hybrid_search
            with pytest.raises(N.AuroraError) as e:
                search(args["ix"], args["kw"], qv, args["fetch"], qt, qo, args["w"], None, args["fusion"], args["k_out"])
            codes.append(e.value.code)
        assert codes[0] == codes[1], codes
        return codes[0]

    assert code(fetch=129, k_out=1) == N.AUR_ERR_UNSUPPORTED
    assert code(fetch=0, k_out=1) == N.AUR_ERR_INVALID
    assert code(k_out=17) == N.AUR_ERR_INVALID
    assert code(k_out=0) == N.AUR_ERR_INVALID
    assert code(fusion=2) == N.AUR_ERR_INVALID
    assert code(w=np.array([0.5, np.nan])) == N.AUR_ERR_INVALID
    assert code(w=np.array([np.inf, 0.5])) == N.AUR_ERR_INVALID
    f32 = Index(DIM, 64, dtype="f32")
    f32.add(qv, np.array([1, 2], np.int64))
    assert code(ix=f32) == N.AUR_ERR_UNSUPPORTED
    if N.load().aur_device_count() > 1:
        other = KeywordIndex(64, device=1)
        assert code(kw=other) == N.AUR_ERR_INVALID
    corpus.check(qv, qt, qo, 8, 16)                        # the handles still work


def test_concurrent_writer_and_readers():
    """One writer appends documents to both stores and removes earlier ones from both; three readers run fused
    searches.  Each answer equals host fusion of the oracle legs (oracle.cosine_topk, oracle/bm25_topk.py) over the two
    prefixes the call reports.  Removed documents point away from every query, so they never reach the dense top-k and
    only the keyword statistics see the removes: the keyword leg answers either before or after the remove that follows
    its prefix."""
    from oracle.bm25_topk import Corpus, bm25_topk
    from oracle.cosine_topk import bf16_bits_to_f32, cosine_topk

    rng = np.random.default_rng(21)
    steps, per, gone_per = 16, 1500, 40
    u = rng.standard_normal(DIM).astype(np.float32)
    nq, fetch, k_out = 6, 16, 32
    qv = (u + 0.3 * rng.standard_normal((nq, DIM))).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=800)
    t, f, off = zipf_docs(rng, steps * per, vocab=800)
    vecs = rng.standard_normal((steps * per, DIM)).astype(np.float32)
    away = np.zeros(steps * per, bool)
    for s in range(steps):
        away[s * per:s * per + gone_per] = True
    vecs[away] = -u + 0.01 * rng.standard_normal((int(away.sum()), DIM)).astype(np.float32)
    ids = np.arange(steps * per, dtype=np.int64) * 3 + 1
    ix, kw = Index(DIM, steps * per), KeywordIndex(steps * per)
    removed = [set()]                                      # removed ids after step s's remove
    answers, errors = [], []
    done = threading.Event()

    def writer():
        try:
            for s in range(steps):
                sl = slice(s * per, (s + 1) * per)
                ix.add(vecs[sl], ids[sl])
                kw.add(ids[sl], t[off[s * per]:off[(s + 1) * per]], f[off[s * per]:off[(s + 1) * per]],
                       off[s * per:(s + 1) * per + 1] - off[s * per])
                gone = ids[(s - 1) * per:(s - 1) * per + gone_per] if s else ids[:0]
                ix.remove(gone)
                kw.remove(gone)
                removed.append(removed[-1] | set(gone.tolist()))
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader(r):
        i = 0
        while not done.is_set():
            fusion = FUSIONS[(i + r) % 2]
            search = (hybrid_search, c_hybrid_search)[(i // 2 + r) % 2]   # both entry points under the writer
            answers.append((fusion, search(ix, kw, qv, fetch, qt, qo, 0.5, None, fusion, k_out)))
            i += 1

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader, args=(r,)) for r in range(3)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors
    snaps = sorted({a[1][3] for a in answers})
    assert len(snaps) >= 2
    rows32 = bf16_bits_to_f32(ix.export()[0])
    wd, ws = np.full(nq, 0.5), np.full(nq, 0.5)
    for fusion, (g_ids, g_sc, g_cs, (rd, rk)) in answers[:: max(1, len(answers) // 16)]:
        if rd == 0 or rk == 0:
            continue
        d_ids, d_sc = cosine_topk(bf16_bits_to_f32(to_bf16_bits(qv)), rows32[:rd], fetch, ids=ids[:rd])
        step = rk // per - 1
        def agrees(rows):
            for q in range(nq):
                wi, ws_, wc = rows[q]
                if not np.array_equal(g_ids[q], wi) or not np.array_equal(np.isnan(g_cs[q]), np.isnan(wc)):
                    return False
                if fusion == N.FUSION_RANKED:                 # ranks only: bit for bit
                    if not np.array_equal(g_sc[q].view(np.int64), ws_.view(np.int64)):
                        return False
                # relative scores carry the cosines, which the oracle may round differently in the last fp32 bit; the
                # two keyword states differ far more (their N and df differ)
                elif not np.allclose(g_sc[q], ws_, rtol=1e-6, atol=0.0):
                    return False
                if not np.allclose(g_cs[q], wc, rtol=0, atol=1e-6, equal_nan=True):
                    return False
            return True

        matched = []
        for gone in (removed[step], removed[step + 1]):   # the keyword leg ran before or after the remove of its step
            live = np.array([int(d) not in gone for d in ids[:rk]])
            s_ids, s_sc = bm25_topk(Corpus(t, f, off, ids, live, n_rows=rk), qt, qo, fetch)
            matched.append(agrees([host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], 0.5, 0.5, fusion, k_out)
                                   for q in range(nq)]))
        assert any(matched), (rd, rk, fusion)


# ----------------------------------------------------------------------------- retriever
DOCS = [
    ("disk full on node-7 after log rotation failed", "u1", None),
    ("cpu spike on api pods; oom killer fired twice", "u1", "o1"),
    ("database latency timeout during failover", "u2", "o1"),
    ("disk pressure evictions, node-7 cordoned", "u2", None),
    ("timeout talking to the payment gateway", "u3", "o2"),
    ("oom kill loop in worker pods, memory limit 512Mi", "u1", None),
]
QUERIES = ["disk node-7", "oom pods memory", "timeout", "nothing matches this", "latency failover disk"]


def _fill(kb, n_rep=30):
    for rep in range(n_rep):
        for j, (text, u, o) in enumerate(DOCS):
            kb.insert(u, f"doc{j}", "f.md", [{"content": f"{text} #{rep % 7}", "chunk_index": rep}], org_id=o)
    for j in range(40):                                    # 40 more tenants: a batch over all of them has > 32 scopes
        kb.insert(f"t{j}", "tdoc", "t.md", [{"content": f"{DOCS[j % 6][0]} tenant {j}", "chunk_index": 0}])


def _shape(objs, exact=True):
    return [(o.uuid, o.metadata.score if exact else round(o.metadata.score, 12),
             None if o.metadata.distance is None else round(o.metadata.distance, 5)) for o in objs]


@pytest.fixture(scope="module")
def kbs():
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder, OracleIndex

    emb = HashEmbedder(64)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(bm25, "VECTORISE_FROM", 1 << 60)
        dev = R.KnowledgeBase(emb, capacity=4096)
        host = R.KnowledgeBase(emb, capacity=4096, index_factory=lambda d, c: OracleIndex(d, c))
        for kb in (dev, host):
            _fill(kb)
            kb.delete_where(lambda p: p.get("document_id") == "doc3" and p.get("chunk_index", 0) % 5 == 0)
    assert dev._hybrid_device and not host._hybrid_device
    return dev, host


def test_retriever_fuses_on_the_device_and_matches_the_host_path(kbs, monkeypatch):
    from aurora_b200.filters import HybridFusion

    dev, host = kbs
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    scopes = (("u1", None), ("u2", "o1"), ("zz", "o2"), ("nobody", None))
    cases = [(q, a, s, fu) for q in QUERIES for a in (0.0, 0.5, 0.999) for s in scopes + (None,)
             for fu in (HybridFusion.RANKED, HybridFusion.RELATIVE_SCORE)]

    def run_single(kb, q, a, s, fu):
        if s is None:
            return kb.query(q, 10, alpha=a, fusion=fu)
        return kb.query(q, 10, user_id=s[0], org_id=s[1], alpha=a, scoped=True, fusion=fu)

    reqs = [("u1", q, 6, a_, None) for q in QUERIES for a_ in (0.0, 0.5, None)] + \
           [("u2", q, 4, 0.3, "o1") for q in QUERIES] + [(None, "disk", 3, 0.5, "o2"), ("t3", "disk", 5, 0.5, None)]
    want_single = [run_single(host, *c) for c in cases]
    want_batch = host.query_batch(reqs)

    def boom(*a, **k):
        raise AssertionError("host fusion on the unfiltered CUDA path")

    monkeypatch.setattr(bm25, "ranked_fusion", boom)
    monkeypatch.setattr(bm25, "relative_score_fusion", boom)
    for c, want in zip(cases, want_single):
        exact = c[3] == HybridFusion.RANKED        # relative scores carry the cosines, which may differ in the last bit
        assert _shape(run_single(dev, *c), exact) == _shape(want, exact), c
    assert [_shape(x) for x in dev.query_batch(reqs)] == [_shape(x) for x in want_batch]


def test_retriever_filtered_and_many_scopes_keep_the_host_path(kbs, monkeypatch):
    from aurora_b200.filters import Filter, HybridFusion

    dev, host = kbs
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    flt = Filter.by_property("document_id").like("doc*") & Filter.by_property("user_id").equal("u1")
    calls = []
    real = bm25.ranked_fusion
    monkeypatch.setattr(bm25, "ranked_fusion", lambda *a, **k: calls.append(1) or real(*a, **k))
    for q in QUERIES:
        for alpha in (0.0, 0.5):
            assert _shape(dev.query(q, 10, filters=flt, alpha=alpha)) == _shape(host.query(q, 10, filters=flt, alpha=alpha))
            got = dev.query(q, 10, filters=flt, alpha=alpha, fusion=HybridFusion.RELATIVE_SCORE)
            want = host.query(q, 10, filters=flt, alpha=alpha, fusion=HybridFusion.RELATIVE_SCORE)
            assert _shape(got, False) == _shape(want, False)
    n = len(calls)
    assert n > 0
    reqs = [(f"t{j}", QUERIES[j % 5], 5, 0.5, None) for j in range(40)]
    assert [_shape(x) for x in dev.query_batch(reqs)] == [_shape(x) for x in host.query_batch(reqs)]
    assert len(calls) == n + 2 * 40                        # 40 scopes > 32: fused on the host, per request


def test_retriever_delete_after_the_fused_call_drops_out(monkeypatch):
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder

    kb = R.KnowledgeBase(HashEmbedder(64), capacity=1024)
    _fill(kb, 3)
    real = bm25.DeviceBM25.search_batch
    gone = []

    def search_then_delete(self, *a, **k):
        out = real(self, *a, **k)
        assert k.get("dense") is not None
        victim = out[0][0][0]
        gone.append(kb._id2key[victim])
        kb._delete_keys([gone[-1]])
        return out

    monkeypatch.setattr(bm25.DeviceBM25, "search_batch", search_then_delete)
    res = kb.query("disk node-7", 5, user_id="u1", alpha=0.5, scoped=True)
    assert res and all(o.uuid != gone[-1] for o in res)
    res = kb.query_batch([("u1", "oom pods", 5, 0.5, None), ("u2", "timeout", 5, 0.0, "o1")])
    assert res[0] and res[1] and all(o.uuid != gone[-1] for objs in res for o in objs)

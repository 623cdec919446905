"""The hybrid query over several shards and keyword stores in one device call (aur_hybrid_search_multi,
engine.hybrid_search over a MultiIndex + MultiKeywordIndex, the retriever's fused path over a MultiIndex).  Every fused
list is held bit for bit (ids, fp64 score bits, fp32 cosine bits, NaN positions) to host fusion (bm25.ranked_fusion /
relative_score_fusion) of MultiIndex.search + MultiKeywordIndex.search, whose per-shard lists the host merges.  The
shards share device 0; where the machine has several GPUs the same cases also run with shard s on GPU s % gpus."""

import ctypes as C
import itertools
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import Index, KeywordIndex, MultiIndex, MultiKeywordIndex, hybrid_search, to_bf16_bits
from tests.keyword_mirror import Mirror, zipf_docs, zipf_queries
from tests.test_gpu_hybrid import ALPHAS, FUSIONS, QUERIES, _fill, _scopes, _shape, assert_row, host_fuse, weights
from tests.test_gpu_keyword_multi import _rows, union_corpus

pytestmark = pytest.mark.gpu

DIM = 128


def _gpus():
    return N.load().aur_device_count()


@pytest.fixture(params=["device0", "per_gpu"])
def layout(request):
    if request.param == "per_gpu" and _gpus() < 2:
        pytest.skip("one shard per GPU needs two or more GPUs; this machine has fewer")
    return request.param


def _devices(n, layout):
    return [0] * n if layout == "device0" else [s % _gpus() for s in range(n)]


class Multi:
    """A MultiIndex and a MultiKeywordIndex on the same devices holding the same ids, texts and tenant codes."""

    def __init__(self, n, layout, capacity):
        devices = _devices(n, layout)
        self.n = n
        self.mi = MultiIndex(DIM, capacity, devices=devices)
        self.mk = MultiKeywordIndex(capacity, devices=devices)

    def add(self, vecs, ids, docs, user=None, org=None):
        self.mi.add(vecs, ids, user, org)
        self.mk.add(ids, *docs, user, org)

    def remove(self, ids):
        self.mi.remove(ids)
        self.mk.remove(ids)

    def check(self, qv, qt, qo, fetch, k_out, q_user=None, q_org=None, fusion=N.FUSION_RANKED, wd=None, ws=None):
        nq = qv.shape[0]
        if wd is None:
            wd, ws = weights(nq)
        got = hybrid_search(self.mi, self.mk, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
        d_ids, d_sc = self.mi.search(qv, fetch, q_user, q_org)
        s_ids, s_sc, _ = self.mk.search(qt, qo, fetch, q_user, q_org)
        for q in range(nq):
            want = host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], wd[q], ws[q], fusion, k_out)
            assert_row((got[0][q], got[1][q], got[2][q]), want, (self.n, q, fetch, k_out, fusion))
        return got

    def close(self):
        self.mi.close()
        self.mk.close()


def _filled(n, layout, n_docs, seed):
    rng = np.random.default_rng(seed)
    m = Multi(n, layout, max(n_docs, 1) * 2)
    vecs = rng.standard_normal((n_docs, DIM)).astype(np.float32)
    docs = zipf_docs(rng, n_docs, vocab=3000)
    ids = rng.permutation(n_docs).astype(np.int64) * 5 + 2
    user = rng.integers(0, 40, n_docs).astype(np.int32)
    org = np.where(rng.random(n_docs) < 0.4, rng.integers(0, 6, n_docs), -1).astype(np.int32)
    m.add(vecs, ids, docs, user, org)
    return m


_CORPORA = {}   # (n, layout) -> the grid's corpus, built once


def _multi(n, layout):
    key = (n, layout)
    if key not in _CORPORA:
        _CORPORA[key] = _filled(n, layout, 12_000, seed=n)
    return _CORPORA[key]


def _queries(nq, seed):
    rng = np.random.default_rng(seed)
    qv = rng.standard_normal((nq, DIM)).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=3000)
    return qv, qt, qo, rng


@pytest.mark.parametrize("scope", ["none", "one", "mixed"])
@pytest.mark.parametrize("fetch", [1, 5, 128])
@pytest.mark.parametrize("nq", [1, 2, 256, 257])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_bit_exact_against_the_host_merge_and_fusion(n, nq, fetch, scope, layout):
    """Both fusions, k_out in {1, fetch, 2 fetch}, alpha cycling over {0, 0.3, 0.5, 0.999} across the queries."""
    m = _multi(n, layout)
    qv, qt, qo, rng = _queries(nq, seed=nq * 7 + fetch + 100 * n)
    q_user, q_org = _scopes(scope, nq, rng)
    wd, ws = weights(nq, shift=nq + n)
    for fusion in FUSIONS:
        full = m.check(qv, qt, qo, fetch, 2 * fetch, q_user, q_org, fusion, wd, ws)
        assert full[3] == (m.mi.stats()["rows_per_shard"], [s["docs"] for s in m.mk.stats()["stores"]])
        for k_out in sorted({1, fetch}):
            ids, sc, cs, _ = hybrid_search(m.mi, m.mk, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
            assert np.array_equal(ids, full[0][:, :k_out])
            assert np.array_equal(sc.view(np.int64), full[1][:, :k_out].view(np.int64))
            assert np.array_equal(cs.view(np.int32), full[2][:, :k_out].view(np.int32))


def test_one_shard_equals_aur_hybrid_search(layout):
    """n = 1 is aur_hybrid_search on the same shard and store: identical arrays."""
    m = _multi(1, layout)
    ix, kw = m.mi.shards[0], m.mk.stores[0]
    qv, qt, qo, rng = _queries(300, seed=4)
    q_user, q_org = _scopes("mixed", 300, rng)
    wd, ws = weights(300)
    for fusion in FUSIONS:
        for fetch, k_out in ((1, 2), (16, 9), (128, 256)):
            a = hybrid_search(m.mi, m.mk, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
            b = hybrid_search(ix, kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, q_user, q_org)
            for x, y in zip(a[:3], b[:3]):
                assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
            assert a[3] == ([b[3][0]], [b[3][1]])


def _dup_corpus(n, layout, n_dup, n_other, seed, skew=False):
    """n_dup copies of one document (same vector, same text) among others.  skew: every copy on shard 0."""
    rng = np.random.default_rng(seed)
    vecs = rng.standard_normal((n_dup + n_other, DIM)).astype(np.float32)
    vecs[:n_dup] = vecs[0]
    t, f, off = zipf_docs(rng, n_other, vocab=3000)
    terms = np.concatenate([np.tile(np.array([3001, 3002], np.int32), n_dup), t])
    tfs = np.concatenate([np.tile(np.array([2, 1], np.int32), n_dup), f])
    offs = np.concatenate([np.arange(0, 2 * n_dup + 1, 2), 2 * n_dup + off[1:]]).astype(np.int64)
    ids = rng.permutation(n_dup + n_other).astype(np.int64) + 1       # spread over the shards
    if skew:
        ids[:n_dup] = np.arange(n_dup, dtype=np.int64) * n * 7 + 7 * n      # all = 0 mod n
        ids[n_dup:] = np.arange(n_other, dtype=np.int64) * n + 1 + (np.arange(n_other) % (n - 1))   # never 0 mod n
    m = Multi(n, layout, (n_dup + n_other) * 2)
    m.add(vecs, ids, (terms, tfs, offs))
    return m, vecs, set(ids[:n_dup].tolist())


@pytest.mark.parametrize("n", [2, 3, 8])
def test_tie_groups_across_shards_are_cut_by_id(n, layout):
    """300 copies spread over the shards: equal fp32 cosines and equal BM25 scores whose group the fetch cut of 128
    falls inside; then the same copies all on shard 0, which holds each leg's whole top-fetch."""
    for skew in (False, True):
        m, vecs, dup_ids = _dup_corpus(n, layout, 300, 2000, seed=5 + n, skew=skew)
        qv = np.repeat(vecs[:1], 4, axis=0)
        qt = np.array([3001, 3002, 3001, 99_999, 3002], np.int32)
        qo = np.array([0, 2, 3, 4, 5], np.int64)           # query 2: an unknown word only -> no keyword match
        for fusion in FUSIONS:
            for alpha in ALPHAS:
                wd, ws = np.full(4, alpha), np.full(4, 1.0 - alpha)
                ids, sc, cs, _ = m.check(qv, qt, qo, 128, 256, fusion=fusion, wd=wd, ws=ws)
                top = ids[0][ids[0] >= 0][:128]
                assert set(top.tolist()) <= dup_ids and (np.diff(top) > 0).all()
                assert min(dup_ids) == top[0]
            m.check(qv, qt, qo, 5, 10, fusion=fusion)
        m.close()


def test_equal_cosines_with_descending_ids_merge_like_the_host(layout):
    """Rows whose fp64 cosines differ below fp32 resolution: a shard lists them by fp64 score, so its equal fp32
    cosines come with descending ids, and the host merge interleaves the shards' lists head by head."""
    n = 3
    rng = np.random.default_rng(8)
    k_small = np.arange(13, 40)                            # cos = 1 / sqrt(1 + 2^-2k): distinct in fp64, 1.0 in fp32
    m_rows = len(k_small) + 9
    vecs = np.zeros((m_rows, DIM), np.float32)
    vecs[:, 0] = 1.0
    for j, k in enumerate(k_small):
        vecs[j, 1 + j % (DIM - 1)] = 2.0 ** -int(k)
    # ids descend as the fp64 cosine rises within every shard; the last 9 rows are exact copies of e0 (cosine 1.0)
    ids = np.concatenate([np.arange(len(k_small), dtype=np.int64)[::-1] * 2 + 10,
                          rng.permutation(9).astype(np.int64) * 2 + 11])   # odd: apart from the even ids
    others = rng.standard_normal((3000, DIM)).astype(np.float32)
    all_vecs = np.concatenate([vecs, others])
    all_ids = np.concatenate([ids, np.arange(3000, dtype=np.int64) + 10_000])
    docs = zipf_docs(rng, len(all_ids), vocab=500)
    m = Multi(n, layout, 8000)
    m.add(all_vecs, all_ids, docs)
    q = np.zeros((2, DIM), np.float32)
    q[:, 0] = 1.0
    qt, qo = zipf_queries(rng, 2, vocab=500)
    d_ids, d_sc = m.mi.search(q, 40)
    assert (d_sc[0][:m_rows] == np.float32(1.0)).all()
    for fusion in FUSIONS:
        for fetch in (5, 20, 36, 40):
            m.check(q, qt, qo, fetch, 2 * fetch, fusion=fusion, wd=np.full(2, 0.7), ws=np.full(2, 0.3))
    m.close()


def test_empty_shards_tombstones_empty_tenants_and_no_keyword_match(layout):
    n = 3
    rng = np.random.default_rng(12)
    n_docs = 3000
    vecs = rng.standard_normal((n_docs, DIM)).astype(np.float32)
    docs = zipf_docs(rng, n_docs, vocab=3000)
    ids = np.arange(n_docs, dtype=np.int64) * 3          # every id = 0 mod 3: shards 1 and 2 stay empty
    m = Multi(n, layout, n * (n_docs + 1000))             # shard 0 takes every row
    m.add(vecs, ids, docs, np.zeros(n_docs, np.int32))
    qv, qt, qo, _ = _queries(6, seed=13)
    qt = np.concatenate([qt[:qo[3]], np.array([99_999], np.int32)])   # queries 3..5: an unknown word / nothing
    qo = np.concatenate([qo[:4], np.full(3, qo[3] + 1)]).astype(np.int64)
    for fusion in FUSIONS:
        m.check(qv, qt, qo, 32, 64, fusion=fusion)
        m.check(qv, qt, qo, 8, 16, np.full(6, 55, np.int32), None, fusion)   # a tenant with no rows
        ids, sc, cs, _ = hybrid_search(m.mi, m.mk, qv, 8, qt, qo, 0.5, None, fusion, 16, np.full(6, 55, np.int32))
        assert (ids == -1).all() and np.isneginf(sc).all() and np.isnan(cs).all()
    # shard 1 receives rows and then loses them all: a shard of tombstones only
    more = np.arange(500, dtype=np.int64) * 3 + 1
    docs2 = zipf_docs(rng, 500, vocab=3000)
    m.add(rng.standard_normal((500, DIM)).astype(np.float32), more, docs2, np.zeros(500, np.int32))
    m.remove(more)
    for fusion in FUSIONS:
        got = m.check(qv, qt, qo, 32, 64, fusion=fusion)
        assert got[3] == (m.mi.stats()["rows_per_shard"], [st["docs"] for st in m.mk.stats()["stores"]])
        assert not np.isin(got[0], more).any()
    m.close()


def test_argument_errors(layout):
    n = 3
    m = _filled(n, layout, 600, seed=30)
    qv, qt, qo, _ = _queries(2, seed=9)
    lib = N.load()
    q = to_bf16_bits(qv)
    wd = ws = np.full(2, 0.5)
    out_s, out_i, out_c = np.empty(32), np.empty(32, np.int64), np.empty(32, np.float32)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)            # noqa: E731

    def call(shards, stores, n_):
        a = (C.c_void_p * max(len(shards), 1))(*[getattr(s, "_h", C.c_void_p()).value if s is not None else None for s in shards])
        b = (C.c_void_p * max(len(stores), 1))(*[getattr(s, "_h", C.c_void_p()).value if s is not None else None for s in stores])
        return lib.aur_hybrid_search_multi(a, b, n_, vp(q), 2, 8, vp(qt), vp(qo), None, None, vp(wd), vp(ws),
                                           N.FUSION_RANKED, 16, vp(out_s), vp(out_i), vp(out_c), None)

    sh, st = m.mi.shards, m.mk.stores
    assert call(sh, st, 0) == N.AUR_ERR_INVALID
    assert call(sh * 22, st * 22, 65) == N.AUR_ERR_INVALID
    assert call([sh[0], None, sh[2]], st, 3) == N.AUR_ERR_INVALID
    assert call(sh, [st[0], st[1], None], 3) == N.AUR_ERR_INVALID
    assert call([sh[0], sh[1], sh[0]], st, 3) == N.AUR_ERR_INVALID
    assert call(sh, [st[0], st[1], st[1]], 3) == N.AUR_ERR_INVALID
    f32 = Index(DIM, 64, dtype="f32")
    f32.add(qv, np.array([1, 2], np.int64))
    assert call([sh[0], f32, sh[2]], st, 3) == N.AUR_ERR_UNSUPPORTED
    f32_multi = MultiIndex(DIM, 64, devices=_devices(n, layout), dtype="f32")
    with pytest.raises(TypeError):
        hybrid_search(f32_multi, m.mk, qv, 8, qt, qo, 0.5)
    m.check(qv, qt, qo, 8, 16)                             # the handles still work
    f32_multi.close()
    m.close()


def test_store_on_another_device_than_its_shard_is_refused():
    if _gpus() < 2:
        pytest.skip("a store on another device than its shard needs two or more GPUs; this machine has fewer")
    ix, kw = Index(DIM, 64, device=0), KeywordIndex(64, device=1)
    qv, qt, qo, _ = _queries(2, seed=9)
    with pytest.raises(N.AuroraError) as e:
        hybrid_search(MultiIndex(DIM, 64, devices=[0], _shards=[ix]), MultiKeywordIndex(64, devices=[0], store_factory=lambda c, p, d: kw),
                      qv, 8, qt, qo, 0.5)
    assert e.value.code == N.AUR_ERR_INVALID


def test_writer_appending_and_removing_under_three_readers(layout):
    """One writer appends documents to every shard and store and removes earlier ones; three readers run fused
    searches.  Each answer equals host fusion of the oracles over the 2n prefixes it reports.  Removed documents point
    away from every query, so they never reach the dense top-k; each keyword store answered either before or after the
    remove that follows its prefix."""
    from oracle.cosine_topk import bf16_bits_to_f32, cosine_topk
    from oracle.bm25_topk import bm25_topk

    n = 3
    rng = np.random.default_rng(21)
    steps, per, gone_per = 12, 900, 30
    u = rng.standard_normal(DIM).astype(np.float32)
    nq, fetch, k_out = 5, 16, 32
    qv = (u + 0.3 * rng.standard_normal((nq, DIM))).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=800)
    t, f, off = zipf_docs(rng, steps * per, vocab=800)
    vecs = rng.standard_normal((steps * per, DIM)).astype(np.float32)
    away = np.zeros(steps * per, bool)
    for s in range(steps):
        away[s * per:s * per + gone_per] = True
    vecs[away] = -u + 0.01 * rng.standard_normal((int(away.sum()), DIM)).astype(np.float32)
    ids = np.arange(steps * per, dtype=np.int64) * 7 + 1
    m = Multi(n, layout, steps * per)
    removed = [set()]
    answers, errors = [], []
    done = threading.Event()

    def writer():
        try:
            for s in range(steps):
                sl = np.arange(s * per, (s + 1) * per)
                m.add(vecs[sl], ids[sl], _rows(t, f, off, sl))
                gone = ids[(s - 1) * per:(s - 1) * per + gone_per] if s else ids[:0]
                m.remove(gone)
                removed.append(removed[-1] | set(gone.tolist()))
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader(r):
        i = 0
        try:
            while not done.is_set():
                fusion = FUSIONS[(i + r) % 2]
                answers.append((fusion, hybrid_search(m.mi, m.mk, qv, fetch, qt, qo, 0.5, None, fusion, k_out)))
                i += 1
        except Exception as e:   # pragma: no cover
            errors.append(e)

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader, args=(r,)) for r in range(3)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors
    assert len({(tuple(a[1][3][0]), tuple(a[1][3][1])) for a in answers}) >= 2
    # every shard's and store's rows in append order (the writer appended in global order, each row to id mod n)
    owner = [np.nonzero(ids % n == s)[0] for s in range(n)]
    q32 = bf16_bits_to_f32(to_bf16_bits(qv))
    v32 = bf16_bits_to_f32(to_bf16_bits(vecs))
    checked = 0
    for fusion, (g_ids, g_sc, g_cs, (rd, rk)) in answers[:: max(1, len(answers) // 10)]:
        if min(rd) == 0 or min(rk) == 0:
            continue
        rows = np.concatenate([owner[s][:rd[s]] for s in range(n)])
        d_ids, d_sc = cosine_topk(q32, v32[rows], fetch, ids=ids[rows])
        steps_of = [int(owner[s][rk[s] - 1]) // per for s in range(n)]   # the step whose append each store reported
        matched = False
        for after in itertools.product((0, 1), repeat=n):             # each store: before / after its step's remove
            parts = []
            for s in range(n):
                mir = Mirror()
                sel = owner[s][:rk[s]]
                mir.add(ids[sel], *_rows(t, f, off, sel))
                mir.remove(list(removed[steps_of[s] + after[s]]))
                parts.append(mir)
            s_ids, s_sc = bm25_topk(union_corpus(parts, [len(p.ids) for p in parts]), qt, qo, fetch)
            ok = True
            for q in range(nq):
                wi, ws_, wc = host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], 0.5, 0.5, fusion, k_out)
                if not np.array_equal(g_ids[q], wi) or not np.array_equal(np.isnan(g_cs[q]), np.isnan(wc)):
                    ok = False
                elif fusion == N.FUSION_RANKED and not np.array_equal(g_sc[q].view(np.int64), ws_.view(np.int64)):
                    ok = False
                # relative scores carry the cosines, which the oracle may round differently in the last fp32 bit
                elif not np.allclose(g_sc[q], ws_, rtol=1e-6, atol=0.0) or \
                        not np.allclose(g_cs[q], wc, rtol=0, atol=1e-6, equal_nan=True):
                    ok = False
                if not ok:
                    break
            if ok:
                matched = True
                break
        assert matched, (rd, rk, fusion)
        checked += 1
    assert checked >= 2
    m.close()


# ----------------------------------------------------------------------------- retriever
@pytest.mark.parametrize("spread", ["device0", "all_gpus"])
def test_retriever_over_a_multi_index_fuses_on_the_device(spread, monkeypatch):
    from aurora_b200 import retriever as R
    from aurora_b200.filters import HybridFusion
    from tests.doubles import HashEmbedder

    if spread == "all_gpus" and _gpus() < 2:
        pytest.skip("a knowledge base over several GPUs needs two or more GPUs; this machine has fewer")
    devices = [0, 0, 0] if spread == "device0" else list(range(_gpus()))
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    kb = R.KnowledgeBase(HashEmbedder(64), capacity=4096, index_factory=lambda d, c: MultiIndex(d, c, devices=devices))
    _fill(kb)
    kb.delete_where(lambda p: p.get("document_id") == "doc3" and p.get("chunk_index", 0) % 5 == 0)
    assert kb._hybrid_device
    scopes = (("u1", None), ("u2", "o1"), ("zz", "o2"), ("nobody", None))
    cases = [(q, a, s, fu) for q in QUERIES for a in (0.0, 0.5, 0.999) for s in scopes + (None,)
             for fu in (HybridFusion.RANKED, HybridFusion.RELATIVE_SCORE)]
    reqs = [("u1", q, 6, a_, None) for q in QUERIES for a_ in (0.0, 0.5, None)] + \
           [("u2", q, 4, 0.3, "o1") for q in QUERIES] + [(None, "disk", 3, 0.5, "o2"), ("t3", "disk", 5, 0.5, None)]

    def run_single(q, a, s, fu):
        if s is None:
            return kb.query(q, 10, alpha=a, fusion=fu)
        return kb.query(q, 10, user_id=s[0], org_id=s[1], alpha=a, scoped=True, fusion=fu)

    kb._hybrid_device = False                              # the same store, fused on the host
    want_single = [_shape(run_single(*c)) for c in cases]
    want_batch = [_shape(x) for x in kb.query_batch(reqs)]
    kb._hybrid_device = True

    def boom(*a, **k):
        raise AssertionError("host fusion on the fused path")

    monkeypatch.setattr(bm25, "ranked_fusion", boom)
    monkeypatch.setattr(bm25, "relative_score_fusion", boom)
    for c, want in zip(cases, want_single):
        assert _shape(run_single(*c)) == want, c
    assert [_shape(x) for x in kb.query_batch(reqs)] == want_batch

"""The filtered hybrid query in one device call (aur_hybrid_search_filtered, engine.hybrid_search with programs, the
retriever's filtered fused path).  Every fused list is held bit for bit (ids, fp64 score bits, fp32 cosine bits, NaN
positions) to host fusion (bm25.ranked_fusion / relative_score_fusion) of the separate calls: Index.search_filtered /
MultiIndex.search_filtered for the dense leg, KeywordIndex.search / MultiKeywordIndex.search with the allow-ids the
test computes in numpy from the codes it wrote and the live ids for the keyword leg."""

import ctypes as C
import os
import shutil
import tempfile
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import Index, KeywordIndex, MultiIndex, MultiKeywordIndex, _ptr, hybrid_search
from aurora_b200.filters import AttrColumn, Filter, compile_program, pack_programs
from oracle.bm25_topk import Corpus, bm25_topk
from oracle.cosine_topk import cosine_topk, round_to_bf16
from tests.gpu_exact import check_host_exact
from tests.keyword_mirror import zipf_docs, zipf_queries
from tests.test_gpu_hybrid import FUSIONS, assert_row, host_fuse, weights

pytestmark = pytest.mark.gpu

DIM = 128
F = Filter.by_property
EXPRS = [
    F("org_id").equal("o3") & F("document_id").like("discovery:*"),    # the prediscovery filter
    F("org_id").equal("o1"),
    F("org_id").equal("nobody"),                                       # matches nothing
    F("n").greater_than(-1),                                           # every row
    F("document_id").equal("discovery:17"),                            # one row
    (F("org_id").equal("o0") | F("org_id").equal("o2")) & F("n").less_than(40),
]


def _gpus():
    return N.load().aur_device_count()


def _props(rng, n):
    org = rng.integers(6, size=n)
    disc = rng.random(n) < 0.5
    return [{"org_id": f"o{o}", "document_id": (f"discovery:{i}" if d else f"doc:{i}"), "n": int(i % 97)}
            for i, (o, d) in enumerate(zip(org, disc))]


class Pair:
    """A vector index and a keyword store (one each, or a MultiIndex + MultiKeywordIndex over n) holding the same ids,
    texts, tenant codes and attribute columns, and the host's record of them."""

    def __init__(self, n, capacity, devices=None):
        self.n = n
        if n == 1 and devices is None:
            self.ix, self.kw = Index(DIM, capacity), KeywordIndex(capacity)
        else:
            devices = devices or [0] * n
            self.ix, self.kw = MultiIndex(DIM, capacity, devices=devices), MultiKeywordIndex(capacity, devices=devices)
        self.cols = {nm: AttrColumn(nm, 2 + i) for i, nm in enumerate(("org_id", "document_id", "n"))}
        self.props, self.user, self.org, self.live = {}, {}, {}, {}   # by id: properties with codes set, tenant, liveness
        self.oracle = None                      # (bf16-rounded vectors, ids, oracle Corpus) of a corpus never mutated

    def add(self, vecs, ids, docs, user, org, props=None):
        self.ix.add(vecs, ids, user, org)
        self.kw.add(ids, *docs, user, org)
        for j, i in enumerate(ids.tolist()):
            self.props[i], self.user[i], self.org[i], self.live[i] = {}, int(user[j]), int(org[j]), True
        if props is not None:
            self.set(ids, props)

    def set(self, ids, props, stores=("ix", "kw")):
        for c in self.cols.values():
            codes = np.array([c.code(p) for p in props], np.int32)
            for st in stores:
                getattr(self, st).set_attrs(c.col, ids, codes)
        for i, p in zip(ids.tolist(), props):
            if i in self.props:
                self.props[i] = p

    def remove(self, ids):
        self.ix.remove(ids)
        self.kw.remove(ids)
        for i in ids.tolist():
            self.live[i] = False

    def program(self, e):
        return compile_program(e, self.cols)

    def allowed(self, e=None, tenant=None):
        out = []
        for i, live in self.live.items():
            if not live:
                continue
            ok = e.matches(self.props[i]) if e is not None else True
            if tenant is not None:
                u, o = tenant
                ok = ok and (self.user[i] == u or (o >= 0 and self.org[i] == o))
            if ok:
                out.append(i)
        return np.array(sorted(out), np.int64)

    def check(self, qv, qt, qo, fetch, k_out, progs, allows, q_prog, fusion, wd, ws, max_list_rows=0, ctx=(), sample=None):
        """The fused call against host fusion of the separate calls; allows[p]: the ids program p admits.  sample: a query
        whose two separate legs are also held to the fp64 oracles (oracle.cosine_topk, oracle/bm25_topk.py) over the
        rows its program admits, so the chain fused call == host fusion of the legs == host fusion of the oracles."""
        got = hybrid_search(self.ix, self.kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, programs=progs, q_program=q_prog,
                            max_list_rows=max_list_rows)
        d_ids, d_sc = self.ix.search_filtered(qv, fetch, progs, q_prog, max_list_rows)[:2]
        s_ids = np.full((len(qv), fetch), -1, np.int64)
        s_sc = np.full((len(qv), fetch), -np.inf)
        for p in np.unique(q_prog):
            qs = np.nonzero(q_prog == p)[0]
            sub_t = [qt[qo[q]:qo[q + 1]] for q in qs]
            sub_o = np.concatenate([[0], np.cumsum([len(t) for t in sub_t])]).astype(np.int64)
            i_, s_, _ = self.kw.search(np.concatenate(sub_t) if len(sub_o) > 1 and sub_o[-1] else np.zeros(0, np.int32),
                                       sub_o, fetch, allow_ids=allows[p])
            s_ids[qs], s_sc[qs] = i_, s_
        for q in range(len(qv)):
            want = host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], wd[q], ws[q], fusion, k_out)
            assert_row((got[0][q], got[1][q], got[2][q]), want, ctx + (q,))
        if sample is not None and self.oracle is not None:
            rows32, ids, corpus = self.oracle
            q, allow = sample, allows[q_prog[sample]]
            check_host_exact((d_ids[q:q + 1], d_sc[q:q + 1]), round_to_bf16(qv[q:q + 1]), rows32, fetch, ids=ids,
                             live=np.isin(ids, allow))
            o_ids, o_sc = corpus.topk(qt[qo[q]:qo[q + 1]], fetch, allow_ids=allow)
            assert np.array_equal(s_ids[q], o_ids) and np.array_equal(s_sc[q].view(np.int64), o_sc.view(np.int64)), ctx
        return got

    def close(self):
        self.ix.close()
        self.kw.close()


def _filled(n, n_docs, seed, devices=None):
    rng = np.random.default_rng(seed)
    pr = Pair(n, n_docs * 2, devices)
    vecs = rng.standard_normal((n_docs, DIM)).astype(np.float32)
    ids = rng.permutation(n_docs).astype(np.int64) * 5 + 2
    user = rng.integers(0, 40, n_docs).astype(np.int32)
    org = np.where(rng.random(n_docs) < 0.4, rng.integers(0, 6, n_docs), -1).astype(np.int32)
    docs = zipf_docs(rng, n_docs, vocab=3000)
    pr.add(vecs, ids, docs, user, org, _props(rng, n_docs))
    pr.oracle = (round_to_bf16(vecs), ids, Corpus(*docs, ids, row_user=user, row_org=org))
    return pr


_CORPORA = {}


def _pair(n, per_gpu=False):
    key = (n, per_gpu)
    if key not in _CORPORA:
        _CORPORA[key] = _filled(n, 12_000, seed=n, devices=[s % _gpus() for s in range(n)] if per_gpu else None)
    return _CORPORA[key]


def _queries(nq, seed):
    rng = np.random.default_rng(seed)
    qv = rng.standard_normal((nq, DIM)).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=3000)
    return qv, qt, qo, rng


def _programs(pr, n_prog, nq, rng, shared):
    """n_prog programs cycling over EXPRS and tenant programs; every query on program 0 (shared) or on its own."""
    tenants = [(3, 2), (7, -1), (-2, 4), (11, 0)]
    memo = {}
    progs, allows = [], []
    for i in range(n_prog):
        if i % 7 == 6:
            t = tenants[(i // 7) % len(tenants)]
            progs.append(compile_program(None, {}, tenant=t))
            key = ("t", t)
            if key not in memo:
                memo[key] = pr.allowed(tenant=t)
        else:
            key = i % len(EXPRS)
            progs.append(pr.program(EXPRS[key]))
            if key not in memo:
                memo[key] = pr.allowed(EXPRS[key])
        allows.append(memo[key])
    q_prog = np.zeros(nq, np.int32) if shared else rng.integers(n_prog, size=nq).astype(np.int32)
    return progs, allows, q_prog


PROGRAM_SETS = [(1, True), (2, False), (33, False), (1024, False), (1024, True)]   # (programs, shared by every query)


@pytest.mark.parametrize("fetch", [1, 5, 128])
@pytest.mark.parametrize("nq", [1, 2, 255, 256, 257])
@pytest.mark.parametrize("n", [1, 2, 3])
def test_bit_exact_against_the_separate_calls(n, nq, fetch):
    """Both fusions, k_out in {1, fetch, 2 fetch}, alpha cycling over {0, 0.3, 0.5, 0.999} across the queries; the program
    set cycles with the case, so each n meets every one of PROGRAM_SETS."""
    n_prog, shared = PROGRAM_SETS[(nq + fetch + n) % len(PROGRAM_SETS)]
    pr = _pair(n)
    qv, qt, qo, rng = _queries(nq, seed=nq * 7 + fetch + 100 * n + n_prog)
    progs, allows, q_prog = _programs(pr, n_prog, nq, rng, shared)
    wd, ws = weights(nq, shift=nq + n)
    for fusion in FUSIONS:
        full = pr.check(qv, qt, qo, fetch, 2 * fetch, progs, allows, q_prog, fusion, wd, ws, ctx=(n, nq, fetch, fusion),
                        sample=int(rng.integers(nq)))
        for k_out in sorted({1, fetch}):
            ids, sc, cs, _ = hybrid_search(pr.ix, pr.kw, qv, fetch, qt, qo, wd, ws, fusion, k_out, programs=progs,
                                           q_program=q_prog)
            assert np.array_equal(ids, full[0][:, :k_out])
            assert np.array_equal(sc.view(np.int64), full[1][:, :k_out].view(np.int64))
            assert np.array_equal(cs.view(np.int32), full[2][:, :k_out].view(np.int32))


def test_shard_per_gpu():
    if _gpus() < 2:
        pytest.skip("one shard per GPU needs two or more GPUs; this machine has fewer")
    pr = _pair(3, per_gpu=True)
    qv, qt, qo, rng = _queries(64, seed=5)
    progs, allows, q_prog = _programs(pr, 33, 64, rng, False)
    wd, ws = weights(64)
    for fusion in FUSIONS:
        pr.check(qv, qt, qo, 32, 64, progs, allows, q_prog, fusion, wd, ws)


def test_one_shard_equals_the_multi_path():
    """n = 1 through a MultiIndex + MultiKeywordIndex and through the Index + KeywordIndex it wraps: identical arrays."""
    rng = np.random.default_rng(3)
    m = _filled(1, 5000, seed=11, devices=[0])
    ix, kw = m.ix.shards[0], m.kw.stores[0]
    qv, qt, qo, rng = _queries(300, seed=4)
    progs, _, q_prog = _programs(m, 40, 300, rng, False)
    wd, ws = weights(300)
    for fusion in FUSIONS:
        a = hybrid_search(m.ix, m.kw, qv, 16, qt, qo, wd, ws, fusion, 20, programs=progs, q_program=q_prog)
        b = hybrid_search(ix, kw, qv, 16, qt, qo, wd, ws, fusion, 20, programs=progs, q_program=q_prog)
        for x, y in zip(a[:3], b[:3]):
            assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
        assert a[3] == ([b[3][0]], [b[3][1]])
    m.close()


@pytest.mark.parametrize("n", [1, 2])
def test_list_path_and_masked_scan_agree(n):
    pr = _pair(n)
    qv, qt, qo, _ = _queries(20, seed=77)
    e = EXPRS[0]
    progs, allows = [pr.program(e)], [pr.allowed(e)]
    q_prog = np.zeros(20, np.int32)
    wd, ws = weights(20)
    shards = pr.ix.shards if n > 1 else [pr.ix]
    outs = []
    for mlr, want_list in ((0, False), (10**9, True)):
        outs.append(pr.check(qv, qt, qo, 32, 64, progs, allows, q_prog, N.FUSION_RANKED, wd, ws, max_list_rows=mlr))
        hybrid_search(pr.ix, pr.kw, qv, 32, qt, qo, wd, ws, N.FUSION_RANKED, 64, programs=progs, q_program=q_prog,
                      max_list_rows=mlr)
        for sh in shards:
            assert (sh.stats()["last_kernel"] == N.KERNEL_LIST) == want_list
    for x, y in zip(outs[0][:3], outs[1][:3]):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_tie_groups_cut_by_fetch():
    """300 copies of one document (same vector, same text) inside the filter: every leg ties, cut by id."""
    rng = np.random.default_rng(8)
    pr = Pair(2, 4000)
    base = rng.standard_normal(DIM).astype(np.float32)
    vecs = np.vstack([np.tile(base, (300, 1)), rng.standard_normal((700, DIM)).astype(np.float32)])
    t, f, o = zipf_docs(rng, 1, vocab=500, min_len=5)
    others = zipf_docs(rng, 700, vocab=500)
    docs = (np.concatenate([np.tile(t, 300), others[0]]), np.concatenate([np.tile(f, 300), others[1]]),
            np.concatenate([np.arange(301) * o[1], others[2][1:] + 300 * o[1]]).astype(np.int64))
    ids = rng.permutation(1000).astype(np.int64) * 3
    props = [{"org_id": "o1" if j < 300 or j % 2 else "o2", "document_id": f"discovery:{j}", "n": 1} for j in range(1000)]
    pr.add(vecs, ids, docs, np.zeros(1000, np.int32), np.full(1000, -1, np.int32), props)
    e = F("org_id").equal("o1")
    qv = np.tile(base, (3, 1))
    kt = min(3, len(t))
    qt = np.tile(t[:kt], 3).astype(np.int32)
    qo = np.arange(4, dtype=np.int64) * kt
    for fetch in (1, 5, 128):
        for fusion in FUSIONS:
            pr.check(qv, qt, qo, fetch, 2 * fetch, [pr.program(e)], [pr.allowed(e)], np.zeros(3, np.int32), fusion,
                     np.array([0.5, 0.3, 0.999]), np.array([0.5, 0.7, 0.001]))
    pr.close()


def test_store_columns_through_tombstones_upserts_compaction_and_capacity():
    rng = np.random.default_rng(12)
    cap, n0 = 3000, 2500
    pr = Pair(1, cap)
    vecs = rng.standard_normal((cap + 1200, DIM)).astype(np.float32)
    ids = rng.permutation(cap + 1200).astype(np.int64) * 7 + 1
    docs = zipf_docs(rng, cap + 1200, vocab=800)

    def sub(a, b):
        t, f, o = docs
        return t[o[a]:o[b]], f[o[a]:o[b]], (o[a:b + 1] - o[a]).astype(np.int64)

    props = _props(rng, cap + 1200)
    user = np.zeros(cap + 1200, np.int32)
    org = rng.integers(-1, 6, cap + 1200).astype(np.int32)
    pr.add(vecs[:n0], ids[:n0], sub(0, n0), user[:n0], org[:n0], props[:n0])
    qv, qt, qo, _ = _queries(12, seed=13)
    e = F("org_id").equal("o2") | F("document_id").like("discovery:1*")
    for c in pr.cols.values():                   # codes of values to come, so the program's bitmaps cover them
        for p in props:
            c.code(p)
    wd, ws = weights(12)

    def check():
        for mlr in (0, 10**9):
            pr.check(qv, qt, qo, 64, 64, [pr.program(e)], [pr.allowed(e)], np.zeros(12, np.int32), N.FUSION_RANKED, wd, ws,
                     max_list_rows=mlr)

    check()
    pr.set(np.array([10**9, 10**9 + 1], np.int64), [props[0], props[1]])   # unknown ids are ignored
    check()
    pr.remove(ids[:400])                                                     # tombstones
    check()
    up = ids[600:900]                                                        # upserts: the new rows start absent
    pr.add(vecs[n0:n0 + 300], up, sub(n0, n0 + 300), user[n0:n0 + 300], org[n0:n0 + 300])
    check()
    pr.set(up, props[n0:n0 + 300])
    check()
    assert pr.ix.compact() == 700 and pr.kw.compact() == 700                 # codes move with their rows
    check()
    a, b = n0 + 300, n0 + 1200                                               # refill to capacity (2100 + 900 rows):
    tail = ids[a:b]                                                          # the rows compaction freed start absent
    pr.add(vecs[a:b], tail, sub(a, b), user[a:b], org[a:b])
    check()
    assert pr.kw.stats()["docs"] == cap and pr.ix.stats()["rows"] == cap
    pr.set(tail, props[a:b])
    check()
    pr.close()


def _raw(shards, stores, qv, qt, qo, tok, off, n_prog, bm, qp, mlr=0, n=None, fetch=5, k_out=5):
    n = len(shards) if n is None else n
    hs = (C.c_void_p * max(len(shards), 1))(*[s._h.value if s is not None else None for s in shards])
    ks = (C.c_void_p * max(len(stores), 1))(*[s._h.value if s is not None else None for s in stores])
    q = np.ascontiguousarray(qv, np.float32)
    from aurora_b200.engine import to_bf16_bits
    qb = to_bf16_bits(q)
    nq = q.shape[0]
    wd, ws = np.full(nq, 0.5), np.full(nq, 0.5)
    scores = np.full((nq, k_out), 7.0)
    ids = np.full((nq, k_out), 77, np.int64)
    cos = np.full((nq, k_out), 3.0, np.float32)
    snaps = np.full(2 * max(n, 1), -9, np.int64)
    rc = N.load().aur_hybrid_search_filtered(hs, ks, n, _ptr(qb), nq, fetch, _ptr(qt), _ptr(qo), _ptr(tok), _ptr(off),
                                             int(n_prog), _ptr(bm), bm.shape[0], _ptr(qp), int(mlr), _ptr(wd), _ptr(ws),
                                             N.FUSION_RANKED, k_out, _ptr(scores), _ptr(ids), _ptr(cos), _ptr(snaps))
    untouched = (scores == 7.0).all() and (ids == 77).all() and (cos == 3.0).all() and (snaps == -9).all()
    return rc, untouched


def test_rejections_leave_the_outputs_untouched():
    rng = np.random.default_rng(2)
    pr = _filled(1, 500, seed=2)
    ix, kw = pr.ix, pr.kw
    qv, qt, qo, _ = _queries(3, seed=1)
    qt = np.ascontiguousarray(qt, np.int32)
    qp = np.zeros(3, np.int32)
    tok, off, bm = pack_programs([pr.program(F("org_id").equal("o1") | F("org_id").equal("o2"))])
    leaf, op = tok[0].copy(), tok[2].copy()
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, qp) == (N.AUR_OK, False)
    cases = {
        "underflow": np.array([leaf, op]),
        "two values left": np.array([leaf, leaf]),
        "column out of range": np.array([[0, 18, 0, 1]]),
        "column never set": np.array([[0, 9, 0, 1]]),
        "slice past the bitmap": np.array([[0, 2, 0, bm.shape[0] * 32 + 1]]),
        "unknown token": np.array([[7, 0, 0, 0]]),
        "33 leaves": np.array([leaf] + [leaf, op] * 32),
    }
    for name, tk in cases.items():
        tk = np.ascontiguousarray(tk, np.int32)
        assert _raw([ix], [kw], qv, qt, qo, tk, np.array([0, len(tk)], np.int32), 1, bm, qp) == (N.AUR_ERR_INVALID, True), name
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 0, bm, qp) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1025, bm, qp) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, np.array([0, 1, 0], np.int32)) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, np.array([0, -1, 0], np.int32)) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, qp, mlr=-1) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, qp, fetch=129, k_out=5) == (N.AUR_ERR_UNSUPPORTED, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, qp, fetch=5, k_out=11) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix], [kw], qv, qt, qo, tok, off, 1, bm, qp, n=0) == (N.AUR_ERR_INVALID, True)
    assert _raw([ix, ix], [kw, kw], qv, qt, qo, tok, off, 1, bm, qp) == (N.AUR_ERR_INVALID, True)
    assert _raw([None], [kw], qv, qt, qo, tok, off, 1, bm, qp) == (N.AUR_ERR_INVALID, True)
    # a column set on the shard but not on the store, and the other way round
    e9 = compile_program(F("x").equal(1), {"x": AttrColumn("x", 9)})
    t9, o9, b9 = pack_programs([e9])
    ix.set_attrs(9, np.array([2], np.int64), np.array([0], np.int32))
    assert _raw([ix], [kw], qv, qt, qo, t9, o9, 1, b9, qp) == (N.AUR_ERR_INVALID, True)
    ix2, kw2 = Index(DIM, 100), KeywordIndex(100)
    kw2.set_attrs(9, np.array([2], np.int64), np.array([0], np.int32))
    assert _raw([ix2], [kw2], qv, qt, qo, t9, o9, 1, b9, qp) == (N.AUR_ERR_INVALID, True)
    ix2.set_attrs(9, np.array([2], np.int64), np.array([0], np.int32))
    assert _raw([ix2], [kw2], qv, qt, qo, t9, o9, 1, b9, qp)[0] == N.AUR_OK
    ix2.close()
    kw2.close()
    with Index(DIM, 100, dtype="f32") as f32:
        f32.set_attrs(2, np.array([2], np.int64), np.array([0], np.int32))
        f32.set_attrs(3, np.array([2], np.int64), np.array([0], np.int32))
        f32.set_attrs(4, np.array([2], np.int64), np.array([0], np.int32))
        assert _raw([f32], [kw], qv, qt, qo, tok, off, 1, bm, qp) == (N.AUR_ERR_UNSUPPORTED, True)
    with pytest.raises(ValueError):
        hybrid_search(ix, kw, qv, 5, qt, qo, 0.5, programs=[pr.program(EXPRS[0])], q_user=np.zeros(3, np.int32))
    assert kw._lib.aur_kw_set_attrs(kw._h, 1, _ptr(np.array([2], np.int64)), _ptr(np.array([0], np.int32)), 1) == N.AUR_ERR_INVALID
    assert kw._lib.aur_kw_set_attrs(kw._h, 18, _ptr(np.array([2], np.int64)), _ptr(np.array([0], np.int32)), 1) == N.AUR_ERR_INVALID
    pr.close()


def test_search_filtered_into_page_locked_outputs():
    """aur_search_filtered, which now runs through the same filtered legs, still writes page-locked caller buffers
    straight from its re-rank kernel: the answer equals the one staged into pageable buffers, on both paths."""
    import torch

    pr = _pair(1)
    qv, _, _, _ = _queries(40, seed=61)
    q = pr.ix._rows_buffer(qv)
    tok, off, bm = pack_programs([pr.program(EXPRS[0])])
    qp = np.zeros(40, np.int32)
    for mlr in (0, 10 ** 9):
        want_i, want_s, _, _ = pr.ix.search_filtered(qv, 32, [pr.program(EXPRS[0])], max_list_rows=mlr)
        s_pin = torch.full((40, 32), 7.0, dtype=torch.float32, pin_memory=True)
        i_pin = torch.full((40, 32), 77, dtype=torch.int64, pin_memory=True)
        rc = pr.ix._lib.aur_search_filtered(pr.ix._h, _ptr(q), 40, 32, _ptr(tok), _ptr(off), 1, _ptr(bm), bm.shape[0],
                                            _ptr(qp), mlr, C.c_void_p(s_pin.data_ptr()), C.c_void_p(i_pin.data_ptr()),
                                            None, None)
        assert rc == N.AUR_OK
        assert np.array_equal(i_pin.numpy(), want_i) and np.array_equal(s_pin.numpy().view(np.uint32), want_s.view(np.uint32))


@pytest.mark.parametrize("n", [1, 2])
def test_concurrent_writer_and_readers(n):
    """One writer appends documents to both stores, sets attribute codes on both and removes earlier documents from
    both; three readers run filtered fused searches (two programs per batch, list path and masked scan alternating).
    Each answer equals host fusion of the oracle legs (oracle.cosine_topk, oracle/bm25_topk.py) over the prefixes it
    reports in snapshot_rows_out, per shard and per store.

    The programs are `kind != "hidden" AND tenant(org 1)` and `tenant(org 2)`.  The writer's code writes (new rows
    "visible", older rows "shown", removed rows "hidden") never change which live row a program admits, so the set_attrs
    scatters race with the readers' mask and count kernels without making an answer depend on their timing; how a search
    sees codes changing under it is held to the dense evaluator by test_gpu_filters.py.  Removed documents point away
    from every query, so they never reach the dense top-k; only the keyword statistics see the removes, and each store's
    leg answers before or after the remove that follows its prefix."""
    rng = np.random.default_rng(31 + n)
    steps, per, gone_per = 12, 1200, 40
    total = steps * per
    u = rng.standard_normal(DIM).astype(np.float32)
    nq, fetch, k_out = 6, 16, 32
    qv = (u + 0.3 * rng.standard_normal((nq, DIM))).astype(np.float32)
    qt, qo = zipf_queries(rng, nq, vocab=800)
    t, f, off = zipf_docs(rng, total, vocab=800)
    vecs = rng.standard_normal((total, DIM)).astype(np.float32)
    away = np.zeros(total, bool)
    for st in range(steps):
        away[st * per:st * per + gone_per] = True
    vecs[away] = -u + 0.01 * rng.standard_normal((int(away.sum()), DIM)).astype(np.float32)
    ids = np.arange(total, dtype=np.int64) * 3 + 1
    user = np.zeros(total, np.int32)
    org = rng.integers(1, 3, total).astype(np.int32)
    pr = Pair(n, total)
    kind = AttrColumn("kind", 5)
    for v in ("hidden", "visible", "shown"):
        kind.code({"kind": v})
    progs = [compile_program(F("kind").not_equal("hidden"), {"kind": kind}, tenant=(-2, 1)),
             compile_program(None, {}, tenant=(-2, 2))]
    mixed = np.array([0, 1, 0, 0, 1, 0], np.int32)

    def put(st):
        sl = slice(st * per, (st + 1) * per)
        pr.ix.add(vecs[sl], ids[sl], user[sl], org[sl])
        pr.kw.add(ids[sl], t[off[st * per]:off[(st + 1) * per]], f[off[st * per]:off[(st + 1) * per]],
                  off[st * per:(st + 1) * per + 1] - off[st * per], user[sl], org[sl])

    def code(idx, v):
        c = np.full(len(idx), kind.code({"kind": v}), np.int32)
        pr.ix.set_attrs(kind.col, ids[idx], c)
        pr.kw.set_attrs(kind.col, ids[idx], c)

    put(0)
    code(np.arange(per), "visible")              # the column exists on every shard and store before any reader runs
    removed = [set()]                            # removed ids after step s's remove
    answers, errors = [], []
    done = threading.Event()

    def writer():
        try:
            for st in range(1, steps):
                put(st)
                code(np.arange(st * per, (st + 1) * per), "visible")
                code(np.arange((st - 1) * per + gone_per, st * per), "shown")
                gone = np.arange((st - 1) * per, (st - 1) * per + gone_per)
                pr.ix.remove(ids[gone])
                pr.kw.remove(ids[gone])
                code(gone, "hidden")
                removed.append(removed[-1] | set(ids[gone].tolist()))
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            done.set()

    def reader(r):
        i = 0
        try:
            while not done.is_set():
                fusion = FUSIONS[(i + r) % 2]
                mode = (i + r) % 3              # 0: one program, masked scan; 1, 2: two programs, list kernels
                q_prog = np.zeros(nq, np.int32) if mode == 0 else mixed
                answers.append((fusion, q_prog, hybrid_search(
                    pr.ix, pr.kw, qv, fetch, qt, qo, 0.5, None, fusion, k_out, programs=progs[:1] if mode == 0 else progs,
                    q_program=q_prog, max_list_rows=0 if mode < 2 else 10 ** 9)))
                i += 1
        except Exception as e:   # pragma: no cover
            errors.append(e)

    ths = [threading.Thread(target=writer)] + [threading.Thread(target=reader, args=(r,)) for r in range(3)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors
    owner = ids % n
    pos = np.zeros(total, np.int64)              # each row's position in its shard's / store's append order
    for sh in range(n):
        pos[owner == sh] = np.arange(int((owner == sh).sum()))

    def prefix(rows):                            # rows seen: a prefix of every shard's / store's append order
        return pos < np.asarray([rows] if n == 1 else rows, np.int64)[owner]

    def store_steps(k_rows, sh):                 # appended steps a store's prefix holds
        return 0 if k_rows == 0 else int(np.nonzero(owner == sh)[0][k_rows - 1] // per) + 1

    rows32 = round_to_bf16(vecs)
    q32 = round_to_bf16(qv)
    wd, ws = np.full(nq, 0.5), np.full(nq, 0.5)
    snaps = {str(a[2][3]) for a in answers}
    assert len(snaps) >= 2, snaps
    checked = 0
    for fusion, q_prog, (g_ids, g_sc, g_cs, (rd, rk)) in answers[:: max(1, len(answers) // 16)]:
        seen_d, seen_k = prefix(rd), prefix(rk)
        q_org = np.where(q_prog == 0, 1, 2).astype(np.int32)      # both programs admit exactly one org's live rows
        d_ids = np.full((nq, fetch), -1, np.int64)
        d_sc = np.full((nq, fetch), -np.inf, np.float32)
        for q in range(nq):                     # removed rows point away: whether a shard saw the remove is moot
            o_i, o_s = cosine_topk(q32[q:q + 1], rows32, fetch, ids=ids, live=seen_d & (org == q_org[q]) & ~away)
            d_ids[q], d_sc[q] = o_i[0], o_s[0]
        kr = [rk] if n == 1 else rk
        steps_k = [store_steps(kr[sh], sh) for sh in range(n)]
        matched = False
        # a store holding steps 0 .. S-1 has applied the removes through step S-2, or through step S-1 when that
        # step's remove (which follows its append) came before the search's lock: either, per store
        for choice in range(2 ** n):
            gone = set()
            for sh in range(n):
                g = removed[max(steps_k[sh] - 2 + ((choice >> sh) & 1), 0)]
                gone |= {d for d in g if d % n == sh}
            live = seen_k & ~np.isin(ids, np.fromiter(gone, np.int64, len(gone)))
            corpus = Corpus(t, f, off, ids, live=live, row_user=user, row_org=org)
            s_ids, s_sc = bm25_topk(corpus, qt, qo, fetch, q_user=np.full(nq, -2, np.int32), q_org=q_org)
            ok = True
            for q in range(nq):
                wi, wsc, wc = host_fuse(d_ids[q], d_sc[q], s_ids[q], s_sc[q], 0.5, 0.5, fusion, k_out)
                if not np.array_equal(g_ids[q], wi) or not np.array_equal(np.isnan(g_cs[q]), np.isnan(wc)):
                    ok = False
                elif fusion == N.FUSION_RANKED and not np.array_equal(g_sc[q].view(np.int64), wsc.view(np.int64)):
                    ok = False              # ranks only: bit for bit
                elif fusion != N.FUSION_RANKED and not np.allclose(g_sc[q], wsc, rtol=1e-6, atol=0.0):
                    ok = False              # relative scores carry the oracle's cosines, last fp32 bit may differ
                elif not np.allclose(g_cs[q], wc, rtol=0, atol=1e-6, equal_nan=True):
                    ok = False
            matched |= ok
        assert matched, (rd, rk, fusion)
        checked += 1
    assert checked >= 4
    pr.close()


# ---------------------------------------------------------------------- the retriever on top
def _shape(objs, exact=True):
    return [(o.uuid, o.metadata.score if exact else round(o.metadata.score, 12),
             None if o.metadata.distance is None else round(o.metadata.distance, 5)) for o in objs]


@pytest.mark.parametrize("multi", [False, True])
def test_knowledge_base_filtered_hybrid_is_one_device_call(multi, monkeypatch):
    from aurora_b200 import retriever as R
    from aurora_b200.filters import HybridFusion
    from tests.doubles import HashEmbedder, OracleIndex

    emb = HashEmbedder(64)
    factory = (lambda d, c: MultiIndex(d, c, devices=[0, 0])) if multi else None
    dev = R.KnowledgeBase(emb, capacity=8192, index_factory=factory)
    host = R.KnowledgeBase(emb, capacity=8192, index_factory=lambda d, c: OracleIndex(d, c))
    assert dev._hybrid_device and not host._hybrid_device
    words = ["disk", "oom", "pod", "latency", "timeout", "node", "memory", "cpu", "network", "failover", "kafka", "dns"]
    for kb in (dev, host):
        r = np.random.default_rng(1)
        for t in range(30):
            for doc in range(3):
                chunks = [{"chunk_index": c, "content": " ".join(r.choice(words, size=6))} for c in range(8)]
                docid = f"discovery:{t}:{doc}" if doc == 0 else f"doc{t}-{doc}"
                kb.insert(f"u{t}", docid, "f.md", chunks, org_id=f"o{t % 7}")
    flts = [F("org_id").equal(o) & F("document_id").like("discovery:*") for o in ("o3", "o5", "none")] + \
           [F("document_id").like("doc*") & F("user_id").equal("u1")]
    cases = [(q, f, a, fu) for q in ("disk node", "oom memory pod", "nothing here") for f in flts
             for a in (0.0, 0.5, 0.999) for fu in (HybridFusion.RANKED, HybridFusion.RELATIVE_SCORE)]
    want = [host.query(q, 10, filters=f, alpha=a, fusion=fu) for q, f, a, fu in cases]
    want_fac = [R._CollectionFacade(host).query.hybrid("disk node", limit=3, alpha=0.5, filters=f).objects for f in flts]
    late = ("u40", "discovery:late", "f.md", [{"chunk_index": 0, "content": "disk node late"}])
    host.insert(*late, org_id="o3")
    want_late = host.query("disk node", 10, filters=flts[0], alpha=0.5)

    def boom(*a, **k):
        raise AssertionError("host step on the device knowledge base's filtered hybrid path")

    monkeypatch.setattr(bm25, "ranked_fusion", boom)
    monkeypatch.setattr(bm25, "relative_score_fusion", boom)
    monkeypatch.setattr(type(dev.index), "filter_ids", boom)
    for c, w in zip(cases, want):
        exact = c[3] == HybridFusion.RANKED        # relative scores carry the cosines, which may differ in the last bit
        assert _shape(dev.query(c[0], 10, filters=c[1], alpha=c[2], fusion=c[3]), exact) == _shape(w, exact), c
    # the prediscovery call's path: _get_weaviate_client().query.hybrid in process and through the daemon client
    from aurora_b200.daemon import Client, serve

    monkeypatch.setattr(R, "_kb_factory", lambda: dev)
    monkeypatch.setattr(R, "_kb", None)
    _, coll = R._get_weaviate_client()
    sock_dir = tempfile.mkdtemp(prefix="aur-", dir="/tmp" if os.path.isdir("/tmp") else None)
    path = os.path.join(sock_dir, "kb.sock")
    srv = serve(path, background=True)
    try:
        _, remote = Client(path)._get_weaviate_client()
        for f, w in zip(flts, want_fac):
            assert _shape(coll.query.hybrid("disk node", limit=3, alpha=0.5, filters=f).objects) == _shape(w)
            assert _shape(remote.query.hybrid(query="disk node", limit=3, alpha=0.5, filters=f).objects) == _shape(w)
    finally:
        srv.shutdown(); srv.close_all(final_save=False); srv.server_close()
        shutil.rmtree(sock_dir, ignore_errors=True)
    dev.insert(*late, org_id="o3")              # a later insert keeps the columns of both stores current
    assert _shape(dev.query("disk node", 10, filters=flts[0], alpha=0.5)) == _shape(want_late)
    dev.index.close()

"""aur_search_filtered / aur_filter_ids: metadata pre-filters evaluated on the device over attribute columns.  Every
answer equals the host-resolved call over the ids the host predicate (``_Expr.matches``) selects -- aur_search_lists or
aur_search_subset, ids and float32 scores bit for bit -- and the fp64 oracle over the matching rows."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index, MultiIndex, _ptr
from aurora_b200.filters import AttrColumn, Filter, compile_program, pack_programs
from oracle import cosine_topk as O
from tests.gpu_exact import check_host_exact

pytestmark = pytest.mark.gpu

F = Filter.by_property


def _props(rng, n, n_org=50):
    org = rng.integers(n_org, size=n)
    disc = rng.random(n) < 0.5
    return [{"org_id": f"o{o}", "document_id": (f"discovery:{i}" if d else f"doc:{i}"), "n": int(i % 97)}
            for i, (o, d) in enumerate(zip(org, disc))]


class Table:
    """Host side of a shard's attribute columns: the properties of every appended row and their columns."""

    def __init__(self, names=("org_id", "document_id", "n")):
        self.cols = {nm: AttrColumn(nm, 2 + i) for i, nm in enumerate(names)}
        self.rows, self.ids = [], np.zeros(0, np.int64)

    def add(self, ix, vecs, ids, props, set_codes=True):
        ix.add(vecs, ids)
        self.rows += props
        self.ids = np.concatenate([self.ids, ids])
        if set_codes:
            self.set(ix, ids, props)

    def set(self, ix, ids, props):
        for c in self.cols.values():
            ix.set_attrs(c.col, ids, np.array([c.code(p) for p in props], np.int32))

    def program(self, expr):
        return compile_program(expr, self.cols)

    def match(self, expr, live):
        return np.array([expr.matches(p) for p in self.rows]) & live


def _corpus(n, d, seed):
    rng = np.random.default_rng(seed)
    C_ = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    ext = rng.permutation(n).astype(np.int64) * 5 + 11
    return rng, C_, ext


def _queries(rng, nq, d):
    return O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))


@pytest.fixture(scope="module")
def big():
    n, d = 200_000, 64
    rng, C_, ext = _corpus(n, d, 21)
    ix = Index(d, n + 1000)
    t = Table()
    t.add(ix, C_, ext, _props(rng, n))
    dead = ext[rng.choice(n, size=5000, replace=False)]
    ix.remove(dead)
    live = ~np.isin(ext, dead)
    yield rng, C_, ext, ix, t, live
    ix.close()


FILTERS = [
    F("org_id").equal("o3") & F("document_id").like("discovery:*"),
    F("org_id").equal("o7"),
    F("org_id").equal("nobody"),
    F("n").greater_than(-1),                                    # every row
    (F("org_id").equal("o1") | F("org_id").equal("o2")) & F("n").less_than(40),
    F("document_id").like("doc:1?[0-5]*"),
]


@pytest.mark.parametrize("fi", range(len(FILTERS)))
def test_filter_ids_equal_host_predicate(big, fi):
    rng, C_, ext, ix, t, live = big
    want = ext[t.match(FILTERS[fi], live)]
    got = ix.filter_ids(t.program(FILTERS[fi]))
    assert np.array_equal(got, want)                            # row order: the append order here


@pytest.mark.parametrize("k", [1, 10, 32, 100, 128])
def test_search_filtered_equals_search_lists(big, k):
    rng, C_, ext, ix, t, live = big
    progs = [t.program(f) for f in FILTERS]
    q_prog = np.repeat(np.arange(len(progs), dtype=np.int32), 3)
    rng.shuffle(q_prog)
    Q = _queries(rng, len(q_prog), C_.shape[1])
    lists = [ext[t.match(f, live)] for f in FILTERS]
    ids, sc, matched, snap = ix.search_filtered(Q, k, progs, q_prog, max_list_rows=0)
    assert ix.stats()["last_kernel"] == N.KERNEL_LIST
    assert list(matched) == [len(x) for x in lists] and snap == len(ext)
    l_ids, l_sc = ix.search_lists(Q, k, lists, q_prog)
    assert np.array_equal(ids, l_ids) and np.array_equal(sc.view(np.uint32), l_sc.view(np.uint32))
    for p in range(len(progs)):
        qs = np.nonzero(q_prog == p)[0]
        check_host_exact((ids[qs], sc[qs]), Q[qs], C_, k, ids=ext, live=t.match(FILTERS[p], live))


@pytest.mark.parametrize("d", [384, 768, 1024])
def test_dims_list_and_dense(d):
    rng, C_, ext = _corpus(30_000, d, 300 + d)
    with Index(d, len(ext)) as ix:
        t = Table()
        t.add(ix, C_, ext, _props(rng, len(ext), n_org=8))
        Q = _queries(rng, 9, d)
        f = F("org_id").equal("o5") & F("document_id").like("discovery:*")
        allow = ext[t.match(f, np.ones(len(ext), bool))]
        for k in (1, 32, 128):
            ids, sc, m, _ = ix.search_filtered(Q, k, [t.program(f)], max_list_rows=len(allow))      # list path
            assert ix.stats()["last_kernel"] == N.KERNEL_LIST and m[0] == len(allow)
            l_ids, l_sc = ix.search_lists(Q, k, [allow], np.zeros(len(Q), np.int32))
            assert np.array_equal(ids, l_ids) and np.array_equal(sc, l_sc)
            ids, sc, m, _ = ix.search_filtered(Q, k, [t.program(f)], max_list_rows=len(allow) - 1)  # masked scan
            kern = ix.stats()["last_kernel"]
            s_ids, s_sc = ix.search_subset(Q, k, allow)
            assert ix.stats()["last_kernel"] == kern
            assert np.array_equal(ids, s_ids) and np.array_equal(sc, s_sc)
            check_host_exact((ids, sc), Q, C_, k, ids=ext, live=np.isin(ext, allow))


def test_dense_path_uses_the_tensor_core_kernel(big):
    rng, C_, ext, ix, t, live = big
    f = F("n").less_than(50)
    allow = ext[t.match(f, live)]
    Q = _queries(rng, 40, C_.shape[1])
    ids, sc, m, _ = ix.search_filtered(Q, 32, [t.program(f)], max_list_rows=1000)
    assert ix.stats()["last_kernel"] in (N.KERNEL_TC1, N.KERNEL_TC2) and m[0] == len(allow)
    s_ids, s_sc = ix.search_subset(Q, 32, allow)
    assert np.array_equal(ids, s_ids) and np.array_equal(sc, s_sc)


@pytest.mark.parametrize("n_prog", [64, 70])
def test_many_programs_over_256_queries(big, n_prog):
    """More programs than one pass evaluates (32): whole passes, and a last pass of 6."""
    rng, C_, ext, ix, t, live = big
    exprs = [F("org_id").equal(f"o{i % 50}") & (F("document_id").like("discovery:*") if i % 2 else F("n").greater_than(i))
             for i in range(n_prog)]
    q_prog = rng.integers(n_prog, size=256).astype(np.int32)
    Q = _queries(rng, 256, C_.shape[1])
    ids, sc, matched, _ = ix.search_filtered(Q, 16, [t.program(e) for e in exprs], q_prog, max_list_rows=10**9)
    lists = [ext[t.match(e, live)] for e in exprs]
    assert list(matched) == [len(x) for x in lists]
    l_ids, l_sc = ix.search_lists(Q, 16, lists, q_prog)
    assert np.array_equal(ids, l_ids) and np.array_equal(sc, l_sc)


def test_tenant_columns_equal_tenant_search():
    d, n = 128, 20_000
    rng, C_, ext = _corpus(n, d, 8)
    user = rng.integers(-1, 30, size=n).astype(np.int32)
    org = rng.integers(-1, 6, size=n).astype(np.int32)
    with Index(d, n) as ix:
        ix.add(C_, ext, user, org)
        Q = _queries(rng, 5, d)
        for u, o in [(4, 2), (-2, 3), (7, -1)]:
            prog = compile_program(None, {}, tenant=(u, o))
            ids, sc, _, _ = ix.search_filtered(Q, 20, [prog], max_list_rows=0)
            want = ix.search(Q, 20, np.full(5, u, np.int32), np.full(5, o, np.int32))
            assert np.array_equal(ids, want[0])
            check_host_exact((ids, sc), Q, C_, 20, ids=ext, live=(user == u) | ((o >= 0) & (org == o)))


def test_upsert_remove_compact_and_capacity_edge():
    d, n = 96, 6000
    rng, C_, ext = _corpus(n + 700, d, 12)
    with Index(d, n + 200) as ix:
        t = Table()
        t.add(ix, C_[:n], ext[:n], _props(rng, n, n_org=4))
        f = F("org_id").equal("o1") & F("document_id").like("discovery:*")
        Q = _queries(rng, 6, d)

        def check():
            rows, ids_, _, _, live = ix.export()
            # the live rows in row order, with the properties last stored under their ids
            pmap = {int(i): p for i, p in zip(t.ids, t.rows)}
            props = [pmap[int(i)] for i in ids_]
            want = ids_[live & np.array([f.matches(p) for p in props])]
            assert np.array_equal(ix.filter_ids(t.program(f)), want)
            got = ix.search_filtered(Q, 10, [t.program(f)], max_list_rows=10**9)
            exp = ix.search_lists(Q, 10, [want], np.zeros(len(Q), np.int32))
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
            rf = rows.view(np.uint16).astype(np.uint32) << 16
            check_host_exact((got[0], got[1]), Q, rf.view(np.float32), 10, ids=ids_, live=live & np.isin(ids_, want))

        check()
        ix.remove(ext[:300])
        check()
        up = ext[1000:1200]                              # upsert up to capacity: new rows start absent until their codes are set
        ix.add(C_[n:n + 200], up)
        t.rows += [{} for _ in up]
        t.ids = np.concatenate([t.ids, up])
        check()
        new_p = [{"org_id": "o1", "document_id": f"discovery:u{i}", "n": 1} for i in range(200)]
        t.set(ix, up, new_p)
        t.rows[-200:] = new_p
        check()
        assert ix.compact() == 500                       # 300 removed + 200 upserted-away rows
        check()
        tail = ext[n + 200:n + 700]                      # refill to capacity: the rows compaction freed (some of them held
        ix.add(C_[n + 200:n + 700], tail)                # matching codes before it) start absent
        t.rows += [{} for _ in tail]
        t.ids = np.concatenate([t.ids, tail])
        check()
        assert ix.stats()["rows"] == ix.capacity


def test_concurrent_writer_and_readers():
    d, n0, step, steps = 64, 4000, 500, 12
    rng, C_, ext = _corpus(n0 + step * steps, d, 9)
    props = [{"org_id": "o1" if i % 3 else "o2", "document_id": f"discovery:{i}"} for i in range(len(ext))]
    with Index(d, len(ext) + 64) as ix:
        t = Table(("org_id", "document_id"))
        t.add(ix, C_[:n0], ext[:n0], props[:n0])
        for a in range(n0, len(ext)):                    # codes of values to come, so the program's bitmaps cover them
            for c in t.cols.values():
                c.code(props[a])
        prog = t.program(F("org_id").equal("o1") & F("document_id").like("discovery:*"))
        Q = _queries(rng, 4, d)
        done, started = [n0], [n0]     # rows appended with all their codes set / rows whose append has begun
        results, id_results, errors = [], [], []

        def writer():
            for i in range(steps):
                a = n0 + i * step
                started[0] = a + step
                ix.add(C_[a:a + step], ext[a:a + step])
                t.set(ix, ext[a:a + step], props[a:a + step])
                done[0] = a + step

        def reader():
            try:
                for _ in range(10):
                    before = done[0]
                    ids, sc, _, _ = ix.search_filtered(Q, 16, [prog], max_list_rows=10**9)
                    results.append((before, started[0], ids, sc))
                    before = done[0]
                    got = ix.filter_ids(prog)       # rows appended past its snapshot must not appear
                    id_results.append((before, started[0], got))
            except Exception as e:          # noqa: BLE001 - surfaced below
                errors.append(e)

        ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
        for th in ts:
            th.start()
        for th in ts:
            th.join()
        assert not errors, errors
        match = np.array([p["org_id"] == "o1" for p in props])
        # a search sees each row's codes as they were when its filter kernel read them: every row completed before it
        # began, and any of the rows being appended meanwhile (those it returned count as seen)
        for before, after, ids, sc in results:
            seen = match[:after] & ((np.arange(after) < before) | np.isin(ext[:after], ids))
            want = O.cosine_topk(Q, C_[:after], 16, ids=ext[:after], live=seen)
            assert np.array_equal(ids, want[0]), (before, after)
        assert id_results
        for before, after, got in id_results:
            head = ext[:before][match[:before]]
            assert np.array_equal(got[:len(head)], head), (before, after)
            tail = np.arange(before, after)[match[before:after]]                # in-flight matching rows, row order
            assert np.array_equal(got[len(head):], ext[tail[np.isin(ext[tail], got)]]), (before, after)


def test_multi_index_three_shards_equal_one_index():
    d, n = 128, 12_000
    rng, C_, ext = _corpus(n, d, 4)
    props = _props(rng, n, n_org=5)
    with MultiIndex(d, 20_000, devices=[0, 0, 0]) as mi, Index(d, n) as one:
        t1, t3 = Table(), Table()
        t1.add(one, C_, ext, props)
        t3.add(mi, C_, ext, props)
        exprs = [F("org_id").equal("o2") & F("document_id").like("discovery:*"), F("n").less_than(90)]
        Q = _queries(rng, 6, d)
        q_prog = np.array([0, 1, 0, 1, 1, 0], np.int32)
        for mlr in (0, 10**9):
            a = mi.search_filtered(Q, 32, [t3.program(e) for e in exprs], q_prog, max_list_rows=mlr)
            b = one.search_filtered(Q, 32, [t1.program(e) for e in exprs], q_prog, max_list_rows=mlr)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        assert np.array_equal(np.sort(mi.filter_ids(t3.program(exprs[0]))), np.sort(one.filter_ids(t1.program(exprs[0]))))


def _raw(ix, Q, k, tok, off, n_prog, bm, qp):
    q = ix._rows_buffer(Q)
    nq = q.shape[0]
    scores = np.full((nq, k), 7.0, np.float32)
    ids = np.full((nq, k), 77, np.int64)
    matched = np.full(max(n_prog, 1), 5, np.int64)
    snap = C.c_int64(-9)
    rc = ix._lib.aur_search_filtered(ix._h, _ptr(q), nq, int(k), _ptr(tok), _ptr(off), int(n_prog), _ptr(bm), bm.shape[0],
                                     _ptr(qp), 0, _ptr(scores), _ptr(ids), _ptr(matched), C.byref(snap))
    return rc, ((scores == 7.0).all() and (ids == 77).all() and (matched == 5).all() and snap.value == -9)


def test_malformed_programs_are_rejected_with_outputs_untouched():
    d = 64
    rng, C_, ext = _corpus(500, d, 2)
    Q = _queries(rng, 3, d)
    qp = np.zeros(3, np.int32)
    with Index(d, 1000) as ix:
        t = Table(("org_id",))
        t.add(ix, C_, ext, _props(rng, 500, n_org=3))
        tok, off, bm = pack_programs([t.program(F("org_id").equal("o1") | F("org_id").equal("o2"))])
        leaf, op = tok[0].copy(), tok[2].copy()
        cases = {
            "underflow": np.array([leaf, op]),
            "two values left": np.array([leaf, leaf]),
            "column out of range": np.array([[0, 18, 0, 1]]),
            "column never set": np.array([[0, 5, 0, 1]]),
            "slice past the bitmap": np.array([[0, 2, 0, bm.shape[0] * 32 + 1]]),
            "negative offset": np.array([[0, 2, -1, 1]]),
            "unknown token": np.array([[7, 0, 0, 0]]),
            "33 leaves": np.array([leaf] + [leaf, op] * 32),
        }
        for name, tk in cases.items():
            tk = np.ascontiguousarray(tk, np.int32)
            o = np.array([0, len(tk)], np.int32)
            rc, untouched = _raw(ix, Q, 5, tk, o, 1, bm, qp)
            assert rc == N.AUR_ERR_INVALID and untouched, name
            n_out = C.c_int64(-3)
            out = np.full(4, 9, np.int64)
            assert ix._lib.aur_filter_ids(ix._h, _ptr(tk), len(tk), _ptr(bm), bm.shape[0], _ptr(out), 4,
                                          C.byref(n_out)) == N.AUR_ERR_INVALID, name
            assert n_out.value == -3 and (out == 9).all()
        rc, untouched = _raw(ix, Q, 5, tok, off, 1, bm, np.array([0, 1, 0], np.int32))     # q_program out of range
        assert rc == N.AUR_ERR_INVALID and untouched
        rc, untouched = _raw(ix, Q, 5, tok, off, 1025, bm, qp)                             # more than 1024 programs
        assert rc == N.AUR_ERR_INVALID and untouched
        rc, untouched = _raw(ix, Q, 129, tok, off, 1, bm, qp)
        assert rc == N.AUR_ERR_UNSUPPORTED and untouched
        assert ix._lib.aur_set_attrs(ix._h, 1, _ptr(ext), _ptr(np.zeros(500, np.int32)), 500) == N.AUR_ERR_INVALID
        rc, _ = _raw(ix, Q, 5, tok, off, 1, bm, qp)
        assert rc == N.AUR_OK
    with Index(d, 1000, dtype="f32") as f32:
        f32.add(C_, ext)
        f32.set_attrs(2, ext, np.zeros(500, np.int32))
        rc, untouched = _raw(f32, Q, 5, tok, off, 1, bm, qp)
        assert rc == N.AUR_ERR_UNSUPPORTED and untouched


# ---------------------------------------------------------------------- the retriever on top
def _shape(objs):
    return [(o.uuid, round(o.metadata.score, 5)) for o in objs]


def _recording(index):
    calls = []
    inner = index.search_filtered

    def search_filtered(*a, **kw):
        out = inner(*a, **kw)
        calls.append((int(out[2][0]), index.stats()["last_kernel"]))
        return out
    index.search_filtered = search_filtered
    return calls


def test_knowledge_base_equals_host_path(monkeypatch):
    from aurora_b200 import incident_knowledge as IK
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder, OracleIndex

    emb = HashEmbedder(64)
    dev = R.KnowledgeBase(emb, capacity=8192)
    host = R.KnowledgeBase(emb, capacity=8192, index_factory=lambda d, c: OracleIndex(d, c))
    calls = _recording(dev.index)
    words = ["disk", "oom", "pod", "latency", "timeout", "node", "memory", "cpu", "network", "failover", "kafka", "dns"]
    for kb in (dev, host):
        r = np.random.default_rng(1)
        for t in range(30):
            for doc in range(3):
                chunks = [{"chunk_index": c, "content": " ".join(r.choice(words, size=6))} for c in range(8)]
                docid = f"discovery:{t}:{doc}" if doc == 0 else f"doc{t}-{doc}"
                kb.insert(f"u{t}", docid, "f.md", chunks, org_id=f"o{t % 7}")
    for q in ("disk node", "oom memory pod"):
        for o in ("o3", "o5", "none"):
            flt = F("org_id").equal(o) & F("document_id").like("discovery:*")     # the prediscovery filter
            for alpha in (None, 1.0, 0.5):
                assert _shape(dev.query(q, 10, filters=flt, alpha=alpha)) == _shape(host.query(q, 10, filters=flt, alpha=alpha))
            fac_d = R._CollectionFacade(dev).query.hybrid(q, limit=8, alpha=0.5, filters=flt).objects
            fac_h = R._CollectionFacade(host).query.hybrid(q, limit=8, alpha=0.5, filters=flt).objects
            assert _shape(fac_d) == _shape(fac_h)
    # the retriever's list-vs-scan rule picked the kernel, as on the host path
    max_list = int(R._LIST_MAX_FRACTION * len(dev._props))
    assert calls and all((k == N.KERNEL_LIST) == (m <= max_list) for m, k in calls)
    assert {m for m, _ in calls} == {0, 4 * 8}                  # an empty org, and orgs of four 8-chunk discovery docs
    # Aurora Learn: an org filter through incident_knowledge; inserts after the columns exist keep them current
    outs = []
    n_calls = len(calls)
    for kb in (dev, host):
        IK.configure(factory=lambda kb=kb: kb, org_resolver=lambda u: "o2" if u != "u9" else None)
        for i in range(12):
            assert IK.store_good_rca(f"u{i % 3}", f"inc{i}", f"fb{i}", f"disk full on node {i}", "svc", "k8s", "sev2",
                                     "root cause", [{"content": "step"}], [], org_id="o2" if i % 2 else None)
        outs.append([IK.search_similar_good_rcas(u, "disk full", "svc", "k8s", limit=5, min_score=-1.0) for u in ("u1", "u9")])
    assert outs[0] == outs[1] and outs[0][0]
    assert len(calls) == n_calls + 2
    dev.index.close()

"""aur_filter_count / aur_remove_filtered: counts and deletes by filter program on the device, and aur_remove's one-launch
tombstones.  Every count equals ``len(filter_ids)`` and the host predicate's; every delete removes exactly the live rows
the host predicate selects, and nothing searches, exports or counts them afterwards.  On top, a ``KnowledgeBase`` that
resolves its deletes on the device ends where its twin on the host scan ends."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import incident_knowledge as IK
from aurora_b200 import retriever as R
from aurora_b200.engine import Index, MultiIndex, _ptr
from aurora_b200.filters import AttrColumn, Filter, compile_program, pack_programs
from oracle import cosine_topk as O
from tests.doubles import HashEmbedder
from tests.test_delete_filtered_cpu import MODULE, OLD, _calls, _objects

pytestmark = pytest.mark.gpu

F = Filter.by_property
NAMES = ("org_id", "document_id", "n")


def _props(rng, n, n_org=20):
    org = rng.integers(n_org, size=n)
    disc = rng.random(n) < 0.5
    return [{"org_id": f"o{o}", "document_id": (f"discovery:{i}" if d else f"doc:{i}"), "n": int(i % 97)}
            for i, (o, d) in enumerate(zip(org, disc))]


class Table:
    """The host side of a shard's attribute columns: every appended row's properties, in append order."""

    def __init__(self):
        self.cols = {nm: AttrColumn(nm, 2 + i) for i, nm in enumerate(NAMES)}
        self.rows = []

    def add(self, ix, vecs, ids, props, user=None):
        ix.add(vecs, ids, user)
        self.rows += props
        for c in self.cols.values():
            ix.set_attrs(c.col, ids, np.array([c.code(p) for p in props], np.int32))

    def program(self, expr):
        return compile_program(expr, self.cols)

    def selected(self, ix, expr):
        """Ids of the live rows ``expr`` matches, in row order: the host predicate over the export."""
        _, ids, _, _, live = ix.export()
        return ids[live & np.array([expr.matches(p) for p in self.rows], bool)]


def _random_expr(rng, depth=0):
    if depth < 3 and rng.random() < 0.6:
        a, b = _random_expr(rng, depth + 1), _random_expr(rng, depth + 1)
        return a & b if rng.random() < 0.5 else a | b
    kind = rng.integers(5)
    if kind == 0:
        return F("org_id").equal(f"o{rng.integers(25)}")
    if kind == 1:
        return F("org_id").not_equal(f"o{rng.integers(25)}")
    if kind == 2:
        return F("document_id").like(["discovery:*", "doc:1*", "doc:?5*"][rng.integers(3)])
    if kind == 3:
        return F("n").less_than(int(rng.integers(100)))
    return F("n").greater_than(int(rng.integers(100)))


def _shard(dtype, n=40_000, d=128, seed=0, cap_extra=10_000):
    """A shard with tenant codes, three attribute columns, removed ids and upserted ids (their old rows tombstones)."""
    rng = np.random.default_rng(seed)
    C_ = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    ext = rng.permutation(n).astype(np.int64) * 3 + 7
    ix = Index(d, n + cap_extra, dtype=dtype)
    t = Table()
    props = _props(rng, n)
    t.add(ix, C_, ext, props, user=rng.integers(5, size=n).astype(np.int32))
    ix.remove(ext[rng.choice(n, size=n // 20, replace=False)])
    up = rng.choice(n, size=500, replace=False)
    t.add(ix, C_[up], ext[up], [props[i] for i in up], user=np.zeros(len(up), np.int32))
    return rng, C_, ext, ix, t


def _raw_remove(ix, tok, bm, cap, out_fill=9, n_fill=-3):
    out = np.full(max(cap, 1), out_fill, np.int64)
    n = C.c_int64(n_fill)
    rc = ix._lib.aur_remove_filtered(ix._h, _ptr(tok), len(tok), _ptr(bm), bm.shape[0], _ptr(out), cap, C.byref(n))
    return rc, out, n.value


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_count_filtered_equals_filter_ids_and_host(dtype):
    rng, C_, ext, ix, t = _shard(dtype, seed=1)
    with ix:
        for _ in range(24):
            e = _random_expr(rng)
            prog = t.program(e)
            n = ix.count_filtered(prog)
            assert n == len(ix.filter_ids(prog)) == len(t.selected(ix, e)), e


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_remove_filtered_removes_what_the_host_selects(dtype):
    rng, C_, ext, ix, t = _shard(dtype, seed=2)
    with ix:
        e = F("org_id").equal("o3") | (F("document_id").like("discovery:*") & F("n").less_than(30))
        want = t.selected(ix, e)
        live0 = ix.stats()["live"]
        got = ix.remove_filtered(t.program(e))
        assert np.array_equal(got, want) and len(np.unique(got)) == len(got)   # row order; an upserted id once
        gone = set(got.tolist())
        assert ix.stats()["live"] == live0 - len(got)
        _, ids, _, _, live = ix.export()
        assert not live[np.isin(ids, got)].any()
        Q = O.round_to_bf16(rng.standard_normal((16, C_.shape[1])).astype(np.float32))
        answers = [ix.search(Q, 64)[0], ix.search(Q, 64, np.arange(16, dtype=np.int32) % 5, np.full(16, -1, np.int32))[0],
                   ix.search_subset(Q, 64, ext)[0], ix.search_lists(Q, 64, [got, ext], np.arange(16, dtype=np.int32) % 2)[0]]
        answers.append(ix.search_filtered(Q, 64, [t.program(F("n").greater_than(-1))], max_list_rows=0)[0])
        answers.append(ix.search_filtered(Q, 64, [t.program(e)], max_list_rows=10**9)[0])
        for a in answers:
            assert not gone & set(a.ravel().tolist())
        assert ix.count_filtered(t.program(e)) == 0 and len(ix.remove_filtered(t.program(e))) == 0
        rows = ix.stats()["rows"]
        assert ix.compact() == rows - ix.stats()["live"] and ix.stats()["rows"] == ix.stats()["live"]
        _, ids, _, _, live = ix.export()
        assert live.all() and not np.isin(ids, got).any() and len(ids) == live0 - len(got)


def test_edge_cases():
    d = 64
    rng = np.random.default_rng(3)
    with Index(d, 4000) as empty:
        t = Table()
        t.add(empty, np.zeros((0, d), np.float32), np.zeros(0, np.int64), [])
        prog = t.program(F("org_id").equal("o1"))
        assert empty.count_filtered(prog) == 0 and len(empty.remove_filtered(prog)) == 0
    C_ = O.round_to_bf16(rng.standard_normal((3000, d)).astype(np.float32))
    ext = np.arange(3000, dtype=np.int64) + 100
    with Index(d, 4000) as ix:
        t = Table()
        t.add(ix, C_, ext, _props(rng, 3000, n_org=4))
        nothing, every = t.program(F("org_id").equal("nobody")), t.program(F("n").greater_than(-1))
        assert ix.count_filtered(nothing) == 0 and len(ix.remove_filtered(nothing)) == 0 and ix.stats()["live"] == 3000
        # no room: nothing removed, the count reported, the ids untouched
        tok, _, bm = pack_programs([t.program(F("org_id").equal("o1"))])
        n1 = len(t.selected(ix, F("org_id").equal("o1")))
        rc, out, n = _raw_remove(ix, tok, bm, n1 - 1)
        assert rc == N.AUR_OK and n == n1 and (out == 9).all() and ix.stats()["live"] == 3000
        rc, out, n = _raw_remove(ix, tok, bm, 0)
        assert rc == N.AUR_OK and n == n1 and ix.stats()["live"] == 3000
        # malformed programs: rejected, nothing removed, outputs untouched
        leaf, op = tok[0].copy(), np.array([N.FILTER_OR, 0, 0, 0], np.int32)
        cases = {"underflow": [leaf, op], "two values left": [leaf, leaf], "column out of range": [[0, 18, 0, 1]],
                 "column never set": [[0, 9, 0, 1]], "slice past the bitmap": [[0, 2, 0, bm.shape[0] * 32 + 1]],
                 "unknown token": [[7, 0, 0, 0]], "33 leaves": [leaf] + [leaf, op] * 32}
        for name, tk in cases.items():
            tk = np.ascontiguousarray(np.array(tk), np.int32)
            rc, out, n = _raw_remove(ix, tk, bm, 5000)
            assert rc == N.AUR_ERR_INVALID and n == -3 and (out == 9).all(), name
            cnt = C.c_int64(-3)
            assert ix._lib.aur_filter_count(ix._h, _ptr(tk), len(tk), _ptr(bm), bm.shape[0], C.byref(cnt)) == N.AUR_ERR_INVALID
            assert cnt.value == -3
        assert ix.stats()["live"] == 3000
        got = ix.remove_filtered(every)
        assert np.array_equal(got, ext) and ix.stats()["live"] == 0 and not ix.export()[4].any()
        assert (ix.search(C_[:4], 8)[0] == -1).all()


def test_remove_many_ids_equals_small_batches():
    d, n = 64, 150_000
    rng = np.random.default_rng(4)
    C_ = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    ext = np.arange(n, dtype=np.int64) * 2
    kill = np.concatenate([rng.choice(ext, size=120_000, replace=False), ext[:10], np.arange(1, 2001, 2)])  # repeats, unknowns
    rng.shuffle(kill)
    with Index(d, n) as a, Index(d, n) as b:
        a.add(C_, ext)
        b.add(C_, ext)
        known = len(np.unique(kill[np.isin(kill, ext)]))
        assert a.remove(kill) == known                      # one call: one upload, one launch
        assert sum(b.remove(kill[i:i + 700]) for i in range(0, len(kill), 700)) == known
        assert a.stats()["live"] == b.stats()["live"] == n - known
        ea, eb = a.export(), b.export()
        assert np.array_equal(ea[4], eb[4]) and np.array_equal(ea[1], eb[1])
        assert np.array_equal(ea[4], ~np.isin(ext, kill))


def test_remove_filtered_while_appending_and_searching():
    d, n0, batch, batches = 128, 20_000, 2000, 15
    rng = np.random.default_rng(5)
    total = n0 + batch * batches
    C_ = O.round_to_bf16(rng.standard_normal((total, d)).astype(np.float32))
    ext = rng.permutation(total).astype(np.int64)
    props = _props(rng, total, n_org=12)
    Q = O.round_to_bf16(rng.standard_normal((8, d)).astype(np.float32))
    gone, lock, errors = set(), threading.Lock(), []
    with Index(d, total) as ix:
        t = Table()
        t.add(ix, C_[:n0], ext[:n0], props[:n0])
        done = threading.Event()

        def writer():
            try:
                for b in range(batches):
                    s = slice(n0 + b * batch, n0 + (b + 1) * batch)
                    t.add(ix, C_[s], ext[s], props[s])
            except Exception as e:   # noqa: BLE001
                errors.append(e)
            finally:
                done.set()

        def remover():
            try:
                for o in range(12):
                    ids = ix.remove_filtered(compile_program(F("org_id").equal(f"o{o}"), t.cols))
                    with lock:
                        gone.update(ids.tolist())
            except Exception as e:   # noqa: BLE001
                errors.append(e)

        def reader():
            try:
                while not done.is_set():
                    with lock:
                        before = set(gone)
                    ids, _, snap = ix.search_snapshot(Q, 32)
                    got = set(ids.ravel().tolist()) - {-1}
                    assert not got & before, "a removed id came back"
                    assert got <= set(ext[:snap].tolist()), "an id outside the snapshot"
            except Exception as e:   # noqa: BLE001
                errors.append(e)

        th = [threading.Thread(target=f) for f in (writer, remover, reader, reader)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert not errors, errors
        _, ids, _, _, live = ix.export()
        assert not live[np.isin(ids, list(gone))].any() and ix.stats()["live"] == total - len(gone)


def test_multi_index_equals_one_index():
    d, n = 128, 12_000
    rng = np.random.default_rng(6)
    C_ = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    ext = rng.permutation(n).astype(np.int64) * 5 + 11
    props = _props(rng, n, n_org=5)
    with MultiIndex(d, 20_000, devices=[0, 0, 0]) as mi, Index(d, n) as one:
        t1, t3 = Table(), Table()
        t1.add(one, C_, ext, props)
        t3.add(mi, C_, ext, props)
        for e in (F("org_id").equal("o2") & F("document_id").like("discovery:*"), F("n").less_than(50), F("org_id").equal("x")):
            assert mi.count_filtered(t3.program(e)) == one.count_filtered(t1.program(e))
            a, b = mi.remove_filtered(t3.program(e)), one.remove_filtered(t1.program(e))
            assert sorted(a.tolist()) == sorted(b.tolist())
        assert mi.stats()["live"] == one.stats()["live"]


# ---------------------------------------------------------------------- the knowledge base on top
def _shape(objs):
    return [(o.uuid, round(o.metadata.score, 5)) for o in objs]


def _answers(kb):
    out = []
    flt = F("org_id").equal("o0") & F("document_id").like("discovery:*")
    for q in ("chunk disk", "oom of d3"):
        for alpha in (None, 0.5):
            out.append(_shape(kb.query(q, 10, alpha=alpha)))
            out.append(_shape(kb.query(q, 10, alpha=alpha, filters=flt)))
            out.append(_shape(kb.query(q, 10, alpha=alpha, user_id="u0", scoped=True)))
    return out


def _kb(dtype, wal, host):
    kb = R.KnowledgeBase(HashEmbedder(128), capacity=8192, dtype=dtype)
    if host:
        kb._device_program = lambda *a, **k: None
    kb.attach_wal(wal)
    return kb


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_knowledge_base_twins(tmp_path, dtype):
    saved = [(m, m._kb, m._kb_factory) for m in (R, IK)]
    kbs = [_kb(dtype, str(tmp_path / f"{name}.wal"), name == "host") for name in ("host", "device")]
    try:
        for kb in kbs:
            for user, org, objs in _objects(7, n_docs=120):
                kb.insert_objects(objs, user, org)
        calls = []
        inner = kbs[1].index.remove_filtered
        kbs[1].index.remove_filtered = lambda prog: calls.append(1) or inner(prog)
        for fn, args in _calls():
            res = []
            for kb in kbs:
                want = [rid for rid, p in kb._props.items() if OLD[fn](*args)(p)]
                mod = MODULE.get(fn, R)
                mod.configure(factory=lambda kb=kb: kb, **({"org_resolver": lambda u: None} if mod is IK else {}))
                res.append(getattr(mod, fn)(*args))
                assert res[-1] == (True if fn == "delete_incident_knowledge" else len(want)), (fn, args)
            assert res[0] == res[1]
        assert calls                                         # the device path ran
        host, dev = kbs
        assert host._props == dev._props and host._key2id == dev._key2id and host.mutations == dev.mutations
        kw = [{k: v for k, v in kb.sparse.stats().items() if k in ("docs", "live", "postings_used", "total_len")} for kb in kbs]
        assert kw[0] == kw[1] and kw[0]["live"] == len(host._props)
        assert host.index.stats()["live"] == dev.index.stats()["live"] == len(host._props)
        assert _answers(host) == _answers(dev)
        for kb in kbs:
            kb._wal.close()
        again = [R.KnowledgeBase(HashEmbedder(128), capacity=8192, dtype=dtype) for _ in kbs]
        for kb, name in zip(again, ("host", "device")):
            kb.attach_wal(str(tmp_path / f"{name}.wal"))
            kb._wal.close()
        assert again[0]._props == again[1]._props == host._props
        assert _answers(again[0]) == _answers(again[1]) == _answers(host)
        for kb in kbs + again:
            kb.index.close()
    finally:
        for m, kb, factory in saved:
            m._kb, m._kb_factory = kb, factory

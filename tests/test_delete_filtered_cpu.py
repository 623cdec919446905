"""Deletes and counts by filter, without a GPU.  The six public delete / count functions pass ``Filter`` trees that match
exactly the objects their former predicates matched (absent and ``None`` values included); over the CPU doubles every
one of them takes the host scan and answers as before; over a double with ``remove_filtered`` / ``count_filtered`` (the
device program evaluated on the host) the device path answers as the host path does, down to the mutation log."""

from __future__ import annotations

import fnmatch
import os
import re

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import incident_knowledge as IK
from aurora_b200 import retriever as R
from aurora_b200.filters import _Expr
from tests.doubles import HashEmbedder, OracleIndex

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "aurora_b200.h")
USERS = ["u0", "u1", "u2", None]
DOCS = ["d0", "d1", "discovery:a", "discovery:b", None]
ORGS = ["o0", "o1", None]
INCIDENTS = ["i0", "i1", None]
STAMPS = [f"2026-01-0{d}T00:00:00+00:00" for d in range(1, 8)]


def _table(seed, n=400):
    """Property dicts with every key sometimes absent and every value sometimes None."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        p = {"user_id": USERS[rng.integers(len(USERS))], "document_id": DOCS[rng.integers(len(DOCS))],
             "org_id": ORGS[rng.integers(len(ORGS))], "incident_id": INCIDENTS[rng.integers(len(INCIDENTS))],
             "created_at": STAMPS[rng.integers(len(STAMPS))]}
        out.append({k: v for k, v in p.items() if rng.random() > 0.15})
    return out


def _old_discovery(org, before):
    def pred(p):
        doc = p.get("document_id")
        ok = p.get("org_id") == org and isinstance(doc, str) and fnmatch.fnmatchcase(doc, "discovery:*")
        return ok and (not before or (p.get("created_at") is not None and p.get("created_at") < before))
    return pred


# every public delete / count function: the predicate it passed before it passed a Filter tree, by its arguments
OLD = {
    "delete_document_chunks": lambda u, d: lambda p: p.get("user_id") == u and p.get("document_id") == d,
    "get_document_chunk_count": lambda u, d: lambda p: p.get("user_id") == u and p.get("document_id") == d,
    "delete_user_chunks": lambda u: lambda p: p.get("user_id") == u,
    "delete_discovery_chunks": _old_discovery,
    "delete_incident_knowledge": lambda u, i: lambda p: p.get("user_id") == u and p.get("incident_id") == i,
    "delete_user_knowledge": lambda u: lambda p: p.get("user_id") == u,
}
MODULE = {"delete_incident_knowledge": IK, "delete_user_knowledge": IK}
CASES = [(fn, (u, d)) for fn in ("delete_document_chunks", "get_document_chunk_count") for u in USERS for d in DOCS]
CASES += [(fn, (u,)) for fn in ("delete_user_chunks", "delete_user_knowledge") for u in USERS]
CASES += [("delete_discovery_chunks", (o, b)) for o in ORGS for b in (None, "", STAMPS[3])]
CASES += [("delete_incident_knowledge", (u, i)) for u in USERS for i in INCIDENTS]


def _run(kb, fn, args):
    mod = MODULE.get(fn, R)
    mod.configure(factory=lambda: kb, **({"org_resolver": lambda u: None} if mod is IK else {}))
    return getattr(mod, fn)(*args)


@pytest.fixture(autouse=True)
def _module_state():
    """The retriever's and Aurora Learn's configured backends, put back after each test."""
    saved = [(m, m._kb, m._kb_factory) for m in (R, IK)]
    yield
    for m, kb, factory in saved:
        m._kb, m._kb_factory = kb, factory


class Recorder:
    """A knowledge base that records what it is asked to delete or count."""

    def __init__(self):
        self.preds = []

    def delete_where(self, pred):
        self.preds.append(pred)
        return 0

    count_where = delete_where


@pytest.mark.parametrize("case", range(len(CASES)))
def test_filter_tree_matches_former_predicate(case):
    fn, args = CASES[case]
    rec = Recorder()
    _run(rec, fn, args)
    (pred,) = rec.preds
    assert isinstance(pred, _Expr)                   # a tree: the knowledge base may resolve it on the device
    old = OLD[fn](*args)
    for seed in range(3):
        table = _table(seed)
        assert [pred.matches(p) for p in table] == [bool(old(p)) for p in table]


def test_exports_list_the_filtered_entry_points():
    with open(HEADER, encoding="utf-8") as f:
        declared = set(re.findall(r"^\s*int\s+(aur_\w+)\s*\(", f.read(), flags=re.M))
    for name in ("aur_filter_count", "aur_remove_filtered"):
        assert name in declared and name in N.EXPORTS


# ---------------------------------------------------------------------- twins: host scan vs. device path (emulated)
class ProgramIndex(OracleIndex):
    """OracleIndex with attribute columns and ``count_filtered`` / ``remove_filtered``: each program evaluated on the host
    over the rows' codes, as the device evaluates it (tests/test_filter_compile.py restates the same rule)."""

    dtype = N.AUR_BF16

    def __init__(self, dim, capacity):
        super().__init__(dim, capacity)
        self.attrs, self.calls = {}, []

    def set_attrs(self, col, ids, codes):
        self.attrs.setdefault(col, {}).update(zip(np.asarray(ids).tolist(), np.asarray(codes).tolist()))

    def search_filtered(self, *a, **kw):
        raise AssertionError("deletes never search")

    def _matches(self, prog):
        leaves, toks = prog
        stack = []
        for t in toks:
            if t >= 0:
                col, bits = leaves[t]
                c = {0: self.user, 1: self.org}.get(col)
                if c is None:
                    c = np.array([self.attrs.get(col, {}).get(int(d), -1) for d in self.ids])
                idx = np.asarray(c, np.int64) + 1
                ok = (idx >= 0) & (idx < len(bits))
                v = np.zeros(len(self.ids), bool)
                v[ok] = np.asarray(bits, bool)[idx[ok]]
                stack.append(v)
            else:
                b, a = stack.pop(), stack.pop()
                stack.append(a & b if t == -1 else a | b)
        return stack[0] & self.live

    def count_filtered(self, prog):
        self.calls.append("count_filtered")
        return int(self._matches(prog).sum())

    def remove_filtered(self, prog):
        self.calls.append("remove_filtered")
        hit = self._matches(prog)
        self.live[hit] = False
        return self.ids[hit]


def _objects(seed, n_docs=60):
    """Seeded (tenant, objects) inserts: None users, objects without org_id, discovery documents, shared timestamps."""
    rng = np.random.default_rng(seed)
    batches = []
    for d in range(n_docs):
        user = USERS[rng.integers(len(USERS))]
        org = ORGS[rng.integers(len(ORGS))]
        doc = f"discovery:{d}" if rng.random() < 0.4 else f"d{d % 7}"
        stamp = STAMPS[rng.integers(len(STAMPS))]
        objs = []
        for c in range(int(rng.integers(1, 6))):
            props = {"user_id": user, "document_id": doc, "chunk_index": c, "content": f"chunk {c} of {doc} disk oom",
                     "heading_context": "", "source_filename": f"{doc}.md", "created_at": stamp}
            if org:
                props["org_id"] = org
            objs.append((R.generate_uuid5(f"{user}:{doc}:{c}"), props, props["content"]))
        batches.append((user, org, objs))
    return batches


def _twins(tmp_path, seed):
    kbs = []
    for name, factory in (("host", OracleIndex), ("device", ProgramIndex)):
        kb = R.KnowledgeBase(HashEmbedder(32), capacity=4096, index_factory=factory)
        kb.attach_wal(str(tmp_path / f"{name}.wal"))
        for user, org, objs in _objects(seed):
            kb.insert_objects(objs, user, org)
        kbs.append(kb)
    return kbs


def _calls():
    """The public delete / count calls of one round, as (function, args)."""
    out = [("get_document_chunk_count", (u, d)) for u in USERS for d in ("d0", "d3", "discovery:5", None)]
    out += [("delete_document_chunks", ("u1", "d2")), ("delete_document_chunks", (None, "d4")),
            ("delete_discovery_chunks", ("o0", STAMPS[4])), ("delete_discovery_chunks", ("o1", None)),
            ("delete_incident_knowledge", ("u0", None)), ("delete_user_chunks", ("u2",)),
            ("delete_user_knowledge", (None,)), ("get_document_chunk_count", ("u0", "d0"))]
    return out


def test_cpu_doubles_take_the_host_scan():
    kb = R.KnowledgeBase(HashEmbedder(32), capacity=4096, index_factory=OracleIndex)
    for user, org, objs in _objects(5):
        kb.insert_objects(objs, user, org)
    assert kb._delete_program(R.Filter.by_property("user_id").equal("u0")) is None
    for fn, args in _calls():
        want = [rid for rid, p in kb._props.items() if OLD[fn](*args)(p)]
        got = _run(kb, fn, args)
        assert got == (True if fn == "delete_incident_knowledge" else len(want)), (fn, args)
        if fn.startswith("delete"):
            assert not set(want) & set(kb._props)
            assert set(kb.index.ids[kb.index.live]) == set(kb._props)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_device_path_answers_as_the_host_scan(tmp_path, seed):
    host, dev = _twins(tmp_path, seed)
    for fn, args in _calls():
        assert _run(host, fn, args) == _run(dev, fn, args), (fn, args)
    assert "remove_filtered" in dev.index.calls and "count_filtered" in dev.index.calls
    assert host._props == dev._props and host._key2id == dev._key2id and host.mutations == dev.mutations
    assert set(host.index.ids[host.index.live]) == set(dev.index.ids[dev.index.live]) == set(host._props)
    q = [kb.query("disk oom chunk", 10, user_id="u0", scoped=True) for kb in (host, dev)]
    assert [o.uuid for o in q[0]] == [o.uuid for o in q[1]]
    # a restart from an empty store replays each log into the same objects
    for name, kb in (("host", host), ("device", dev)):
        kb._wal.close()
        fresh = R.KnowledgeBase(HashEmbedder(32), capacity=4096, index_factory=OracleIndex)
        fresh.attach_wal(str(tmp_path / f"{name}.wal"))
        assert fresh._props == host._props and fresh.mutations == host.mutations
        fresh._wal.close()

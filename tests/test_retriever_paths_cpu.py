"""Characterisation of KnowledgeBase.query and query_batch over CPU doubles: for every way a request reaches an answer
(pure vector, tenant-scoped, unscoped, alpha <= 0, hybrid with the device keyword leg, fused on the device, filtered by
a device program, filtered by a host allow-list) the encoder, index and keyword-store calls each one makes, with their
arguments, and the answers it gives, held to ``tests/golden/retriever_paths.json``.

Three knowledge bases cover the paths: ``host`` (an index without device filters and the host ``BM25Index``), ``kw``
(device filter programs, and ``DeviceBM25`` over a store double, so the device keyword branches run) and ``fused`` (the
same, with hybrid queries fused on the device by a host emulation of ``engine.hybrid_search``).  Calls are recorded per
object; a batch of one makes the same calls as ``query``."""

from __future__ import annotations

import hashlib
import json
import os

import numpy as np
import pytest

from aurora_b200 import bm25
from aurora_b200 import retriever as R
from aurora_b200.filters import Filter, HybridFusion
from oracle import cosine_topk as O
from oracle.bm25_topk import bm25_topk
from tests.doubles import HashEmbedder, OracleIndex
from tests.keyword_mirror import Mirror

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "retriever_paths.json")
WORDS = ["disk", "oom", "pod", "latency", "timeout", "node", "memory", "cpu", "network", "failover", "kafka", "dns"]


def _digest(a):
    """An argument as JSON: arrays by shape, dtype and a hash of their bytes."""
    if a is None or isinstance(a, (bool, int, float, str)):
        return a
    if isinstance(a, (list, tuple)) and all(isinstance(x, (int, np.integer)) for x in a):
        return sorted(int(x) for x in a)            # an allow-list: a set of ids
    if isinstance(a, (list, tuple)):
        return [_digest(x) for x in a]
    if isinstance(a, np.ndarray):
        a = np.ascontiguousarray(a)
        return [list(a.shape), str(a.dtype), hashlib.sha1(a.tobytes()).hexdigest()[:16]]
    if isinstance(a, (np.integer, np.floating)):
        return a.item()
    raise TypeError(type(a))


def _program(prog):
    leaves, toks = prog
    return [[int(c), _digest(np.asarray(b, bool))] for c, b in leaves] + [" ".join(map(str, toks))]   # postfix order


class Encoder(HashEmbedder):
    def __init__(self, log):
        super().__init__(64)
        self.log = log

    def encode(self, texts):
        self.log.append(("enc", list(texts)))
        return super().encode(texts)


class Index(OracleIndex):
    """OracleIndex with list searches, attribute columns and filter programs evaluated on the host; records its calls."""

    def __init__(self, dim, capacity, log):
        super().__init__(dim, capacity)
        self.log, self.attrs = log, {}

    def _rec(self, name, *args):
        self.log.append(("ix", name, [_digest(a) for a in args]))

    def search(self, queries, k, q_user=None, q_org=None):
        self._rec("search", queries, k, q_user, q_org)
        return super().search(queries, k, q_user, q_org)

    def search_subset(self, queries, k, allow_ids):
        self._rec("search_subset", queries, k, allow_ids)
        return super().search_subset(queries, k, allow_ids)

    def search_lists(self, queries, k, lists, q_list):
        self._rec("search_lists", queries, k, list(lists), q_list)
        return self._topk(queries, k, [np.isin(self.ids, np.asarray(lists[l], np.int64)) for l in q_list])

    def _topk(self, queries, k, masks):
        q = O.round_to_bf16(np.asarray(queries, dtype=np.float32))
        ids = np.full((len(q), k), -1, np.int64)
        sc = np.full((len(q), k), -np.inf, np.float32)
        for i, m in enumerate(masks):
            ids[i], sc[i] = (a[0] for a in O.cosine_topk(q[i:i + 1], self.rows, k, ids=self.ids, live=self.live & m))
        return ids, sc


class FilterIndex(Index):
    dtype = R.AUR_BF16

    def set_attrs(self, col, ids, codes):
        self._rec("set_attrs", col, np.asarray(ids), np.asarray(codes))
        self.attrs.setdefault(col, {}).update(zip(np.asarray(ids).tolist(), np.asarray(codes).tolist()))

    def matches(self, prog):
        """The rows a program matches (the device's evaluation, as tests/test_filter_compile.py restates it)."""
        leaves, toks = prog
        cols = {0: self.user, 1: self.org}
        stack = []
        for t in toks:
            if t >= 0:
                col, bits = leaves[t]
                c = cols[col] if col in cols else np.array([self.attrs.get(col, {}).get(int(d), -1) for d in self.ids])
                idx = np.asarray(c, np.int64) + 1
                ok = (idx >= 0) & (idx < len(bits))
                v = np.zeros(len(self.ids), bool)
                v[ok] = np.asarray(bits, bool)[idx[ok]]
                stack.append(v)
            else:
                b, a = stack.pop(), stack.pop()
                stack.append(a & b if t == -1 else a | b)
        return stack[0]

    def search_filtered(self, queries, k, programs, q_program=None, max_list_rows=0):
        self._rec("search_filtered", queries, k, [_program(p) for p in programs], q_program, max_list_rows)
        ql = np.zeros(len(queries), np.int64) if q_program is None else q_program
        ids, sc = self._topk(queries, k, [self.matches(programs[p]) for p in ql])
        return ids, sc, None, 0

    def filter_ids(self, prog):
        self._rec("filter_ids", _program(prog))
        return self.ids[self.live & self.matches(prog)]


class Store:
    """KeywordIndex double: the rows as the device appends them, searched by the fp64 BM25 oracle."""

    def __init__(self, log):
        self.log, self.m = log, Mirror()

    def add(self, ids, terms, tfs, offsets, user=None, org=None):
        self.m.add(ids, terms, tfs, offsets, user, org)

    def remove(self, ids):
        self.m.remove(ids)
        return len(ids)

    def set_attrs(self, col, ids, codes):
        self.log.append(("kw", "set_attrs", [_digest(a) for a in (col, np.asarray(ids), np.asarray(codes))]))

    def topk(self, q_terms, q_off, k, q_user=None, q_org=None, allow_ids=None):
        ids, sc = bm25_topk(self.m.corpus(), q_terms, q_off, k, q_user, q_org, allow_ids)
        return ids, sc, None

    def search(self, q_terms, q_off, k, q_user=None, q_org=None, allow_ids=None):
        self.log.append(("kw", "search", [_digest(a) for a in (q_terms, q_off, k, q_user, q_org, allow_ids)]))
        return self.topk(q_terms, q_off, k, q_user, q_org, allow_ids)


class DeviceKeywords(bm25.DeviceBM25):
    """DeviceBM25 over the store double; its fused hybrid call is recorded and answered on the host."""

    def _run_hybrid(self, queries, fetch, q_user, q_org, index, vectors, w_dense, fusion, k_out, programs=None,
                    q_program=None, max_list_rows=0):
        self.store.log.append(("kw", "hybrid", [list(queries), fetch, _digest(q_user), _digest(q_org), _digest(vectors),
                                                _digest(np.asarray(w_dense)), fusion, k_out,
                                                None if programs is None else [_program(p) for p in programs],
                                                _digest(q_program), max_list_rows]))
        q_terms, q_off = bm25.query_csr(self.vocab, queries)
        out = []
        for q in range(len(queries)):
            terms, off = q_terms[q_off[q]:q_off[q + 1]], [0, q_off[q + 1] - q_off[q]]
            if programs is not None:
                mask = index.matches(programs[0 if q_program is None else q_program[q]])
                d_ids, d_sc = index._topk(vectors[q:q + 1], fetch, [mask])
                k_ids, k_sc, _ = self.store.topk(terms, off, fetch, allow_ids=index.ids[index.live & mask])
            else:
                u = None if q_user is None else q_user[q:q + 1]
                o = None if q_org is None else q_org[q:q + 1]
                d_ids, d_sc = OracleIndex.search(index, vectors[q:q + 1], fetch, u, o)
                k_ids, k_sc, _ = self.store.topk(terms, off, fetch, u, o)
            dense = [(int(d), float(s)) for d, s in zip(d_ids[0], d_sc[0]) if d >= 0]
            sparse = [(int(d), float(s)) for d, s in zip(k_ids[0], k_sc[0]) if d >= 0]
            w = float(w_dense[q])
            if fusion == R.FUSION_RELATIVE_SCORE:
                fused = bm25.relative_score_fusion([(w, dense), (1.0 - w, sparse)], k_out)
            else:
                fused = bm25.ranked_fusion([(w, [d for d, _ in dense]), (1.0 - w, [d for d, _ in sparse])], k_out)
            cos = dict(dense) if w > 0.0 else {}
            out.append([(d, (fs, cos.get(d))) for d, fs in fused])
        return out


class HostKeywords(bm25.BM25Index):
    def __init__(self, log):
        super().__init__()
        self.log = log

    def search(self, query, limit, allow=None, allowed=None, allowed_sorted=None):
        self.log.append(("kw", "search", [query, limit, _digest(None if allowed is None else list(allowed)),
                                          _digest(allowed_sorted)]))
        return super().search(query, limit, allow, allowed, allowed_sorted)


def _kb(kind):
    log = []
    cls = Index if kind == "host" else FilterIndex
    kb = R.KnowledgeBase(Encoder(log), capacity=8192, index_factory=lambda d, c: cls(d, c, log))
    if kind == "host":
        kb.sparse = HostKeywords(log)
    else:
        kb.sparse, kb._kw_device, kb._hybrid_device = DeviceKeywords(store=Store(log)), True, kind == "fused"
    r = np.random.default_rng(1)
    for t in range(40):
        for doc in range(2):
            chunks = [{"chunk_index": c, "content": " ".join(r.choice(WORDS, size=5))} for c in range(4)]
            kb.insert(f"u{t}", f"discovery:{t}" if doc == 0 else f"doc{t}", "f.md", chunks, org_id=f"o{t % 12}")
    # list values have no attribute code: filters on "labels" stay on the host everywhere
    kb.insert_objects([(f"lab{i}", {"user_id": "u1", "document_id": "lab", "chunk_index": i, "labels": ["a", f"b{i}"],
                                    "content": " ".join(r.choice(WORDS, size=5))}, " ".join(r.choice(WORDS, size=5)))
                       for i in range(6)], "u1")
    log.clear()
    return kb, log


def _res(objs):
    return [[o.uuid, o.metadata.score, o.metadata.distance] for o in objs]


def _streams(log):
    return {s: [list(e[1:]) for e in log if e[0] == s] for s in ("enc", "ix", "kw")}


DISC3 = Filter.by_property("org_id").equal("o3") & Filter.by_property("document_id").like("discovery:*")
ONE = Filter.by_property("document_id").equal("doc7") & Filter.by_property("chunk_index").equal(2)
LABELS = Filter.by_property("labels").equal(["a", "b2"])
NOBODY = Filter.by_property("org_id").equal("nobody")

# name -> (query, limit, keyword arguments of KnowledgeBase.query)
SINGLE = {
    "vector_unscoped": ("disk node", 7, {}),
    "vector_user": ("disk node", 5, dict(user_id="u3", scoped=True)),
    "vector_user_org": ("kafka dns", 9, dict(user_id="u3", org_id="o5", scoped=True)),
    "vector_org_only": ("oom pod", 4, dict(org_id="o2")),
    "vector_alpha_1": ("latency", 6, dict(user_id="u4", alpha=1.0, scoped=True)),
    "vector_unknown_user": ("disk", 5, dict(user_id="nobody")),
    "hybrid_unscoped": ("disk node timeout", 5, dict(alpha=0.5)),
    "hybrid_user": ("disk node timeout", 5, dict(user_id="u1", alpha=0.5, scoped=True)),
    "hybrid_user_org": ("memory cpu", 8, dict(user_id="u1", org_id="o7", alpha=0.3, scoped=True)),
    "hybrid_relative": ("memory cpu", 8, dict(user_id="u2", org_id="o7", alpha=0.6, scoped=True,
                                              fusion=HybridFusion.RELATIVE_SCORE)),
    "hybrid_alpha_0": ("kafka failover", 5, dict(user_id="u5", alpha=0.0, scoped=True)),
    "hybrid_alpha_neg_unscoped": ("kafka failover", 5, dict(alpha=-0.5)),
    "hybrid_fusion_none": ("dns network", 3, dict(user_id="u9", alpha=0.5, fusion=None)),
    "filter_vector": ("disk node", 10, dict(filters=DISC3)),
    "filter_vector_tenant": ("disk node", 10, dict(filters=DISC3, user_id="u3", org_id="o3", scoped=True)),
    "filter_hybrid": ("kafka dns", 10, dict(filters=DISC3, alpha=0.5)),
    "filter_hybrid_tenant_relative": ("kafka dns", 6, dict(filters=DISC3, user_id="u15", alpha=0.25,
                                                           fusion=HybridFusion.RELATIVE_SCORE, scoped=True)),
    "filter_hybrid_alpha_0": ("kafka dns", 6, dict(filters=DISC3, alpha=0.0)),
    "filter_one_row": ("disk", 5, dict(filters=ONE)),
    "filter_one_row_hybrid": ("disk", 5, dict(filters=ONE, alpha=0.5)),
    "filter_host_labels": ("oom", 5, dict(filters=LABELS)),
    "filter_host_labels_hybrid": ("oom", 5, dict(filters=LABELS, user_id="u1", alpha=0.5, scoped=True)),
    "filter_host_user_eq": ("oom memory", 5, dict(filters=Filter.by_property("user_id").equal("u1") | LABELS,
                                                  alpha=0.7)),
    "filter_empty": ("disk", 5, dict(filters=NOBODY)),
    "filter_empty_hybrid": ("disk", 5, dict(filters=NOBODY, alpha=0.5)),
    "filter_scoped_no_tenant": ("disk", 5, dict(filters=DISC3, scoped=True, alpha=0.5)),
    "limit_0": ("disk", 0, dict(alpha=0.5, user_id="u1")),
    "scoped_no_tenant": ("disk", 5, dict(alpha=0.5, scoped=True)),
}


def _batch(n_scopes):
    """A vector and a hybrid request for each of ``n_scopes`` tenant scopes (two result sizes, alpha 1, 0.5, 0.3, 0 and
    below), a limit past the fused list's length, and the requests that find nothing (limit 0, no tenant)."""
    rng = np.random.default_rng(n_scopes)
    reqs = []
    for t in range(n_scopes):
        u, o = f"u{t}", None if t % 3 else f"o{(t + 5) % 12}"
        reqs.append((u, " ".join(rng.choice(WORDS, size=3)), 3 if t % 7 == 3 else 6, None if t % 5 else 1.0, o))
        reqs.append((u, " ".join(rng.choice(WORDS, size=3)), 5 + t % 3, [0.5, 0.0, 0.3, -1.0][t % 4], o))
    if n_scopes > 1:
        reqs += [("u1", "disk", 6, None, None), ("u1", "disk oom", 300, 0.5, None), ("u1", "disk oom", 0, 0.5, None),
                 (None, "disk", 5, 0.5, None), ("", "disk", 5, None, None)]
    return reqs


BATCHES = {f"batch_{n}": n for n in (1, 31, 40)}


def _run_single(kind, name):
    q, lim, kw = SINGLE[name]
    kb, log = _kb(kind)
    return {"res": _res(kb.query(q, lim, **kw)), **_streams(log)}


def _run_batch(kind, name):
    kb, log = _kb(kind)
    return {"res": [_res(x) for x in kb.query_batch(_batch(BATCHES[name]))], **_streams(log)}


def _record():
    """Every case on every knowledge base: the golden file's contents (written with ``json.dump(_record(), f,
    separators=(",", ":"), sort_keys=True)``; rewrite it only for a change meant to alter the calls or the answers)."""
    out = {}
    for kind in ("host", "kw", "fused"):
        for name in SINGLE:
            out[f"{kind}/{name}"] = _run_single(kind, name)
        for name in BATCHES:
            out[f"{kind}/{name}"] = _run_batch(kind, name)
    return json.loads(json.dumps(out))


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN, encoding="utf-8") as f:
        return json.load(f)


@pytest.mark.parametrize("kind", ["host", "kw", "fused"])
@pytest.mark.parametrize("name", list(SINGLE))
def test_single_request_calls_and_answer(golden, kind, name):
    assert json.loads(json.dumps(_run_single(kind, name))) == golden[f"{kind}/{name}"]


@pytest.mark.parametrize("kind", ["host", "kw", "fused"])
@pytest.mark.parametrize("name", list(BATCHES))
def test_batch_calls_and_answers(golden, kind, name):
    assert json.loads(json.dumps(_run_batch(kind, name))) == golden[f"{kind}/{name}"]


@pytest.mark.parametrize("kind", ["host", "kw", "fused"])
def test_batch_of_one_is_query(kind):
    """query_batch([(u, q, lim, a, o)])[0] is query(q, lim, user_id=u, org_id=o, alpha=a, scoped=True): same answer,
    same calls on the encoder, the index and the keyword store."""
    kb, log = _kb(kind)
    reqs = _batch(40) + [("u2", "disk", 5, -1.0, "o3"), ("u7", "kafka", 200, 0.5, None), ("u7", "kafka", 200, None, None)]
    for u, q, lim, a, o in reqs:
        log.clear()
        one = _res(kb.query(q, lim, user_id=u, org_id=o, alpha=a, scoped=True))
        single = _streams(log)
        log.clear()
        batch = _res(kb.query_batch([(u, q, lim, a, o)])[0])
        assert batch == one and _streams(log) == single, (u, q, lim, a, o)


def test_the_cases_reach_every_path():
    """The table above exercises each entry point it is meant to (a guard on the characterisation itself)."""
    with open(GOLDEN, encoding="utf-8") as f:
        g = json.load(f)
    seen = {(k.split("/")[0], e[0]) for k, v in g.items() for s in ("ix", "kw") for e in v[s]}
    assert {("host", n) for n in ("search", "search_subset", "search_lists")} <= seen
    assert {("kw", n) for n in ("search", "search_filtered", "filter_ids", "set_attrs", "search_lists")} <= seen
    assert {("fused", n) for n in ("hybrid", "search", "search_lists", "search_filtered")} <= seen
    assert not g["host/filter_empty"]["ix"] and not g["kw/limit_0"]["enc"] and not g["fused/scoped_no_tenant"]["kw"]
    # more than 32 scopes: the hybrid requests take the two legs, and the largest vector group one list search
    assert [e[0] for e in g["fused/batch_31"]["kw"]] == ["hybrid"]
    assert [e[0] for e in g["fused/batch_40"]["kw"]] == ["search"]
    assert "search_lists" in [e[0] for e in g["fused/batch_40"]["ix"]]
    assert "search_lists" not in [e[0] for e in g["fused/batch_31"]["ix"]]

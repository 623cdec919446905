"""Host logic of the retriever's list searches, over CPU doubles: which index entry point a filtered query and a batch of
many tenant scopes take, and the lists they build."""

from __future__ import annotations

import numpy as np

from aurora_b200 import retriever as R
from aurora_b200.engine import lists_csr
from aurora_b200.filters import Filter
from oracle import cosine_topk as O
from tests.doubles import HashEmbedder, OracleIndex

WORDS = ["disk", "oom", "pod", "latency", "timeout", "node", "memory", "cpu", "network", "failover", "kafka", "dns"]


class RecordingIndex(OracleIndex):
    """OracleIndex that records its search calls."""

    def __init__(self, dim, capacity):
        super().__init__(dim, capacity)
        self.calls = []

    def search(self, queries, k, q_user=None, q_org=None):
        self.calls.append(("search", len(queries)))
        return super().search(queries, k, q_user, q_org)

    def search_subset(self, queries, k, allow_ids):
        self.calls.append(("search_subset", len(allow_ids)))
        return super().search_subset(queries, k, allow_ids)


class ListOracleIndex(RecordingIndex):
    """RecordingIndex with ``search_lists``: query q over the live rows whose ids are in lists[q_list[q]]."""

    def search_lists(self, queries, k, lists, q_list):
        self.calls.append(("search_lists", [np.asarray(a).copy() for a in lists], np.asarray(q_list).copy()))
        q = O.round_to_bf16(np.asarray(queries, dtype=np.float32))
        ids = np.full((len(q), k), -1, np.int64)
        sc = np.full((len(q), k), -np.inf, np.float32)
        for i, l in enumerate(q_list):
            live = self.live & np.isin(self.ids, np.asarray(lists[l], dtype=np.int64))
            ids[i], sc[i] = (a[0] for a in O.cosine_topk(q[i:i + 1], self.rows, k, ids=self.ids, live=live))
        return ids, sc


def _kb(index_cls):
    kb = R.KnowledgeBase(HashEmbedder(64), capacity=8192, index_factory=lambda d, c: index_cls(d, c))
    r = np.random.default_rng(1)
    for t in range(40):
        for doc in range(2):
            chunks = [{"chunk_index": c, "content": " ".join(r.choice(WORDS, size=5))} for c in range(4)]
            kb.insert(f"u{t}", f"discovery:{t}" if doc == 0 else f"doc{t}", "f.md", chunks, org_id=f"o{t % 12}")
    return kb


def _shape(objs):
    return [(o.uuid, round(o.metadata.score, 6)) for o in objs]


def _reqs(n_scopes):
    rng = np.random.default_rng(n_scopes)
    return [(f"u{t}", " ".join(rng.choice(WORDS, size=3)), 6, None, None if t % 3 else f"o{(t + 5) % 12}")
            for t in range(n_scopes)] + [("u1", "disk", 6, None, None)]


def test_more_than_32_scopes_run_as_one_list_search_of_the_tenants_rows():
    lists_kb, plain_kb = _kb(ListOracleIndex), _kb(RecordingIndex)
    reqs = _reqs(40)
    lists_kb.index.calls.clear()
    got = lists_kb.query_batch(reqs)
    assert [_shape(x) for x in got] == [_shape(x) for x in plain_kb.query_batch(reqs)]
    calls = [c for c in lists_kb.index.calls if c[0] != "search"]
    assert len(calls) == 1 and calls[0][0] == "search_lists"
    _, lists, q_list = calls[0]
    assert len(lists) == 40 and len(q_list) == len(reqs)       # ("u1", no org) is asked twice: one list
    assert q_list[1] == q_list[-1]
    with lists_kb._lock:
        for (u, _, _, _, o), l in zip(reqs, q_list):
            want = lists_kb._by_user.get(u, set()) | (lists_kb._by_org.get(o, set()) if o else set())
            assert set(lists[l].tolist()) == want and np.all(np.diff(lists[l]) > 0)
    assert not any(c[0] == "search" for c in lists_kb.index.calls)


def test_32_scopes_or_fewer_keep_the_masked_search():
    kb = _kb(ListOracleIndex)
    kb.index.calls.clear()
    kb.query_batch(_reqs(32)[:-1])
    assert [c[0] for c in kb.index.calls] == ["search"]


def test_filtered_query_uses_search_lists_when_the_index_has_it(monkeypatch):
    monkeypatch.setattr(R, "_LIST_MAX_FRACTION", 0.06)          # the filters below allow 16 of 320 objects (5 %)
    lists_kb, plain_kb = _kb(ListOracleIndex), _kb(RecordingIndex)
    for kb in (lists_kb, plain_kb):
        kb.index.calls.clear()
    for o in ("o3", "o7"):
        flt = Filter.by_property("org_id").equal(o) & Filter.by_property("document_id").like("discovery:*")
        for q in ("disk node", "kafka dns"):
            assert _shape(lists_kb.query(q, 10, filters=flt)) == _shape(plain_kb.query(q, 10, filters=flt))
    assert {c[0] for c in lists_kb.index.calls} == {"search_lists"}
    assert {c[0] for c in plain_kb.index.calls} == {"search_subset"}           # fallback: no search_lists
    call = lists_kb.index.calls[0]
    assert len(call[1]) == 1 and list(call[2]) == [0]


def test_filter_above_the_list_fraction_keeps_search_subset(monkeypatch):
    kb = _kb(ListOracleIndex)
    flt = Filter.by_property("org_id").equal("o3") & Filter.by_property("document_id").like("discovery:*")
    for frac, want in ((0.04, "search_subset"), (0.05, "search_lists")):   # 16 allowed of 320 objects
        monkeypatch.setattr(R, "_LIST_MAX_FRACTION", frac)
        kb.index.calls.clear()
        kb.query("disk node", 10, filters=flt)
        assert [c[0] for c in kb.index.calls] == [want]


def test_empty_filter_makes_no_device_call():
    for cls in (ListOracleIndex, RecordingIndex):
        kb = _kb(cls)
        kb.index.calls.clear()
        assert kb.query("disk", 5, filters=Filter.by_property("org_id").equal("nobody")) == []
        assert kb.index.calls == []


def test_lists_csr():
    flat, off = lists_csr([np.array([5, 6]), [], np.array([7])])
    assert off.tolist() == [0, 2, 2, 3] and flat[:3].tolist() == [5, 6, 7]
    flat, off = lists_csr([[]])
    assert off.tolist() == [0, 0] and len(flat) >= 1

"""The alert-correlation mirror (aurora_b200/correlation.py) and its daemon operations, on the CPU: ``score`` against the
reference's own results, ``score_many`` / ``score_alerts`` against ``score`` over a client double, and the daemon's
embed / embed_batch / similarity_scores round trip with its coalescing and its unreachable-daemon fallback."""

import json
import os
import shutil
import tempfile
import threading

import numpy as np
import pytest

from aurora_b200 import correlation as K
from aurora_b200 import encoder as E
from aurora_b200 import retriever as R
from aurora_b200.correlation import SimilarityStrategy
from aurora_b200.daemon import Client, serve
from tests.doubles import HashEmbedder, OracleIndex

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


class TableClient:
    """embed from a table (None for a text it does not hold), as the reference's tests mock the client."""

    def __init__(self, table):
        self.table = table

    def embed(self, text):
        return self.table.get(text)


class VectorClient:
    """EmbeddingClient double: hashed bag-of-words vectors (fp32, as the encoder returns them); None for blank text and
    for texts containing "novec".  ``similarities`` is numpy fp64 over the same vectors, clamped."""

    def __init__(self, dim=64):
        self.h = HashEmbedder(dim)
        self.similarity_calls = []

    def _vec(self, text):
        if not text or not text.strip() or "novec" in text:
            return None
        return self.h.encode([text])[0]

    def embed(self, text):
        v = self._vec(text)
        return None if v is None else v.tolist()

    def embed_batch(self, texts):
        return [self.embed(t) for t in texts]

    def similarities(self, pairs):
        self.similarity_calls.append(list(pairs))
        out = []
        for a, b in pairs:
            va, vb = self._vec(a), self._vec(b)
            if va is None or vb is None:
                out.append(None)
                continue
            x, y = va.astype(np.float64), vb.astype(np.float64)
            den = np.sqrt(x @ x) * np.sqrt(y @ y)
            out.append(float(min(1.0, max(0.0, (x @ y) / den))) if den > 0 else 0.0)
        return out


@pytest.fixture()
def client(monkeypatch):
    c = VectorClient()
    monkeypatch.setattr(K, "get_embedding_client", lambda: c)
    return c


def test_score_equals_the_reference_on_every_golden_case(monkeypatch):
    cases = json.load(open(os.path.join(GOLDEN, "similarity_ref.json")))["cases"]
    assert len(cases) >= 50
    kinds = {"vectors": 0, "fallback": 0, "blank": 0}
    for c in cases:
        table = {c["alert_title"]: c["vec_alert"], c["incident_title"]: c["vec_incident"]}
        monkeypatch.setattr(K, "get_embedding_client", lambda: TableClient(table))
        got = SimilarityStrategy().score(c["alert_title"], c["alert_service"], c["incident_title"], c["incident_services"])
        assert got == c["score"], c
        kinds["blank" if not c["alert_title"] or not c["incident_title"] else
              "fallback" if c["vec_alert"] is None or c["vec_incident"] is None else "vectors"] += 1
    assert all(kinds.values()), kinds
    for c in json.load(open(os.path.join(GOLDEN, "cosine_ref.json")))["score_weighting"]:
        table = {"alert title": c["vec_a"], "incident title": c["vec_b"]}
        monkeypatch.setattr(K, "get_embedding_client", lambda: TableClient(table))
        assert SimilarityStrategy().score("alert title", c["alert_service"], "incident title", c["incident_services"]) == c["score"]


def test_a_failing_client_falls_back_to_jaccard(monkeypatch):
    def down():
        raise RuntimeError("no encoder")

    monkeypatch.setattr(K, "get_embedding_client", down)
    s = SimilarityStrategy()
    want = 0.7 * s._jaccard_similarity("redis down on db-1", "redis db-1 unreachable") + 0.3 * 1.0
    assert s.score("redis down on db-1", "redis", "redis db-1 unreachable", ["redis"]) == want
    assert s.score_many("redis down on db-1", "redis", [("redis db-1 unreachable", ["redis"])]) == [want]


ALERTS = [
    ("High CPU usage on api-server", "api-server", [("API server CPU high", ["api-server"]), ("Disk full on node-3", ["node"]),
                                                    ("novec kafka lag", ["kafka"]), ("", ["api-server"]), ("   ", []),
                                                    ("API server CPU high", ["web", "api-gateway"])]),
    ("Payment 5xx errors", "payment-service", [("Payment service 5xx", ["payment-service"]), ("payment 5xx errors", None)]),
    ("", "svc", [("anything", ["svc"])]),
    ("novec title", "svc", [("svc title", ["svc"]), ("other", [])]),
    ("Café latency über p99", "café", [("cafe latency uber p99", ["café"]), ("Café latency über p99", ["café"])]),
    ("zero candidates", "svc", []),
]


def test_score_many_and_score_alerts_equal_score_per_candidate(client):
    s = SimilarityStrategy()
    want = [[s.score(t, svc, c[0], c[1]) for c in cands] for t, svc, cands in ALERTS]
    got = s.score_alerts(ALERTS)
    assert len(client.similarity_calls) == 1                          # every alert's pairs in one call
    assert [p for p in client.similarity_calls[0] if not p[0] or not p[1]] == []   # empty titles never sent
    assert [len(r) for r in got] == [len(r) for r in want]
    for g, w in zip(sum(got, []), sum(want, [])):
        assert abs(g - w) <= 1e-12, (g, w)
    client.similarity_calls.clear()
    for (t, svc, cands), w in zip(ALERTS, want):
        g = s.score_many(t, svc, cands)
        assert len(g) == len(w) and all(abs(a - b) <= 1e-12 for a, b in zip(g, w))
    assert len(client.similarity_calls) == sum(1 for t, _, cands in ALERTS if t and any(c[0] for c in cands))
    assert s.score_alerts([]) == [] and s.score_many("t", "s", []) == []


def test_none_pairs_take_jaccard_and_failures_take_it_everywhere(client, monkeypatch):
    s = SimilarityStrategy()
    got = s.score_many("novec alert on redis", "redis", [("redis alert", ["redis"]), ("redis alert", ["redis"])])
    want = 0.7 * s._jaccard_similarity("novec alert on redis", "redis alert") + 0.3
    assert got == [want, want]                                          # duplicate titles, the same value
    monkeypatch.setattr(client, "similarities", lambda pairs: (_ for _ in ()).throw(RuntimeError("device lost")))
    got = s.score_many("High CPU usage", "api", [("CPU usage high", ["api"])])
    assert got == [0.7 * s._jaccard_similarity("High CPU usage", "CPU usage high") + 0.3]


def test_a_client_without_similarities_is_scored_pair_by_pair(monkeypatch):
    c = VectorClient()
    monkeypatch.setattr(K, "get_embedding_client", lambda: TableClient({t: c.embed(t) for t in
                                                                        ("High CPU usage on api-server", "API server CPU high")}))
    s = SimilarityStrategy()
    got = s.score_many("High CPU usage on api-server", "api-server", [("API server CPU high", ["api-server"]), ("", [])])
    assert got == [s.score("High CPU usage on api-server", "api-server", "API server CPU high", ["api-server"]), 0.0]


# ---------------------------------------------------------------------- daemon
@pytest.fixture()
def sock_dir():
    d = tempfile.mkdtemp(prefix="aur-", dir="/tmp" if os.path.isdir("/tmp") else None)
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture()
def served(sock_dir):
    c = VectorClient()
    E.configure_embedding_client(lambda: c)
    R.configure(encoder=HashEmbedder(64), capacity=64, index_factory=lambda dim, cap: OracleIndex(dim, cap))
    path = os.path.join(sock_dir, "kb.sock")
    srv = serve(path, background=True, coalesce_us=200000)
    yield path, c
    srv.shutdown(); srv.close_all(final_save=False); srv.server_close()
    E._factory = None
    E.get_embedding_client.cache_clear()
    R.configure(factory=lambda: (_ for _ in ()).throw(RuntimeError("backend down")))


def test_daemon_embed_and_similarity_scores_round_trip(served):
    """The daemon answers with its own embedding client (encoder.configure_embedding_client in its process)."""
    path, local = served
    kb = Client(path)
    assert kb.embed("redis failover") == local.embed("redis failover")
    assert kb.embed("  ") is None and kb.embed("novec") is None
    assert kb.embed_batch(["a b", "", "novec x"]) == [local.embed("a b"), None, None]
    got = kb.similarity_scores(ALERTS)
    assert len(local.similarity_calls) == 1
    assert got == SimilarityStrategy().score_alerts(ALERTS)


def test_concurrent_similarity_scores_share_one_similarities_call(served):
    path, local = served
    results, errs, go = {}, [], threading.Barrier(2)

    def worker(i):
        try:
            c = Client(path)
            go.wait()
            results[i] = c.similarity_scores([ALERTS[i]])
        except Exception as e:      # pragma: no cover
            errs.append(e)

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errs, errs
    assert len(local.similarity_calls) == 1                              # two alerts, one device call
    s = SimilarityStrategy()
    for i in range(2):
        t, svc, cands = ALERTS[i]
        want = [s.score(t, svc, c[0], c[1]) for c in cands]
        assert len(results[i]) == 1 and len(results[i][0]) == len(cands)
        assert all(abs(g - w) <= 1e-12 for g, w in zip(results[i][0], want))


def test_daemon_down_gives_jaccard_scores_and_no_embeddings(sock_dir, monkeypatch):
    kb = Client(os.path.join(sock_dir, "nobody.sock"))
    assert kb.embed("redis failover") is None and kb.embed_batch(["a", "b"]) == [None, None]
    monkeypatch.setattr(K, "get_embedding_client", lambda: TableClient({}))   # what `score` sees when embed gives None
    s = SimilarityStrategy()
    want = [[s.score(t, svc, c[0], c[1]) for c in cands] for t, svc, cands in ALERTS]
    assert kb.similarity_scores(ALERTS) == want
    monkeypatch.setattr(K, "get_embedding_client", lambda: kb)
    assert s.score_alerts(ALERTS) == want

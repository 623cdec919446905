#!/usr/bin/env python
"""Generate tests/golden/similarity_ref.json by running the REAL reference ``SimilarityStrategy.score``.

Run in the authoring container only (``/root/reference`` does not exist on the GPU box):
``python oracle/gen_golden_similarity.py``.  The output is committed; nothing at test time reads the reference.

The embedding client is mocked as ``oracle/gen_golden.py`` mocks it for ``score_weighting`` (the reference's own test
technique, test_similarity_strategy.py:16-65): ``embed`` answers from a table of vectors, None for a text it does not
hold, so a case covers the vector path, the Jaccard fallback, or both (one title embedded, the other not).

Cases: vectors present and missing, stop-words and one-character words in the titles, exact / partial / disjoint /
empty / missing services, empty and whitespace-only titles, non-ASCII text.  Every case records the arguments of
``score``, the vectors ``embed`` returned for each title (null for None) and the reference's result.
"""

from __future__ import annotations

import json
import os
import sys
from unittest.mock import MagicMock, patch

import numpy as np

sys.dont_write_bytecode = True
REF = "/root/reference/server"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "similarity_ref.json")


def main() -> None:
    sys.path.insert(0, REF)
    from services.correlation.strategies.similarity import SimilarityStrategy  # noqa: E402

    rng = np.random.default_rng(20261019)
    titles = ["High CPU usage on api-server", "API server CPU is high at the edge", "Disk pressure on node a",
              "The a an is are was for in on at", "x y z 1 2", "Café latency über p99 — ошибка", "cafe latency uber p99",
              "payment-service 5xx errors", "Payment service returning 5xx", "   ", "", "kafka consumer lag", "b"]
    vecs = {t: [float(x) for x in rng.standard_normal(8).astype(np.float32)] for t in titles if t.strip()}
    vecs["kafka consumer lag"] = [0.0] * 8                                        # a zero vector: cosine 0.0
    vecs["Payment service returning 5xx"] = [-x for x in vecs["payment-service 5xx errors"]]   # opposite: clamped to 0
    missing = {"Disk pressure on node a", "x y z 1 2"}                          # embed gives None: Jaccard fallback
    services = [("api-server", ["api-server"]), ("api-server", ["api-gateway", "web"]), ("payment-service", ["billing"]),
                ("", ["api-server"]), ("api-server", []), ("api-server", None), ("the-a-x", ["at-on-y"]),
                ("Café-svc", ["café-svc"]), ("café svc", ["svc-café"])]
    strat = SimilarityStrategy()
    cases = []
    for i, a in enumerate(titles):
        for j, b in enumerate(titles):
            if (i * 7 + j * 3) % 4 and not (a.strip() == "" or b.strip() == "" or i == j):
                continue
            svc, inc = services[(i + 2 * j) % len(services)]
            table = {t: (None if t in missing else vecs.get(t)) for t in (a, b)}
            with patch("services.correlation.strategies.similarity.get_embedding_client") as g:
                client = MagicMock()
                client.embed.side_effect = lambda text: table.get(text)
                g.return_value = client
                val = strat.score(a, svc, b, inc)
            cases.append({"alert_title": a, "alert_service": svc, "incident_title": b, "incident_services": inc,
                          "vec_alert": table[a], "vec_incident": table[b], "score": val})
    with open(OUT, "w") as f:
        json.dump({"generator": "oracle/gen_golden_similarity.py", "reference_commit": "e907d997",
                   "python": sys.version.split()[0], "cases": cases}, f, ensure_ascii=False)
    print("wrote", OUT, f"({len(cases)} cases)")


if __name__ == "__main__":
    main()

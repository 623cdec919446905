"""The hybrid query's last stage on the GPU: the fused call against the host-fused pipeline, one JSON line.

Setup: 1M documents (default) with seeded 768-d bf16 vectors in an engine.Index and hybrid_bench.py's synthetic texts
(~250 Zipf words over a 50k vocabulary) in a bm25.DeviceBM25 over an engine.KeywordIndex on the same GPU, every row with
one of 64 tenant codes; 256 hybrid requests (alpha 0.5, limit 5) scoped to 16 of those tenants, and also nq = 1.

  host    the pipeline before device fusion, composed from unchanged pieces: Index.search (dense leg, top-128) +
          DeviceBM25.search_batch (keyword leg, top-128) + per-request bm25.ranked_fusion + result shaping;
  fused   DeviceBM25.search_batch with ``dense`` (engine.hybrid_search: both legs and the fusion in one device call,
          top-5 back) + the same shaping.

Both run on the same inputs, alternated, --reps times after --warmup; reported are median wall ms per batch and each
leg's device ms (aur_stats.last_total_ms of the dense leg, aur_kw_stats.last_ms of the keyword leg: the CUDA events
around each leg; in the fused call the two legs overlap and the fusion kernel is not inside either).  Parity, checked in
the same run: the fused lists (ids, fp64 scores, cosines) of every request must be bit-identical to the host pipeline's,
at limit 5 and at the full 256; the run fails otherwise.  The card's name and power limit are read in the same run.

    python tools/fusion_bench.py [--docs 1000000] [--reps 20] [--warmup 3]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aurora_b200 import _native as N  # noqa: E402
from aurora_b200 import bm25  # noqa: E402
from aurora_b200.engine import Index, KeywordIndex  # noqa: E402
from hybrid_bench import card, corpus, queries  # noqa: E402

DIM, FETCH, LIMIT = 768, 128, 5
PROPS = {"content": "x", "heading_context": "", "source_filename": "f", "document_id": "d", "chunk_index": 0}


def shape(picked):
    """The retriever's result objects and search_knowledge_base's dicts for one request."""
    objs = [SimpleNamespace(properties=dict(PROPS), uuid=None,
                            metadata=SimpleNamespace(score=float(s), distance=None if c is None else 1.0 - float(c)))
            for _, s, c in picked]
    return [{"content": o.properties["content"], "score": o.metadata.score} for o in objs]


def host_pipeline(ix, kw, vecs, texts, q_user, q_org, limit):
    """What query_batch did before device fusion: two device legs, then fusion and shaping per request on the host."""
    ids, scores = ix.search(vecs, FETCH, q_user, q_org)
    lists = kw.search_batch(texts, FETCH, q_user, q_org)
    out, res = [], []
    for q in range(len(texts)):
        dense = [(int(r), float(s)) for r, s in zip(ids[q], scores[q]) if r >= 0]
        cos = dict(dense)
        fused = bm25.ranked_fusion([(0.5, [d for d, _ in dense]), (0.5, [d for d, _ in lists[q]])], limit)
        picked = [(r, fs, cos.get(r)) for r, fs in fused]
        out.append(picked)
        res.append(shape(picked))
    return out


def fused_pipeline(ix, kw, vecs, texts, q_user, q_org, limit):
    lists = kw.search_batch(texts, FETCH, q_user, q_org,
                            dense=(ix, vecs, np.full(len(texts), 0.5), N.FUSION_RANKED, limit))
    out, res = [], []
    for lst in lists:
        picked = [(r, fs, c) for r, (fs, c) in lst][:limit]
        out.append(picked)
        res.append(shape(picked))
    return out


def same(a, b):
    """Bit-identical fused lists: ids, fp64 scores, cosines (None for ids the dense list does not hold)."""
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if len(x) != len(y):
            return False
        for (i1, s1, c1), (i2, s2, c2) in zip(x, y):
            if i1 != i2 or np.float64(s1).view(np.int64) != np.float64(s2).view(np.int64):
                return False
            if (c1 is None) != (c2 is None) or (c1 is not None and np.float32(c1).view(np.int32) != np.float32(c2).view(np.int32)):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=250)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    t0 = time.perf_counter()
    terms, tfs, offsets = corpus(rng, args.docs, args.tokens, args.vocab)
    qt, qo = queries(rng, 256, args.vocab)
    texts = [" ".join(f"t{t}" for t in qt[qo[q]:qo[q + 1]]) for q in range(256)]
    ids = np.arange(args.docs, dtype=np.int64) * 3 + 1
    users = rng.integers(0, 64, args.docs).astype(np.int32)
    orgs = np.full(args.docs, -1, np.int32)
    ix = Index(DIM, args.docs)
    store = KeywordIndex(args.docs, postings_capacity=len(terms))
    step = 100_000
    for d0 in range(0, args.docs, step):
        d1 = min(args.docs, d0 + step)
        ix.add(rng.standard_normal((d1 - d0, DIM), dtype=np.float32), ids[d0:d1], users[d0:d1], orgs[d0:d1])
        sl = slice(offsets[d0], offsets[d1])
        store.add(ids[d0:d1], terms[sl], tfs[sl], offsets[d0:d1 + 1] - offsets[d0], users[d0:d1], orgs[d0:d1])
    kw = bm25.DeviceBM25(store=store)
    kw.vocab = {f"t{i}": i for i in range(args.vocab)}          # the synthetic texts' words are "t<term id>"
    kw._docs = set(ids.tolist())
    setup_s = time.perf_counter() - t0
    vecs = rng.standard_normal((256, DIM), dtype=np.float32)
    q_user = rng.integers(0, 16, 256).astype(np.int32)            # 16 tenants: <= 32 scopes, one tensor-core launch
    q_org = np.full(256, -1, np.int32)

    result = {"docs": args.docs, "dim": DIM, "mean_tokens": args.tokens, "vocab": args.vocab, "postings": int(len(terms)),
              "fetch": FETCH, "limit": LIMIT, "tenants": 16, "setup_s": round(setup_s, 1)}
    ok = True
    for nq in (256, 1):
        a = (ix, kw, vecs[:nq], texts[:nq], q_user[:nq], q_org[:nq])
        for limit in (LIMIT, 2 * FETCH):
            ok &= same(host_pipeline(*a, limit), fused_pipeline(*a, limit))
        for _ in range(args.warmup):
            host_pipeline(*a, LIMIT)
            fused_pipeline(*a, LIMIT)
        wall = {"host": [], "fused": []}
        dev = {"host": [], "fused": []}
        for _ in range(args.reps):
            for name, fn in (("host", host_pipeline), ("fused", fused_pipeline)):
                w0 = time.perf_counter()
                fn(*a, LIMIT)
                wall[name].append((time.perf_counter() - w0) * 1e3)
                dev[name].append((ix.stats()["last_total_ms"], store.stats()["last_ms"]))
        row = {}
        for name in ("host", "fused"):
            d = np.median(np.asarray(dev[name]), axis=0)
            row[name] = {"wall_ms": round(float(np.median(wall[name])), 3), "wall_ms_min": round(float(np.min(wall[name])), 3),
                         "dense_leg_device_ms": round(float(d[0]), 3), "keyword_leg_device_ms": round(float(d[1]), 3)}
        row["wall_speedup"] = round(row["host"]["wall_ms"] / row["fused"]["wall_ms"], 3)
        result[f"nq{nq}"] = row
    result["parity"] = bool(ok)
    name, power = card()
    result["card"] = name
    result["power_limit"] = power
    print(json.dumps(result), flush=True)
    ix.close()
    store.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()

"""The hybrid query over a multi-GPU knowledge base: the fused multi-shard call against the host-fused pipeline, one
JSON line.

Setup: tools/fusion_bench.py's corpus (1M documents by default, seeded 768-d bf16 vectors, hybrid_bench.py's synthetic
texts, 64 tenant codes) in an engine.MultiIndex and a bm25.DeviceBM25 over an engine.MultiKeywordIndex with one shard
and one keyword store per visible GPU (documents placed by id mod n).  On a one-GPU machine both run 2 shards on device
0 (the line's "devices" says so).  256 hybrid requests (alpha 0.5, limit 5) scoped to 16 tenants, and also nq = 1.

  host    MultiIndex.search (every shard's top-128, merged on the host) + DeviceBM25.search_batch (every store's
          top-128, merged on the host) + per-request bm25.ranked_fusion + result shaping;
  fused   DeviceBM25.search_batch with ``dense`` (engine.hybrid_search -> aur_hybrid_search_multi: every leg, the
          merges and the fusion in one device call, top-5 back) + the same shaping.

Both run on the same inputs, alternated, --reps times after --warmup; reported are median wall ms per batch and each
leg's device ms, the largest over the shards / stores (aur_stats.last_total_ms of the dense legs, aur_kw_stats.last_ms
of the keyword legs).  Parity, checked in the same run: the fused lists (ids, fp64 scores, cosines) of every request
must be bit-identical to the host pipeline's, at limit 5 and at the full 256; the run fails otherwise.  The card's
name, the GPU count and the power limit are read in the same run.

    python tools/fusion_multi_bench.py [--docs 1000000] [--reps 20] [--warmup 3]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aurora_b200 import _native as N  # noqa: E402
from aurora_b200 import bm25  # noqa: E402
from aurora_b200.engine import MultiIndex, MultiKeywordIndex  # noqa: E402
from fusion_bench import DIM, FETCH, LIMIT, fused_pipeline, host_pipeline, same  # noqa: E402
from hybrid_bench import card, corpus, queries  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=250)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    gpus = N.load().aur_device_count()
    devices = list(range(gpus)) if gpus > 1 else [0, 0]
    rng = np.random.default_rng(args.seed)
    t0 = time.perf_counter()
    terms, tfs, offsets = corpus(rng, args.docs, args.tokens, args.vocab)
    qt, qo = queries(rng, 256, args.vocab)
    texts = [" ".join(f"t{t}" for t in qt[qo[q]:qo[q + 1]]) for q in range(256)]
    ids = np.arange(args.docs, dtype=np.int64) * 3 + 1
    users = rng.integers(0, 64, args.docs).astype(np.int32)
    orgs = np.full(args.docs, -1, np.int32)
    mi = MultiIndex(DIM, args.docs, devices=devices)
    store = MultiKeywordIndex(args.docs, devices=devices, postings_capacity=len(terms))
    step = 100_000
    for d0 in range(0, args.docs, step):
        d1 = min(args.docs, d0 + step)
        mi.add(rng.standard_normal((d1 - d0, DIM), dtype=np.float32), ids[d0:d1], users[d0:d1], orgs[d0:d1])
        sl = slice(offsets[d0], offsets[d1])
        store.add(ids[d0:d1], terms[sl], tfs[sl], offsets[d0:d1 + 1] - offsets[d0], users[d0:d1], orgs[d0:d1])
    kw = bm25.DeviceBM25(store=store)
    kw.vocab = {f"t{i}": i for i in range(args.vocab)}          # the synthetic texts' words are "t<term id>"
    kw._docs = set(ids.tolist())
    setup_s = time.perf_counter() - t0
    vecs = rng.standard_normal((256, DIM), dtype=np.float32)
    q_user = rng.integers(0, 16, 256).astype(np.int32)            # 16 tenants: <= 32 scopes, one tensor-core launch
    q_org = np.full(256, -1, np.int32)

    def leg_ms():
        return (max(sh.stats()["last_total_ms"] for sh in mi.shards), max(s["last_ms"] for s in store.stats()["stores"]))

    result = {"devices": devices, "gpus": gpus, "docs": args.docs, "dim": DIM, "mean_tokens": args.tokens,
              "vocab": args.vocab, "postings": int(len(terms)), "fetch": FETCH, "limit": LIMIT, "tenants": 16,
              "setup_s": round(setup_s, 1)}
    ok = True
    for nq in (256, 1):
        a = (mi, kw, vecs[:nq], texts[:nq], q_user[:nq], q_org[:nq])
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
                dev[name].append(leg_ms())
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
    mi.close()
    store.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()

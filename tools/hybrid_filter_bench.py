"""The filtered hybrid query as one device call against the host pipeline it replaces, one JSON line.

Setup: fusion_bench.py's corpus -- 1M documents (default) with seeded 768-d bf16 vectors in an engine.Index and
hybrid_bench.py's synthetic Zipf texts in a bm25.DeviceBM25 over an engine.KeywordIndex on the same GPU -- with
filter_bench.py's metadata: disjoint orgs of 1k, 10k and 100k rows at the front, the remaining rows in 61 more orgs,
every other row under a "discovery:" document id, a "tier" property every row shares (the 1M "org").  The attribute
columns are set on both stores, as retriever.KnowledgeBase keeps them.  The filter is the prediscovery call's
`org_id == o AND document_id LIKE "discovery:*"` (rca_prompt_builder.py:286-298), alpha 0.5, ranked fusion, limit 3.

  host    the parent's filtered pipeline, composed from unchanged pieces: Index.search_filtered (dense leg, top-128, the
          retriever's list-vs-scan rule) + Index.filter_ids (every matching id to the host) + DeviceBM25.search with
          those ids as its allow-list (keyword leg, top-128) + bm25.ranked_fusion + shaping, once per request;
  fused   DeviceBM25.search_batch with ``dense`` and ``programs`` (engine.hybrid_search: both legs evaluate the program on
          the GPU, fused there) + the same shaping.

Workloads: one request (nq = 1) per org size 1k / 10k / 100k / 1M, and nq = 256 requests over the 64 orgs (the host
arm then answers 256 single requests: the parent has no batched filtered form).  Arms alternated, --reps times after
--warmup; reported are the median wall ms per workload and each leg's device ms of the last call (aur_stats.last_total_ms
of the dense leg, aur_kw_stats.last_ms of the keyword leg; in the fused call the legs overlap).  Parity, checked in the
same run: the fused lists (ids, fp64 scores, fp32 cosines) of every request bit-identical to the host arm's; the run
fails otherwise.  The card's name and power limit are read in the same run.  Needs a GPU.

    python tools/hybrid_filter_bench.py [--docs 1000000] [--reps 20] [--warmup 3]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from aurora_b200 import _native as N  # noqa: E402
from aurora_b200 import bm25  # noqa: E402
from aurora_b200.engine import Index, KeywordIndex  # noqa: E402
from aurora_b200.filters import AttrColumn, Filter, compile_program  # noqa: E402
from fusion_bench import same, shape  # noqa: E402
from hybrid_bench import card, corpus, queries  # noqa: E402

DIM, FETCH, LIMIT, ALPHA = 768, 128, 3, 0.5
LIST_MAX_FRACTION = 0.005                  # retriever._LIST_MAX_FRACTION
SIZES = (1_000, 10_000, 100_000)           # the first three orgs; the 1M "org" is the shared tier
N_ORGS = 64


def host_request(ix, kw, vec, text, prog, max_list):
    """The parent's KnowledgeBase.query for one filtered hybrid request."""
    ids, scores, _, _ = ix.search_filtered(vec, FETCH, [prog], max_list_rows=max_list)
    dense = [(int(r), float(s)) for r, s in zip(ids[0], scores[0]) if r >= 0]
    allowed = ix.filter_ids(prog).tolist()
    sparse = kw.search(text, FETCH, allowed=allowed)
    cos = dict(dense)
    fused = bm25.ranked_fusion([(ALPHA, [d for d, _ in dense]), (1.0 - ALPHA, [d for d, _ in sparse])], LIMIT)
    picked = [(r, fs, cos.get(r)) for r, fs in fused]
    shape(picked)
    return picked


def host_arm(ix, kw, vecs, texts, progs, q_prog, max_list):
    return [host_request(ix, kw, vecs[q:q + 1], texts[q], progs[q_prog[q]], max_list) for q in range(len(texts))]


def fused_arm(ix, kw, vecs, texts, progs, q_prog, max_list):
    lists = kw.search_batch(texts, FETCH, dense=(ix, vecs, np.full(len(texts), ALPHA), N.FUSION_RANKED, LIMIT),
                            programs=progs, q_program=q_prog, max_list_rows=max_list)
    out = []
    for lst in lists:
        picked = [(r, fs, c) for r, (fs, c) in lst][:LIMIT]
        shape(picked)
        out.append(picked)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=250)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if N.load().aur_device_count() == 0:
        raise SystemExit("hybrid_filter_bench needs a CUDA device (aurora_b200 has no CPU path)")
    rng = np.random.default_rng(args.seed)
    t0 = time.perf_counter()
    n = args.docs
    terms, tfs, offsets = corpus(rng, n, args.tokens, args.vocab)
    qt, qo = queries(rng, 256, args.vocab)
    texts = [" ".join(f"t{t}" for t in qt[qo[q]:qo[q + 1]]) for q in range(256)]
    ids = np.arange(n, dtype=np.int64) * 3 + 1
    ix = Index(DIM, n)
    store = KeywordIndex(n, postings_capacity=len(terms))
    step = 100_000
    for d0 in range(0, n, step):
        d1 = min(n, d0 + step)
        ix.add(rng.standard_normal((d1 - d0, DIM), dtype=np.float32), ids[d0:d1])
        sl = slice(offsets[d0], offsets[d1])
        store.add(ids[d0:d1], terms[sl], tfs[sl], offsets[d0:d1 + 1] - offsets[d0])
    kw = bm25.DeviceBM25(store=store)
    kw.vocab = {f"t{i}": i for i in range(args.vocab)}          # the synthetic texts' words are "t<term id>"
    kw._docs = set(ids.tolist())
    # orgs: the three sized ones at the front, the rest of the rows split over the other 61
    bounds = list(np.cumsum((0,) + SIZES))
    rest = np.linspace(bounds[-1], n, N_ORGS - len(SIZES) + 1).astype(np.int64)
    bounds = np.array(bounds[:-1] + rest.tolist(), np.int64)
    org_of = np.searchsorted(bounds, np.arange(n), side="right") - 1
    cols = {nm: AttrColumn(nm, 2 + j) for j, nm in enumerate(("org_id", "document_id", "tier"))}
    codes = {"org_id": org_of.astype(np.int32), "tier": np.zeros(n, np.int32),
             "document_id": np.arange(n, dtype=np.int32)}
    for o in range(N_ORGS):                      # the dictionaries the codes index, in code order
        cols["org_id"].code({"org_id": f"org{o}"})
    cols["tier"].code({"tier": "all"})
    for i in range(n):
        cols["document_id"].code({"document_id": f"discovery:{i}" if i % 2 else f"doc:{i}"})
    for nm, c in cols.items():
        ix.set_attrs(c.col, ids, codes[nm])
        store.set_attrs(c.col, ids, codes[nm])
    setup_s = time.perf_counter() - t0
    disc = Filter.by_property("document_id").like("discovery:*")
    org_prog = [compile_program(Filter.by_property("org_id").equal(f"org{o}") & disc, cols) for o in range(N_ORGS)]
    all_prog = compile_program(Filter.by_property("tier").equal("all") & disc, cols)
    max_list = int(LIST_MAX_FRACTION * n)
    vecs = rng.standard_normal((256, DIM), dtype=np.float32)

    work = [(f"org{s}_nq1", [org_prog[j]], np.zeros(1, np.int32), s) for j, s in enumerate(SIZES)]
    work.append(("org1M_nq1", [all_prog], np.zeros(1, np.int32), n))
    work.append(("orgs64_nq256", org_prog, (np.arange(256) % N_ORGS).astype(np.int32), None))
    result = {"tool": "hybrid_filter_bench", "docs": n, "dim": DIM, "mean_tokens": args.tokens, "vocab": args.vocab,
              "fetch": FETCH, "limit": LIMIT, "alpha": ALPHA, "max_list_rows": max_list, "reps": args.reps,
              "setup_s": round(setup_s, 1)}
    parity = True
    rows = []
    for name, progs, q_prog, size in work:
        nq = len(q_prog)
        a = (ix, kw, vecs[:nq], texts[:nq], progs, q_prog, max_list)
        ok = same(host_arm(*a), fused_arm(*a))
        for _ in range(args.warmup):
            host_arm(*a)
            fused_arm(*a)
        wall = {"host": [], "fused": []}
        dev = {}
        for _ in range(args.reps):
            for arm, fn in (("host", host_arm), ("fused", fused_arm)):
                w0 = time.perf_counter()
                fn(*a)
                wall[arm].append((time.perf_counter() - w0) * 1e3)
                dev[arm] = (ix.stats()["last_total_ms"], store.stats()["last_ms"])
        row = {"workload": name, "org_rows": size, "queries": nq, "parity": bool(ok)}
        for arm in ("host", "fused"):
            row[arm] = {"wall_ms": round(float(np.median(wall[arm])), 3), "wall_ms_min": round(float(np.min(wall[arm])), 3),
                        "dense_leg_device_ms_last": round(float(dev[arm][0]), 3),
                        "keyword_leg_device_ms_last": round(float(dev[arm][1]), 3)}
        row["wall_speedup"] = round(row["host"]["wall_ms"] / row["fused"]["wall_ms"], 3)
        rows.append(row)
        parity &= ok
    result["workloads"] = rows
    result["parity"] = bool(parity)
    result["card"], result["power_limit"] = card()
    print(json.dumps(result), flush=True)
    ix.close()
    store.close()
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()

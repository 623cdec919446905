"""The keyword store's term-major index against its forward scan, on the GPU: one JSON line.

The corpus is tools/hybrid_bench.py's (default 1M documents of ~250 Zipf words over a 50k vocabulary, about 131.6 M
postings), ingested in 100k-document batches (the writer builds and rebuilds the index as it goes), then indexed in full
by one timed aur_kw_reindex.  Reported:
  * build: the last build's ms and the index's bytes, and how many builds the ingest made;
  * the keyword leg's device ms (CUDA events inside aur_kw_search) with kw_path forced to the index, forced forward and
    on the cost rule (auto), alternated rep by rep, medians, at nq 1 / 8 / 32 / 256 for rare-word queries (2-4 of the
    2 000 words of lowest df) and Zipf-word queries (hybrid_bench's), with the postings each path read and the path auto took;
  * the fused hybrid call's wall ms (engine.hybrid_search, a bf16 Index of the same ids) at nq 1 and 256, per path;
  * the filtered hybrid call's wall ms at nq 1 for a tenant program whose org holds 1 000 documents, per path;
  * parity: every measured batch's ids and scores bit-identical across the three paths, and sampled queries equal to
    oracle/bm25_topk.py over the whole corpus; the run fails otherwise;
  * the card's name and power limit, read in the same run.

    python tools/keyword_index_bench.py [--docs 1000000] [--reps 15] [--dim 384]
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from hybrid_bench import card, corpus, queries  # noqa: E402

from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import Index, KeywordIndex, hybrid_search  # noqa: E402
from aurora_b200.filters import compile_program  # noqa: E402

PATHS = {"index": N.KW_PATH_INDEX_OPT, "forward": N.KW_PATH_FORWARD_OPT, "auto": N.KW_PATH_AUTO_OPT}
PATH_NAMES = {0: "none", N.KW_PATH_FORWARD: "forward", N.KW_PATH_INDEX: "index", 3: "both"}


def rare_queries(rng, nq, df):
    live = np.nonzero(df > 0)[0]
    pool = live[np.argsort(df[live], kind="stable")[:2000]]
    terms, off = [], [0]
    for _ in range(nq):
        q = np.unique(rng.choice(pool, int(rng.integers(2, 5)), replace=False)).astype(np.int32)
        terms.append(q)
        off.append(off[-1] + len(q))
    return np.concatenate(terms), np.asarray(off, np.int64)


def same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1]).view(np.int64), np.asarray(b[1]).view(np.int64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=250)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--dim", type=int, default=384)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parity", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    terms, tfs, offsets = corpus(rng, args.docs, args.tokens, args.vocab)
    zq_t, zq_o = queries(rng, 256, args.vocab)
    df = np.bincount(terms, minlength=args.vocab)
    rq_t, rq_o = rare_queries(rng, 256, df)
    ids = np.arange(args.docs, dtype=np.int64)
    org = np.full(args.docs, -1, np.int32)
    org[rng.choice(args.docs, 1000, replace=False)] = 7          # the 1k-row org of the filtered call
    user = rng.integers(0, 1000, args.docs).astype(np.int32)

    kw = KeywordIndex(args.docs, postings_capacity=len(terms))
    ix = Index(args.dim, args.docs)
    step = 100_000
    t0 = time.perf_counter()
    for d0 in range(0, args.docs, step):
        d1 = min(args.docs, d0 + step)
        sl = slice(offsets[d0], offsets[d1])
        kw.add(ids[d0:d1], terms[sl], tfs[sl], offsets[d0:d1 + 1] - offsets[d0], user[d0:d1], org[d0:d1])
        ix.add(rng.standard_normal((d1 - d0, args.dim), dtype=np.float32), ids[d0:d1], user[d0:d1], org[d0:d1])
    ingest_s = time.perf_counter() - t0
    builds_ingest = kw.index_stats()["builds"]
    kw.reindex()
    st = kw.index_stats()
    result = {"docs": args.docs, "postings": int(kw.stats()["postings_used"]), "vocab": args.vocab, "dim": args.dim,
              "ingest_s": round(ingest_s, 2), "builds_during_ingest": int(builds_ingest),
              "build_ms": round(st["last_build_ms"], 2), "index_bytes": int(st["index_bytes"]),
              "indexed_rows": int(st["indexed_rows"])}
    parity = True
    k = 128

    def run(path, fn):
        kw.set_path(PATHS[path])
        return fn()

    def measure(fn, key):
        """fn() per path, alternated; medians of the key's number; the outputs must agree bit for bit."""
        vals = {p: [] for p in PATHS}
        info = {}
        outs = {}
        for r in range(args.warmup + args.reps):
            for p in PATHS:
                w0 = time.perf_counter()
                out = run(p, fn)
                wall = (time.perf_counter() - w0) * 1e3
                if r >= args.warmup:
                    vals[p].append(kw.stats()["last_ms"] if key == "device_ms" else wall)
                outs[p] = out
                s = kw.index_stats()
                info[p] = (PATH_NAMES[s["last_path"]], int(s["last_postings"]))
        ok = same(outs["index"], outs["forward"]) and same(outs["auto"], outs["forward"])
        return {p: {key: round(float(np.median(v)), 3), "path": info[p][0], "postings": info[p][1]}
                for p, v in vals.items()}, ok, outs["forward"]

    for kind, (qt, qo) in (("rare", (rq_t, rq_o)), ("zipf", (zq_t, zq_o))):
        for nq in (1, 8, 32, 256):
            q_off = qo[: nq + 1]
            res, ok, out = measure(lambda: kw.search(qt, q_off, k)[:2], "device_ms")
            parity &= ok
            result[f"kw_{kind}_nq{nq}"] = res
            if nq == 256 and args.parity:
                from oracle.bm25_topk import Corpus, bm25_topk

                cp = Corpus(terms, tfs, offsets, ids)
                for q in np.linspace(0, 255, args.parity).astype(int):
                    wi, ws = bm25_topk(cp, qt[qo[q]:qo[q + 1]], np.array([0, qo[q + 1] - qo[q]]), k)
                    parity &= bool(np.array_equal(out[0][q], wi[0]) and np.array_equal(out[1][q].view(np.int64), ws[0].view(np.int64)))

    vecs = rng.standard_normal((256, args.dim), dtype=np.float32)
    for kind, (qt, qo) in (("rare", (rq_t, rq_o)), ("zipf", (zq_t, zq_o))):
        for nq in (1, 256):
            res, ok, _ = measure(lambda: hybrid_search(ix, kw, vecs[:nq], k, qt, qo[: nq + 1], 0.5, k_out=10)[:2], "wall_ms")
            parity &= ok
            result[f"hybrid_{kind}_nq{nq}"] = res
    prog = [compile_program(None, {}, tenant=(-2, 7))]
    for kind, (qt, qo) in (("rare", (rq_t, rq_o)), ("zipf", (zq_t, zq_o))):
        res, ok, _ = measure(lambda: hybrid_search(ix, kw, vecs[:1], k, qt, qo[:2], 0.5, k_out=10, programs=prog)[:2],
                             "wall_ms")
        parity &= ok
        result[f"filtered_1k_org_{kind}_nq1"] = res
    result["parity"] = bool(parity)
    name, power = card()
    result["card"] = name
    result["power_limit"] = power
    print(json.dumps(result), flush=True)
    kw.close()
    ix.close()
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()

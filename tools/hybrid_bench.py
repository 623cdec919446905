"""Keyword leg of the hybrid query on the GPU: one JSON line.

A seeded synthetic corpus (default 1M documents of ~250 Zipf-distributed words over a 50k vocabulary) goes into the
device keyword store (engine.KeywordIndex); 256 queries of 2-8 words are searched in batches of 1, 32 and 256.  Reported:
  * device time per batch (CUDA events inside aur_kw_search: table upload, scoring pass, selection, folds) and the host
    wall time of the synchronous call, median over --reps after --warmup;
  * postings and bytes one batch reads (every row's postings, 8 B each, plus 13 B of row data), and that over the
    device time as a share of the H100 SXM data-sheet 3.35 TB/s;
  * the host BM25Index per-query time on the first --host-docs documents (stated; not extrapolated);
  * the host fusion + shaping time of a 256-request batch (bm25.ranked_fusion + result dicts);
  * the card's name and power limit, read in the same run.
--devices "0" (default) puts the corpus in one store on GPU 0; "all" or a list "0,1,..." shards it by id mod n over one
store per listed device (engine.MultiKeywordIndex, searched as one corpus; a device may be listed more than once).  The
device time of a sharded batch is the slowest store's; the line lists the stores' devices and postings.
Parity: --parity sampled queries of the 256 batch are held to oracle/bm25_topk.py over the whole corpus bit for bit; the
run fails otherwise.

    python tools/hybrid_bench.py [--docs 1000000] [--tokens 250] [--reps 20] [--devices 0|all|0,1,...]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aurora_b200 import bm25  # noqa: E402
from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import KeywordIndex, MultiKeywordIndex  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def corpus(rng, n_docs, tokens, vocab, a=1.2):
    """CSR (term ids ascending per doc, tf, offsets) of n_docs documents with Poisson(tokens) Zipf words."""
    lens = rng.poisson(tokens, n_docs).astype(np.int64)
    doc = np.repeat(np.arange(n_docs, dtype=np.int64), lens)
    words = ((rng.zipf(a, len(doc)) - 1) % vocab).astype(np.int64)
    key = np.sort(doc << 20 | words)
    first = np.concatenate([[True], key[1:] != key[:-1]])
    starts = np.nonzero(first)[0]
    tf = np.diff(np.append(starts, len(key))).astype(np.int32)
    ukey = key[starts]
    terms = (ukey & ((1 << 20) - 1)).astype(np.int32)
    per_doc = np.bincount(ukey >> 20, minlength=n_docs)
    offsets = np.concatenate([[0], np.cumsum(per_doc)]).astype(np.int64)
    return terms, tf, offsets


def queries(rng, nq, vocab, a=1.2):
    terms, off = [], [0]
    for _ in range(nq):
        q = np.unique((rng.zipf(a, int(rng.integers(2, 9))) - 1) % vocab).astype(np.int32)
        terms.append(q)
        off.append(off[-1] + len(q))
    return np.concatenate(terms), np.asarray(off, np.int64)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--tokens", type=int, default=250)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-docs", type=int, default=30_000)
    ap.add_argument("--host-queries", type=int, default=64)
    ap.add_argument("--parity", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--devices", default="0", help='"0" = one store on GPU 0; "all" or "0,1,..." = one store per device')
    args = ap.parse_args()
    if args.devices == "all":
        devices = list(range(N.load().aur_device_count()))
    else:
        devices = [int(d) for d in args.devices.split(",")]
    rng = np.random.default_rng(args.seed)
    t0 = time.perf_counter()
    terms, tfs, offsets = corpus(rng, args.docs, args.tokens, args.vocab)
    gen_s = time.perf_counter() - t0
    qt, qo = queries(rng, 256, args.vocab)
    ids = np.arange(args.docs, dtype=np.int64)

    sharded = len(devices) > 1
    if sharded:
        store = MultiKeywordIndex(args.docs, devices=devices, postings_capacity=len(terms))
    else:
        store = KeywordIndex(args.docs, postings_capacity=len(terms), device=devices[0])
    t0 = time.perf_counter()
    step = 100_000
    for d0 in range(0, args.docs, step):
        d1 = min(args.docs, d0 + step)
        sl = slice(offsets[d0], offsets[d1])
        store.add(ids[d0:d1], terms[sl], tfs[sl], offsets[d0:d1 + 1] - offsets[d0])
    ingest_s = time.perf_counter() - t0
    st = store.stats()

    result = {"docs": args.docs, "mean_tokens": args.tokens, "vocab": args.vocab, "postings": int(st["postings_used"]),
              "ingest_s": round(ingest_s, 2), "corpus_gen_s": round(gen_s, 2), "stores": len(devices), "devices": devices,
              "postings_per_store": [int(p["postings_used"]) for p in st["stores"]] if sharded else [int(st["postings_used"])]}
    bytes_per_batch = int(st["postings_used"]) * 8 + args.docs * 13
    result["bytes_per_batch"] = bytes_per_batch
    k = 128
    for nq in (1, 32, 256):
        q_off = qo[: nq + 1]
        for _ in range(args.warmup):
            store.search(qt, q_off, k)
        dev, wall = [], []
        for _ in range(args.reps):
            w0 = time.perf_counter()
            store.search(qt, q_off, k)
            wall.append((time.perf_counter() - w0) * 1e3)
            dev.append(store.stats()["last_ms"])
        d = float(np.median(dev))
        result[f"nq{nq}"] = {"device_ms": round(d, 3), "device_ms_min": round(float(np.min(dev)), 3),
                             "wall_ms": round(float(np.median(wall)), 3), "launches": int(store.stats()["last_launches"]),
                             "bytes_per_s": round(bytes_per_batch / (d * 1e-3), 1),
                             "share_of_3.35TBps": round(bytes_per_batch / (d * 1e-3) / HBM_BYTES_PER_S, 4)}

    # parity: sampled queries of the 256 batch against the fp64 oracle, bit for bit
    from oracle.bm25_topk import Corpus, bm25_topk

    got_i, got_s, snap = store.search(qt, qo, k)
    assert (sum(snap) if sharded else snap) == args.docs
    cp = Corpus(terms, tfs, offsets, ids)                    # the whole corpus, however it is sharded
    sample = np.linspace(0, 255, args.parity).astype(int)
    ok = True
    for q in sample:
        wi, ws = bm25_topk(cp, qt[qo[q]:qo[q + 1]], np.array([0, qo[q + 1] - qo[q]]), k)
        ok &= bool(np.array_equal(got_i[q], wi[0]) and np.array_equal(got_s[q].view(np.int64), ws[0].view(np.int64)))
    result["parity"] = ok
    result["parity_queries"] = int(len(sample))

    # host BM25Index on a down-sampled corpus (its default path, numpy fast path included)
    hd = min(args.host_docs, args.docs)
    host = bm25.BM25Index()
    for d in range(hd):
        sl = slice(offsets[d], offsets[d + 1])
        host.add(d, " ".join(f"t{t} " * int(f) for t, f in zip(terms[sl], tfs[sl])))
    texts = [" ".join(f"t{t}" for t in qt[qo[q]:qo[q + 1]]) for q in range(args.host_queries)]
    for q in texts[:4]:
        host.search(q, k)
    h0 = time.perf_counter()
    for q in texts:
        host.search(q, k)
    result["host_bm25"] = {"docs": hd, "queries": len(texts),
                           "ms_per_query": round((time.perf_counter() - h0) * 1e3 / len(texts), 3)}

    # host fusion + shaping of a 256-request batch (what query_batch does after the two device legs)
    dense = [[(int(i), 0.9 - 0.001 * r) for r, i in enumerate(rng.permutation(args.docs)[:k])] for _ in range(256)]
    sparse = [[(int(i), float(s)) for i, s in zip(got_i[q], got_s[q]) if i >= 0] for q in range(256)]
    props = {"content": "x", "heading_context": "", "source_filename": "f", "document_id": "d", "chunk_index": 0}
    f0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        for q in range(256):
            cos = dict(dense[q])
            fused = bm25.ranked_fusion([(0.5, [d for d, _ in dense[q]]), (0.5, [d for d, _ in sparse[q]])], 5)
            objs = [SimpleNamespace(properties=dict(props), uuid=None,
                                    metadata=SimpleNamespace(score=fs, distance=None if cos.get(r) is None else 1 - cos[r]))
                    for r, fs in fused]
            [{"content": o.properties["content"], "score": o.metadata.score} for o in objs]
    result["host_fusion_ms_per_256"] = round((time.perf_counter() - f0) * 1e3 / reps, 3)
    name, power = card()
    result["card"] = name
    result["power_limit"] = power
    print(json.dumps(result), flush=True)
    store.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()

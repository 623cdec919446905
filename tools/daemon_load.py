#!/usr/bin/env python
"""Load test of the engine daemon on a GPU: the reference's call pattern -- many client threads, ONE query per call
(server/routes/knowledge_base/weaviate_client.py:252-259; 2 gunicorn workers x 4 threads + Celery + chatbot,
docker-compose.yaml:191,283-285) -- against (a) one caller at a time and (b) 64 concurrent callers whose requests the
daemon coalesces into one encoder batch + one dense launch per tenant scope.

  python tools/daemon_load.py [out.json]          (bge-base dims, random-init weights, synthetic vocabulary)
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aurora_b200.daemon import Client, serve  # noqa: E402


def client_main(argv):
    """One client process: `threads` threads, `per_thread` single-query calls each (no GPU, no engine import)."""
    path, threads, per_thread, n_tenants, pid, out, qfile = argv[0], int(argv[1]), int(argv[2]), int(argv[3]), int(argv[4]), argv[5], argv[6]
    queries = json.load(open(qfile))
    lat, errs = [], []

    def worker(i):
        try:
            c = Client(path)
            for j in range(per_thread):
                t1 = time.time()
                r = c.search_knowledge_base(f"user{(pid * 7 + i + j) % n_tenants}", queries[(pid * 131 + i * 31 + j) % len(queries)], limit=5)
                lat.append(time.time() - t1)
                assert isinstance(r, list) and len(r) == 5, r
        except Exception as e:      # pragma: no cover
            errs.append(repr(e))

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(threads)]
    t0 = time.time()
    [t.start() for t in ts]; [t.join() for t in ts]
    json.dump({"lat": lat, "t0": t0, "t1": time.time(), "errs": errs}, open(out, "w"))
    sys.exit(1 if errs else 0)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/daemon_load.json"
    import bench
    from aurora_b200 import retriever as R
    from aurora_b200.encoder import Encoder, EncoderConfig, TextEncoder
    from aurora_b200.wordpiece import NativeTokenizer

    cfg = EncoderConfig()
    rng = np.random.default_rng(5)
    lens = np.clip(np.rint(rng.normal(200, 60, 96)), 16, 400).astype(np.int64)
    pieces, texts = bench.synth_vocab_and_texts(cfg.vocab, lens, 99)
    enc = Encoder(cfg, max_tokens=65536, max_seqs=512, device=0)
    enc.load_weights(bench.random_bert_weights(cfg, 7))
    te = TextEncoder(enc, NativeTokenizer(pieces))
    n_tenants, docs_per_tenant = 8, 40
    R.configure(encoder=te, capacity=1 << 18, device=0)
    t0 = time.perf_counter()
    for t in range(n_tenants):
        for d in range(docs_per_tenant):
            chunks = [{"content": texts[(t * 7 + d * 3 + i) % len(texts)] + f" tenant{t} doc{d} part{i}", "heading_context": f"T{t} > D{d}", "chunk_index": i}
                      for i in range(12)]
            R.insert_chunks(f"user{t}", f"doc-{t}-{d}", "runbook.md", chunks, org_id=f"org{t % 3}")
    ingest_s = time.perf_counter() - t0
    n_chunks = n_tenants * docs_per_tenant * 12
    queries = [" ".join(texts[i % len(texts)].split()[:24]) for i in range(256)]
    res = {"chunks_ingested": n_chunks, "ingest_chunks_per_s": n_chunks / ingest_s, "tenants": n_tenants}
    with tempfile.TemporaryDirectory() as tmp:
        qfile = os.path.join(tmp, "queries.json")
        json.dump(queries, open(qfile, "w"))
        for label, coalesce_us, n_threads, per_thread in (("single_caller", 0, 1, 300), ("64_callers_no_coalescing", 0, 64, 60),
                                                          ("64_callers_coalesced", 300, 64, 60)):
            path = os.path.join(tmp, f"{label}.sock")
            srv = serve(path, background=True, coalesce_us=coalesce_us)
            Client(path).search_knowledge_base("user0", queries[0], limit=5)      # warm
            # clients are separate PROCESSES, like gunicorn workers / Celery children in the reference: the daemon's
            # interpreter is not shared with them
            n_procs = min(n_threads, 8)
            per_proc = n_threads // n_procs
            outs = [os.path.join(tmp, f"{label}.{i}.json") for i in range(n_procs)]
            t0 = time.perf_counter()
            procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "--client", path, str(per_proc), str(per_thread),
                                       str(n_tenants), str(i), outs[i], qfile]) for i in range(n_procs)]
            rcs = [pr.wait() for pr in procs]
            wall = time.perf_counter() - t0
            errs = [f"client process {i} exited {rc}" for i, rc in enumerate(rcs) if rc != 0]
            lat, spans = [], []
            for o in outs:
                if os.path.exists(o):
                    d = json.load(open(o)); lat += d["lat"]; spans.append((d["t0"], d["t1"]))
            if spans:
                wall = max(b for _, b in spans) - min(a for a, _ in spans)      # first request sent .. last answer received
            h = Client(path).health()
            srv.shutdown(); srv.close_all(final_save=False); srv.server_close()
            if errs:
                raise SystemExit(f"{label}: {errs[0]}")
            n_req = n_threads * per_thread
            res[label] = {"requests": n_req, "threads": n_threads, "requests_per_s": n_req / wall, "p50_ms": float(np.median(lat) * 1e3),
                          "p99_ms": float(np.percentile(lat, 99) * 1e3), "coalesced_batches": h.get("coalesced_batches", 0)}
            print(label, res[label], flush=True)
    res["speedup_vs_single_caller"] = res["64_callers_coalesced"]["requests_per_s"] / res["single_caller"]["requests_per_s"]
    res["note"] = ("every request = JSON over a Unix socket -> tokenise -> encoder forward (bge-base dims) -> tenant-scoped hybrid search "
                   "(dense leg on the tensor-core kernel + BM25 + ranked fusion) -> result dicts; Python daemon threads")
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    json.dump(res, open(out, "w"), indent=1)
    print(json.dumps(res))
    R.configure(encoder=None)
    enc.close()


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--client":
        client_main(sys.argv[2:])
    else:
        main()

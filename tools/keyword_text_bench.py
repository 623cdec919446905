"""Keyword ingest: text analysed on the GPU (aur_kw_add_text) against the host path (bm25.build_csr + aur_kw_add).

Prints one JSON line.  The corpus is seeded and synthetic, chunks of about 1,500 characters (the chunker's target,
document_processor.py): Zipf words in mixed case, digits, IP-like and hex tokens, and a little non-ASCII including
U+0130 and U+212A.  The text path is timed at batch sizes 1, 50 (one document's chunks) and 4,096 with a warm
vocabulary, on the host clock around calls that return after their device work.  Device time comes from torch.profiler's
CUDA activity (CUPTI) of one 4,096-chunk call: the analysis kernels alone, and every kernel, copy and memset of the
call (the store's copies included).  The host path is timed on a stated sample, not extrapolated.
Parity compares the rows (aur_kw_read_rows) and the vocabulary of the whole corpus with build_csr's in the same run.

    python tools/keyword_text_bench.py [--chunks 20000] [--host-sample 2000]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import bm25  # noqa: E402
from aurora_b200.engine import KeywordIndex, KeywordVocab  # noqa: E402

EXTRA = ["İstanbul", "Kelvin", "café", "naïve", "Überweisung", "日本語", "résumé"]


def corpus(n, seed=0, chars=1500, vocab=30000):
    rng = np.random.default_rng(seed)
    base = [f"w{i}" for i in range(vocab)]
    out = []
    for _ in range(n):
        parts, size = [], 0
        while size < chars:
            r = rng.random()
            if r < 0.80:
                w = base[(int(rng.zipf(1.2)) - 1) % vocab]
                w = w.upper() if rng.random() < 0.05 else (w.capitalize() if rng.random() < 0.15 else w)
            elif r < 0.88:
                w = str(int(rng.integers(0, 100000)))
            elif r < 0.93:
                w = ".".join(str(int(x)) for x in rng.integers(0, 256, 4))
            elif r < 0.97:
                w = "0x" + "".join(rng.choice(list("0123456789abcdefABCDEF"), 8))
            else:
                w = EXTRA[int(rng.integers(0, len(EXTRA)))]
            parts.append(w)
            size += len(w) + 1
        out.append(" ".join(parts))
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as exc:   # noqa: BLE001
        return f"unknown ({exc})", "unknown"


def text_path(texts, vocab, batch, n_docs):
    store = KeywordIndex(n_docs + batch + 16, postings_capacity=(n_docs + batch) * 200)
    store.add_text(vocab, np.arange(batch) + n_docs, texts[:batch])     # warm the store's buffers
    t0 = time.perf_counter()
    done = 0
    while done < n_docs:
        b = texts[done:done + batch]
        store.add_text(vocab, np.arange(done, done + len(b)), b)
        done += len(b)
    dt = time.perf_counter() - t0
    mb = sum(len(t.encode()) for t in texts[:done]) / 1e6
    store.close()
    return done / dt, (mb / dt if mb else None), dt / done * 1e6


def host_path(texts, batch, n_docs):
    ref = {}
    bm25.build_csr(ref, texts)                                  # a warm vocabulary, as on the text path
    store = KeywordIndex(n_docs + 16, postings_capacity=n_docs * 200)
    t0 = time.perf_counter()
    for i in range(0, n_docs, batch):
        b = texts[i:i + batch]
        t, f, o = bm25.build_csr(ref, b)
        store.add(np.arange(i, i + len(b)), t, f, o)
    dt = time.perf_counter() - t0
    store.close()
    return n_docs / dt, dt / n_docs * 1e6


def device_ms(texts, vocab):
    """Device time of one add_text call from torch.profiler's CUDA activity (CUPTI): (the analysis kernels -- the
    tx_* and CUB kernels, summed -- , every kernel, copy and memset of the call, the store's copies included)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    store = KeywordIndex(len(texts) + 16, postings_capacity=len(texts) * 200)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        store.add_text(vocab, np.arange(len(texts)), texts)
    kernels = total = 0.0
    for ev in prof.events():
        if ev.device_type.name == "CUDA":
            t = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            total += t
            if not ev.name.startswith(("Memcpy", "Memset")):
                kernels += t
    store.close()
    return kernels / 1e3, total / 1e3


def parity(texts):
    vocab = KeywordVocab(0)
    store = KeywordIndex(len(texts) + 16, postings_capacity=len(texts) * 200)
    ref, rows = {}, []
    for i in range(0, len(texts), 4096):
        b = texts[i:i + 4096]
        store.add_text(vocab, np.arange(i, i + len(b)), b)
        rows.append(bm25.build_csr(ref, b))
    t = np.concatenate([r[0] for r in rows])
    f = np.concatenate([r[1] for r in rows])
    lens = np.concatenate([np.diff(r[2]) for r in rows])
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    ids, goff, gt, gf = store.read_rows(0, len(texts))
    ok = (np.array_equal(ids, np.arange(len(texts))) and np.array_equal(goff, off) and np.array_equal(gt, t)
          and np.array_equal(gf, f) and vocab.read() == list(ref))
    store.close(); vocab.close()
    return bool(ok), len(ref)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=20000)
    ap.add_argument("--host-sample", type=int, default=2000)
    a = ap.parse_args()
    texts = corpus(a.chunks)
    name, power = card()
    ok, words = parity(texts)
    vocab = KeywordVocab(0)
    KeywordIndex(len(texts) + 16, postings_capacity=len(texts) * 200).add_text(vocab, np.arange(len(texts)), texts)   # warm
    res = {"metric": "keyword_text_ingest", "card": name, "power_limit": power, "parity": ok, "chunks": len(texts),
           "vocab_words": words, "mean_chunk_bytes": round(float(np.mean([len(t.encode()) for t in texts])), 1)}
    for batch, n in ((1, min(len(texts), 300)), (50, min(len(texts), 3000)), (4096, min(len(texts), 16384))):
        dps, mbps, us = text_path(texts, vocab, batch, n)
        res[f"text_b{batch}"] = {"docs_per_s": round(dps, 1), "mb_per_s": None if mbps is None else round(mbps, 2),
                                 "us_per_doc": round(us, 2), "docs": n}
    for batch in (50, 4096):
        n = min(a.host_sample, len(texts))
        dps, us = host_path(texts[:n], batch, n)
        res[f"host_b{batch}"] = {"docs_per_s": round(dps, 1), "us_per_doc": round(us, 2), "sample_docs": n}
    kern, total = device_ms(texts[:4096], vocab)
    res["device_ms_4096"] = {"analysis_kernels": round(kern, 3), "all_device_activity": round(total, 3),
                             "source": "torch.profiler CUDA activity of one add_text call"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Deletes and counts by filter: KnowledgeBase.delete_where / count_where resolved on the device (aur_remove_filtered,
aur_filter_count) against the host scan they replace (a Python predicate over every object's properties), on twin
knowledge bases built from the same inserts.  Prints one JSON line.  Needs a GPU.

Corpus per size (100k and 1M objects by default): 100 orgs, one user per org, documents of 10 chunks, every fourth
document a "discovery:" one; each org's documents arrive in four insert calls with four created_at values (one value
per insert call, as KnowledgeBase.insert stamps them).  Vectors come from a seeded normal table picked by checksums of the text
(the same text, the same vector), dim 256, bf16.  The host twin's ``_device_program`` returns None, so every filter it gets takes
the host scan; the device twin resolves the same filters on the GPU.

Reported per size, wall ms medians over ``--calls`` calls of distinct arguments, each twin in turn:
  * delete_document_chunks(user, doc), delete_discovery_chunks(org, before), get_document_chunk_count(user, doc);
  * first_use_ms: the first call of each twin, which on the device twin builds the attribute columns of the properties
    the filters name (a one-time O(N) pass per property);
  * query_p50_ms / query_p99_ms: tenant-scoped vector queries issued from another thread while the deletes run (the
    knowledge-base lock makes them wait), and query_idle_* with no delete running;
  * remove_100k_ms: Index.remove of 100k ids (one upload, one tombstone launch) and per_row_copy_100k_ms: the per-row
    4-byte cudaMemcpyAsync loop aur_remove ran before, replayed with the same calls on a scratch buffer.
parity: the twins return the same values, and end with the same property keys, export() live flags, keyword stats()
and query answers.  The card's name and power limit are read in the same run."""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import threading
import time
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import _native as N                      # noqa: E402
from aurora_b200 import retriever as R                    # noqa: E402
from tools.list_bench import card                         # noqa: E402

DIM, ORGS, CHUNKS, BATCHES, SEED = 256, 100, 10, 4, 1234
STAMPS = [f"2026-03-0{b + 1}T00:00:00+00:00" for b in range(BATCHES)]


class SeededEmbedder:
    """A text's vector is the sum of two rows of a seeded normal table, picked by two checksums of the text: the same
    text gets the same vector in both twins, whatever else each has encoded."""

    def __init__(self, dim: int = DIM, seed: int = SEED, rows: int = 1 << 16):
        self.table = np.random.default_rng(seed).standard_normal((2, rows, dim)).astype(np.float32)

    @property
    def dim(self) -> int:
        return self.table.shape[2]

    def encode(self, texts):
        raw = [t.encode("utf-8") for t in texts]
        a = np.array([zlib.crc32(b) for b in raw], np.int64) % self.table.shape[1]
        b = np.array([zlib.adler32(b) for b in raw], np.int64) % self.table.shape[1]
        return self.table[0, a] + self.table[1, b]


def _fill(kb, n):
    """n objects over ORGS orgs (user u<o> in org o<o>), CHUNKS chunks per document, every fourth a discovery document."""
    per_org = n // ORGS
    docs = per_org // CHUNKS
    for b in range(BATCHES):
        for o in range(ORGS):
            objs = []
            for d in range(b * docs // BATCHES, (b + 1) * docs // BATCHES):
                doc = f"discovery:{o}:{d}" if d % 4 == 0 else f"doc:{o}:{d}"
                for c in range(CHUNKS):
                    props = {"user_id": f"u{o}", "document_id": doc, "chunk_index": c, "content": f"chunk {c} of {doc}",
                             "heading_context": "", "source_filename": f"{doc}.md", "created_at": STAMPS[b], "org_id": f"o{o}"}
                    objs.append((R.generate_uuid5(f"u{o}:{doc}:{c}"), props, props["content"]))
            kb.insert_objects(objs, f"u{o}", f"o{o}")
    return docs


def _twins(n):
    kbs = []
    for host in (True, False):
        kb = R.KnowledgeBase(SeededEmbedder(), capacity=n + 1024)
        if host:
            kb._device_program = lambda *a, **k: None
        kbs.append(kb)
    docs = [_fill(kb, n) for kb in kbs][0]
    return kbs, docs


def _call(kb, fn, *args):
    R.configure(factory=lambda: kb)
    t0 = time.perf_counter()
    out = getattr(R, fn)(*args)
    return out, (time.perf_counter() - t0) * 1e3


def _queries(kb, stop, lat):
    """Tenant-scoped vector queries until ``stop`` is set; their wall ms into ``lat``."""
    i = 0
    while not stop.is_set():
        t0 = time.perf_counter()
        kb.query("chunk 3", 10, user_id=f"u{i % ORGS}", scoped=True)
        lat.append((time.perf_counter() - t0) * 1e3)
        i += 1


def _pct(lat):
    return (round(float(np.percentile(lat, 50)), 3), round(float(np.percentile(lat, 99)), 3)) if lat else (None, None)


def _state(kb):
    _, _, _, _, live = kb.index.export()
    answers = [[o.uuid for o in kb.query(q, 10, user_id=f"u{u}", scoped=True)] for q in ("chunk 1", "chunk 7") for u in (0, 5, 42)]
    kw = {k: v for k, v in kb.sparse.stats().items() if k in ("docs", "live", "postings_used", "total_len")}
    return sorted(kb._props), live.tolist(), kw, answers


def _one_size(n, calls):
    (host, dev), docs = _twins(n)
    out = {"objects": n, "documents_per_org": docs}
    parity = True
    plan = [("get_document_chunk_count", (f"u{o}", f"doc:{o}:{1 + 4 * (o % (docs // 4))}")) for o in range(calls)]
    plan += [("delete_document_chunks", (f"u{o}", f"doc:{o}:{1 + 4 * (o % (docs // 4))}")) for o in range(calls, 2 * calls)]
    plan += [("delete_discovery_chunks", (f"o{o}", STAMPS[2])) for o in range(2 * calls, 3 * calls)]
    first = {}
    for name, kb in (("host", host), ("device", dev)):   # first use: the device twin builds its attribute columns
        r1, ms1 = _call(kb, "get_document_chunk_count", "nobody", "nothing")
        r2, ms2 = _call(kb, "delete_discovery_chunks", "nobody", STAMPS[1])
        first[name] = round(ms1 + ms2, 3)
        parity &= r1 == 0 and r2 == 0
    out["first_use_ms"] = first
    for name, kb in (("host", host), ("device", dev)):
        lat = []
        stop = threading.Event()
        th = threading.Thread(target=_queries, args=(kb, stop, lat))
        th.start()
        time.sleep(0.5)
        idle = list(lat)
        res, times = [], {}
        for fn, args in plan:
            r, ms = _call(kb, fn, *args)
            res.append(r)
            times.setdefault(fn, []).append(ms)
        stop.set()
        th.join()
        busy = lat[len(idle):]
        out[name] = {fn: round(float(np.median(v)), 3) for fn, v in times.items()}
        out[name]["query_idle_p50_ms"], out[name]["query_idle_p99_ms"] = _pct(idle)
        out[name]["query_p50_ms"], out[name]["query_p99_ms"] = _pct(busy)
        out[name]["results"] = res
    parity &= out["host"].pop("results") == out["device"].pop("results")
    parity &= _state(host) == _state(dev)
    out["parity"] = bool(parity)
    for kb in (host, dev):
        kb.index.close()
    return out


def _remove_100k():
    """Index.remove of 100k ids, and the per-row 4-byte copy loop it replaced (same cudaMemcpyAsync calls, scratch buffer)."""
    import torch

    from aurora_b200.engine import Index

    n, m = 200_000, 100_000
    rng = np.random.default_rng(SEED)
    with Index(64, n) as ix:
        ix.add(rng.standard_normal((n, 64)).astype(np.float32), np.arange(n, dtype=np.int64))
        kill = rng.choice(n, size=m, replace=False).astype(np.int64)
        t0 = time.perf_counter()
        removed = ix.remove(kill)
        new_ms = (time.perf_counter() - t0) * 1e3
    import nvidia.cuda_runtime as cr

    lib = C.CDLL(os.path.join(list(cr.__path__)[0], "lib", "libcudart.so.12"))
    torch.cuda.init()
    buf = torch.zeros(n, dtype=torch.float32, device="cuda:0")
    s = C.c_void_p()
    assert lib.cudaStreamCreateWithFlags(C.byref(s), 1) == 0
    nan = C.c_float(float("nan"))
    rows = rng.choice(n, size=m, replace=False)
    base = buf.data_ptr()
    t0 = time.perf_counter()
    for r in rows.tolist():
        lib.cudaMemcpyAsync(C.c_void_p(base + 4 * r), C.byref(nan), C.c_size_t(4), 1, s)
    assert lib.cudaStreamSynchronize(s) == 0
    old_ms = (time.perf_counter() - t0) * 1e3
    lib.cudaStreamDestroy(s)
    ok = removed == m and int(torch.isnan(buf).sum()) == m
    return {"remove_100k_ms": round(new_ms, 3), "per_row_copy_100k_ms": round(old_ms, 3), "remove_ok": bool(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="100000,1000000")
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    if N.load().aur_device_count() == 0:
        raise SystemExit("delete_bench needs a CUDA device (aurora_b200 has no CPU path)")
    name, power = card()
    out = {"bench": "delete_filtered", "gpu": name, "power_limit": power, "dim": DIM, "orgs": ORGS, "calls": args.calls}
    out.update(_remove_100k())
    out["sizes"] = [_one_size(int(s), args.calls) for s in args.sizes.split(",")]
    out["parity"] = all(s["parity"] for s in out["sizes"]) and out["remove_ok"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Full ``KnowledgeBase.save`` against incremental ``KnowledgeBase.checkpoint`` on a CUDA shard (DESIGN.md section 9).

A knowledge base of ``--chunks`` chunks (default 1M) of 768-d bf16 rows on one ``engine.Index``, each with synthetic
properties of about 1.5 kB, is saved in full, checkpointed as a base, changed by ``--mutations`` upserts, inserts and
deletes, and checkpointed as a delta.  For each: seconds, bytes written and the milliseconds spent under the knowledge
base's lock.  A second thread issues single-query ``kb.query`` calls back to back while idle, during the save and
during each checkpoint; their p50 / p99 / max are reported.  Last, the checkpoint is restored and compared with the live
store: the same live rows by id, the same properties, and the same answers to sampled queries (``parity``).  The card
and its power limit are read in the same run.  Prints one JSON line.

The store is filled directly (rows through ``Index.add``, properties into its table) rather than through an encoder:
what is measured is the snapshot, not the ingest.  Files go to a temporary directory, removed at the end.
"""

from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import retriever as R          # noqa: E402
from aurora_b200.engine import Index, grow_for  # noqa: E402

DIM = 768


class SeededEncoder:
    """Deterministic text -> vector (a seeded Gaussian per text): what the queries and the mutations encode with."""

    dim = DIM

    def encode(self, texts):
        out = np.empty((len(texts), DIM), np.float32)
        for i, t in enumerate(texts):
            seed = int.from_bytes(hashlib.sha1(t.encode()).digest()[:8], "little")
            out[i] = np.random.default_rng(seed).standard_normal(DIM)
        return out


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:      # noqa: BLE001
        return f"unknown ({e})", "unknown"


def _fill(kb, n, rng):
    text = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz     "), size=1 << 20))
    users, orgs = [f"user{u}" for u in range(64)], [f"org{o}" for o in range(8)]
    for u in users:
        kb._code(kb._user_code, u, True)
    for o in orgs:
        kb._code(kb._org_code, o, True)
    step = 65536
    for r0 in range(0, n, step):
        m = min(step, n - r0)
        ids = np.arange(r0, r0 + m, dtype=np.int64)
        u = (ids % 64).astype(np.int32)
        o = (ids % 8).astype(np.int32)
        grow_for(kb.index, ids)
        kb.index.add(rng.standard_normal((m, DIM)).astype(np.float32), ids, u, o)
        for i in ids.tolist():
            at = (i * 7919) % ((1 << 20) - 1500)
            key = R.generate_uuid5(f"bench:{i}")
            props = {"user_id": users[i % 64], "org_id": orgs[i % 8], "document_id": f"doc{i // 50}",
                     "chunk_index": i % 50, "content": text[at:at + 1400], "heading_context": "section",
                     "source_filename": f"doc{i // 50}.md", "created_at": "2026-10-19T00:00:00+00:00"}
            kb._props[i] = props
            kb._key2id[key] = i
            kb._id2key[i] = key
            kb._by_user.setdefault(props["user_id"], set()).add(i)
            kb._by_org.setdefault(props["org_id"], set()).add(i)
    kb._next_id = n
    kb.mutations = n


def _mutate(kb, n, rng, round_):
    """n mutations: a third upserts of existing chunks, a third new chunks, a third deletes."""
    third = n // 3
    up = rng.choice(kb._next_id, size=third, replace=False)
    objs = []
    for i in up.tolist():
        key = kb._id2key.get(i)
        if key is not None:
            p = dict(kb._props[i], content=f"revised {round_} {i}")
            objs.append((key, p, p["content"]))
    kb.insert_objects(objs, "user1", "org1")
    new = [(R.generate_uuid5(f"new:{round_}:{j}"), {"user_id": "user1", "org_id": "org1", "document_id": f"new{round_}",
            "chunk_index": j, "content": f"new chunk {round_} {j}"}, f"new chunk {round_} {j}") for j in range(third)]
    kb.insert_objects(new, "user1", "org1")
    dels = [i for i in rng.choice(kb._next_id, size=n - 2 * third, replace=False).tolist() if i in kb._props]
    kb._delete_ids(dels)


def _during(kb, fn, queries):
    """fn() on this thread while another thread runs single queries back to back: (fn's result, latencies ms)."""
    lat, stop = [], threading.Event()

    def run():
        i = 0
        while not stop.is_set():
            t = time.perf_counter()
            kb.query(queries[i % len(queries)], 10)
            lat.append((time.perf_counter() - t) * 1e3)
            i += 1
    th = threading.Thread(target=run)
    th.start()
    time.sleep(0.05)
    try:
        res = fn()
    finally:
        stop.set()
        th.join()
    return res, lat


def _pct(lat):
    a = np.asarray(lat) if lat else np.zeros(1)
    return {"n": len(lat), "p50_ms": round(float(np.percentile(a, 50)), 3), "p99_ms": round(float(np.percentile(a, 99)), 3),
            "max_ms": round(float(a.max()), 3)}


def _dir_bytes(d):
    return sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=1_000_000)
    ap.add_argument("--mutations", type=int, default=2000)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    card, power = _card()
    enc = SeededEncoder()
    kb = R.KnowledgeBase(enc, capacity=args.chunks + 65536, index_factory=lambda dim, cap: Index(dim, cap))
    t = time.perf_counter()
    _fill(kb, args.chunks, rng)
    fill_s = time.perf_counter() - t
    queries = [f"query {i} about incident runbooks" for i in range(64)]
    for q in queries[:8]:
        kb.query(q, 10)                                   # warm up
    root = tempfile.mkdtemp(prefix="aur-snapshot-")
    out = {"bench": "snapshot", "card": card, "power_limit": power, "chunks": args.chunks, "dim": DIM, "dtype": "bf16",
           "mutations": args.mutations, "fill_s": round(fill_s, 1)}
    try:
        _, lat = _during(kb, lambda: time.sleep(2.0), queries)
        out["query_idle"] = _pct(lat)

        full = os.path.join(root, "full")

        def save():
            t0 = time.perf_counter()
            kb.save(full)
            return time.perf_counter() - t0
        secs, lat = _during(kb, save, queries)
        out["save"] = {"seconds": round(secs, 3), "bytes": _dir_bytes(full), "locked_ms": round(secs * 1e3, 1),
                       "query": _pct(lat)}
        shutil.rmtree(full)

        ck = os.path.join(root, "ckpt")
        res, lat = _during(kb, lambda: kb.checkpoint(ck), queries)
        out["checkpoint_base"] = dict(res, query=_pct(lat))
        _mutate(kb, args.mutations, rng, 0)
        res, lat = _during(kb, lambda: kb.checkpoint(ck), queries)
        out["checkpoint_delta"] = dict(res, query=_pct(lat))
        _mutate(kb, args.mutations, rng, 1)
        res, lat = _during(kb, lambda: kb.checkpoint(ck), queries)
        out["checkpoint_delta2"] = dict(res, query=_pct(lat))

        # parity: the restored store against the live one
        t0 = time.perf_counter()
        back = R.KnowledgeBase.load(ck, enc, capacity=args.chunks + 65536, index_loader=lambda p, cap: Index.load(p, capacity=cap))
        out["restore_s"] = round(time.perf_counter() - t0, 1)

        def live(ix):
            rows, ids, user, org, lv = ix.export_raw()
            keep = lv > 0
            order = np.argsort(ids[keep])
            return rows[keep][order], ids[keep][order], user[keep][order], org[keep][order]
        a, b = live(kb.index), live(back.index)
        same_rows = all(np.array_equal(x, y) for x, y in zip(a, b))
        del a, b
        sample = rng.choice(list(kb._props), size=2000, replace=False).tolist()
        same_props = (len(kb._props) == len(back._props) and kb._key2id == back._key2id
                      and all(kb._props[i] == back._props[i] for i in sample))
        same_answers = all([(o.uuid, o.metadata.score) for o in kb.query(q, 10)] ==
                           [(o.uuid, o.metadata.score) for o in back.query(q, 10)] for q in queries)
        out["parity"] = bool(same_rows and same_props and same_answers)
        out["parity_detail"] = {"rows": same_rows, "props": same_props, "answers": same_answers}
    finally:
        shutil.rmtree(root, ignore_errors=True)
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""Encoder ingest of a multi-GPU knowledge base (one owner process, engine.MultiIndex with one shard per device): the
route through one encoder against aur_encode_append_multi with one encoder replica per shard.  Prints one JSON line.

Workload: bge-base dimensions with random-init weights (seed 7), cfg3's chunk lengths N(384, 96) clipped to [16, 512]
with [CLS] 101 / [SEP] 102 (oracle/bert_encoder.synth_batch), ``--chunks`` chunks per round on every device.

Arms, alternated round by round in one run, each into its own MultiIndex over ``--devices``:
  (a) one encoder on the first device, pooled fp32 vectors to the host, bf16 there, MultiIndex.add (the route a
      multi-GPU knowledge base took before replicas; kept here only as the baseline);
  (b) aur_encode_append_multi with one replica per shard, rows never leaving their device.
Per arm: chunks/s and tokens/s over the timed rounds, and the encoder GEMM FLOP of those rounds computed from the
shapes (2 * tokens * (4 H^2 + 2 H I) * layers).  Parity: every shard's export (rows, ids, codes, live flags) of (a) and
(b) equal bit for bit; the run fails otherwise.

Search latency under ingest: a KnowledgeBase per arm (text in, through the native tokenizer over a synthetic vocabulary
whose pieces are the token ids) ingests documents in a writer thread while the main thread times KnowledgeBase.query.
Arm (a) encodes outside the knowledge-base lock and appends under it; arm (b) encodes and appends under it, as the
single-GPU fused path does.  p50 / p99 in ms, and the number of queries behind them.

With ``--devices 0,0`` (both shards on one GPU) the replicas share that GPU: the run checks parity and no speed-up is
expected.  The card's name, power limit and SM clock are read in the same run.  Needs a GPU: there is no CPU path."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return [[s.strip() for s in line.split(",")] for line in out]
    except Exception as e:  # noqa: BLE001
        return [[f"unknown ({e})", "unknown", "unknown"]]


def gemm_flop(tokens: int, cfg) -> float:
    h, i = cfg.hidden, cfg.inter
    return 2.0 * tokens * (4.0 * h * h + 2.0 * h * i) * cfg.layers


def pct(xs, q):
    return round(float(np.percentile(np.asarray(xs) * 1e3, q)), 3) if xs else None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--devices", default="all", help="'all' or a comma list, e.g. 0,1,2,3 (0,0: two shards on one GPU)")
    ap.add_argument("--chunks", type=int, default=4096, help="chunks per round and device")
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds per arm, alternated")
    ap.add_argument("--max-tokens", type=int, default=32768, help="encoder workspace (tokens) of every replica")
    ap.add_argument("--docs", type=int, default=6, help="documents per arm in the search-latency phase")
    ap.add_argument("--doc-chunks", type=int, default=256, help="chunks per document in the search-latency phase")
    args = ap.parse_args()

    from aurora_b200 import _native as N
    from aurora_b200 import retriever as R
    from aurora_b200.encoder import Encoder, EncoderConfig, TextEncoder, encode_append_multi
    from aurora_b200.engine import MultiIndex, to_bf16_bits
    from aurora_b200.wordpiece import NativeTokenizer
    from oracle import bert_encoder as B

    ndev = N.load().aur_device_count()
    if ndev == 0:
        raise SystemExit("multi_ingest_bench needs a CUDA device (aurora_b200 has no CPU path)")
    devices = list(range(ndev)) if args.devices == "all" else [int(x) for x in args.devices.split(",")]
    n = len(devices)
    cfg_o = B.BGE_BASE
    cfg = EncoderConfig()
    t_init = time.perf_counter()
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    enc = Encoder(cfg, max_tokens=args.max_tokens, max_seqs=2048, device=devices[0])
    enc.load_weights(w)
    del w
    reps = {devices[0]: enc}
    for d in devices:
        if d not in reps:
            reps[d] = enc.replicate(d)
    encs = [reps[d] for d in devices]
    per_round = args.chunks * n
    tok, cu = B.synth_batch(cfg_o, per_round, seed=3)
    seqs = [tok[cu[i]:cu[i + 1]] for i in range(per_round)]
    tokens_per_round = int(cu[-1])
    cap = per_round * (args.rounds + 1)
    ix_a = MultiIndex(cfg.hidden, cap, devices=devices)
    ix_b = MultiIndex(cfg.hidden, cap, devices=devices)

    def arm_a(ids):
        ix_a.add(to_bf16_bits(enc.encode(seqs)), ids)

    def arm_b(ids):
        encode_append_multi(encs, ix_b.shards, tok, cu, ids)

    arms = {"a_one_encoder_host_add": arm_a, "b_replicas_append_multi": arm_b}
    wall = {k: [] for k in arms}
    for r in range(args.rounds + 1):                    # round 0 warms both arms up
        ids = np.arange(r * per_round, (r + 1) * per_round, dtype=np.int64)
        for key, fn in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
            t0 = time.perf_counter()
            fn(ids)                                     # both return once the rows are in their shards
            if r:
                wall[key].append(time.perf_counter() - t0)
    ex_a = [sh.export_raw() for sh in ix_a.shards]
    ex_b = [sh.export_raw() for sh in ix_b.shards]
    parity = all(np.array_equal(x, y) for pa, pb in zip(ex_a, ex_b) for x, y in zip(pa, pb))
    ix_a.close()
    ix_b.close()

    out = {"tool": "multi_ingest_bench", "gpus": [dict(zip(("card", "power_limit", "max_sm_clock"), c)) for c in card()],
           "devices": devices, "model": "bge-base dims, random-init (seed 7)", "chunks_per_round": per_round,
           "tokens_per_round": tokens_per_round, "rounds": args.rounds, "max_tokens": args.max_tokens,
           "setup_s": round(time.perf_counter() - t_init, 1), "parity": bool(parity)}
    for key, ts in wall.items():
        t = float(np.sum(ts))
        out[key] = {"s": round(t, 3), "chunks_per_s": round(per_round * len(ts) / t, 1),
                    "tokens_per_s": round(tokens_per_round * len(ts) / t, 1),
                    "gemm_flop": gemm_flop(tokens_per_round * len(ts), cfg),
                    "gemm_tflop_per_s": round(gemm_flop(tokens_per_round * len(ts), cfg) / t / 1e12, 1)}
    out["speedup_b_over_a"] = round(out["b_replicas_append_multi"]["chunks_per_s"] / out["a_one_encoder_host_add"]["chunks_per_s"], 3)

    # ---- search latency under ingest, through the knowledge base
    pieces = [f"w{i}" for i in range(cfg.vocab)]
    for i, p in ((0, "[PAD]"), (100, "[UNK]"), (101, "[CLS]"), (102, "[SEP]"), (103, "[MASK]")):
        pieces[i] = p
    tk = NativeTokenizer(pieces)
    texts = [" ".join(f"w{t}" for t in s[1:-1]) for s in seqs[:args.doc_chunks * args.docs]]
    queries = texts[:64]

    class HostRoute:        # the encoder as a multi-GPU knowledge base used it before replicas: encode, then index.add
        def __init__(self, te):
            self.dim, self._te = te.dim, te

        def encode(self, t):
            return self._te.encode(t)

    te = TextEncoder(enc, tk)
    te_b = TextEncoder(enc, tk).replicate(devices)
    lat = {}
    for key, encoder in (("a_one_encoder_host_add", HostRoute(te)), ("b_replicas_append_multi", te_b)):
        kb = R.KnowledgeBase(encoder, capacity=len(texts) + 64,
                             index_factory=lambda dim, c: MultiIndex(dim, c, devices=devices))
        kb.insert("u0", "warm", "w.md", [{"chunk_index": 0, "content": texts[0]}])
        kb.query(queries[0], 5, user_id="u0")
        done, times = threading.Event(), []

        def writer():
            try:
                for d in range(args.docs):
                    part = texts[d * args.doc_chunks:(d + 1) * args.doc_chunks]
                    kb.insert(f"u{d % 4}", f"doc{d}", "f.md", [{"chunk_index": c, "content": x} for c, x in enumerate(part)])
            finally:
                done.set()

        th = threading.Thread(target=writer)
        t0 = time.perf_counter()
        th.start()
        i = 0
        while not done.is_set():
            q0 = time.perf_counter()
            kb.query(queries[i % len(queries)], 5, user_id=f"u{i % 4}")
            times.append(time.perf_counter() - q0)
            i += 1
        th.join()
        ingest_s = time.perf_counter() - t0
        lat[key] = {"query_p50_ms": pct(times, 50), "query_p99_ms": pct(times, 99), "queries": len(times),
                    "ingest_s": round(ingest_s, 3), "ingest_chunks_per_s": round(len(texts) / ingest_s, 1)}
        kb.index.close()
    out["search_under_ingest"] = lat
    if len(set(devices)) == 1:
        out["note"] = ("every shard is on one GPU: the replicas share it, so this run checks parity only; "
                       "no speed-up is expected")
    else:
        out["note"] = f"{len(set(devices))} GPUs: (b) encodes every shard's share on its own GPU at once"
    print(json.dumps(out))
    if not parity:
        raise SystemExit("parity failed: the two arms stored different rows")


if __name__ == "__main__":
    main()

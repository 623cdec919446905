"""Ingest of texts longer than the encoder's position table: the host route (windows averaged on the host, then
index.add) against TextEncoder.encode_append (windows, forward, mean and append on the device).  Prints one JSON line.

Workload: bge-base dimensions with random-init weights (seed 7) and a synthetic vocabulary whose pieces "w<id>" are
one token each, so a text's token count is exact.  cfg3's lengths N(384, 96) clipped to [16, 512] ([CLS] and [SEP]
included); a fraction p of the texts gets 513 .. 4 096 tokens instead, and every round with p > 0 adds two texts of
``--huge`` tokens, longer than one workspace batch.  ``--chunks`` texts per round.

Arms, alternated round by round in one run, over an engine.Index and over an engine.MultiIndex of ``--devices``:
  (a) the route before this tool: the texts that fit, truncated at 512, through encode_append_multi; each over-long
      text's windows (its whole tokenisation re-cut in Python) through Encoder.encode in workspace batches, numpy mean
      and norm, and index.add;
  (b) TextEncoder.encode_append: one aur_tokenize_windows and one aur_encode_append_texts_multi call.
Per arm: chunks/s, real tokens/s counting every window's tokens, and GEMM TFLOP/s from the shapes
(2 * tokens * (4 H^2 + 2 H I) * layers).  Query latency under ingest: p50 / p99 of Index.search of 8 bf16 queries in
the main thread while a thread ingests one round.

Check: (b)'s rows equal oracle/window_mean.py applied to Encoder.encode_packed window vectors, bit for bit; the run
fails otherwise.  Reported for information only: the share of rows where (a) and (b) are bit-identical and their
largest difference in bf16 ulps (numpy's mean and BLAS norm are not the device arithmetic).  The card's name, power
limit and SM clock are read in the same run.  Needs a GPU: there is no CPU path."""

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


def pct(xs, q):
    return round(float(np.percentile(np.asarray(xs) * 1e3, q)), 3) if xs else None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--devices", default="all", help="'all' or a comma list for the MultiIndex (one GPU: two shards on it)")
    ap.add_argument("--chunks", type=int, default=1024, help="texts per round")
    ap.add_argument("--rounds", type=int, default=2, help="timed rounds per arm and workload, alternated")
    ap.add_argument("--fractions", default="0,0.1,0.5", help="fractions p of over-long texts")
    ap.add_argument("--huge", type=int, default=40000, help="tokens of the two texts longer than a workspace batch")
    ap.add_argument("--max-tokens", type=int, default=32768, help="encoder workspace (tokens)")
    args = ap.parse_args()

    from aurora_b200 import _native as N
    from aurora_b200.encoder import Encoder, EncoderConfig, TextEncoder, encode_append_multi, pack_sequences
    from aurora_b200.engine import Index, MultiIndex, to_bf16_bits
    from aurora_b200.wordpiece import NativeTokenizer
    from oracle import bert_encoder as B
    from oracle.window_mean import fold_texts

    ndev = N.load().aur_device_count()
    if ndev == 0:
        raise SystemExit("long_text_bench needs a CUDA device (aurora_b200 has no CPU path)")
    devices = list(range(ndev)) if args.devices == "all" else [int(x) for x in args.devices.split(",")]
    if len(devices) == 1:
        devices = devices * 2
    cfg_o, cfg = B.BGE_BASE, EncoderConfig()
    enc = Encoder(cfg, max_tokens=args.max_tokens, max_seqs=2048, device=devices[0])
    enc.load_weights(B.init_weights(cfg_o, seed=7, bf16=True))
    pieces = [f"w{i}" for i in range(cfg.vocab)]
    for i, p in ((0, "[PAD]"), (100, "[UNK]"), (101, "[CLS]"), (102, "[SEP]"), (103, "[MASK]")):
        pieces[i] = p
    tk = NativeTokenizer(pieces)
    te = TextEncoder(enc, tk).replicate(sorted(set(devices)))
    step = cfg.max_pos - 2

    def texts_for(p, seed):
        rng = np.random.default_rng(seed)
        n = args.chunks
        lens = np.clip(np.rint(rng.normal(384, 96, n)), 16, 512).astype(np.int64)
        long = rng.random(n) < p
        lens[long] = rng.integers(513, 4097, int(long.sum()))
        if p > 0:
            lens[:2] = args.huge
        return [" ".join(f"w{t}" for t in rng.integers(1000, cfg.vocab, int(L) - 2)) for L in lens]

    def arm_a(index, texts, ids):
        tok, cu = tk.encode_packed(texts, cfg.max_pos)
        lens = np.diff(cu)
        cand = np.nonzero(lens >= cfg.max_pos)[0]
        full = tk.lengths([texts[i] for i in cand], max_len=0x7FFFFFFF) if len(cand) else np.zeros(0, np.int64)
        long = cand[full > cfg.max_pos]
        keep = np.ones(len(texts), bool)
        keep[long] = False
        c = np.zeros(int(keep.sum()) + 1, np.int32)
        np.cumsum(lens[keep], out=c[1:])
        shards = list(index.shards) if isinstance(index, MultiIndex) else [index]
        encode_append_multi([te._encs[sh.device] for sh in shards], shards, tok[np.repeat(keep, lens)], c, ids[keep])
        if len(long):
            wins, owner = [], []
            for t, i in enumerate(long):
                ft, fc = tk.encode_packed([texts[i]], int(tk.lengths([texts[i]], max_len=0x7FFFFFFF)[0]))
                body = ft[1:-1]
                w = [np.concatenate(([ft[0]], body[k:k + step], [ft[-1]])).astype(np.int32) for k in range(0, len(body), step)]
                wins += w
                owner += [t] * len(w)
            vecs = enc.encode(wins)
            owner = np.asarray(owner)
            out = np.empty((len(long), cfg.hidden), np.float32)
            for t in range(len(long)):
                v = vecs[owner == t].mean(axis=0)
                out[t] = v / float(np.linalg.norm(v))
            index.add(out, ids[long])

    def arm_b(index, texts, ids):
        te.encode_append(index, texts, ids)

    def rows_of(index):
        out = {}
        for sh in (index.shards if isinstance(index, MultiIndex) else [index]):
            rows, rid, _, _, live = sh.export_raw()
            for r, i, lv in zip(rows, rid, live):
                if lv:
                    out[int(i)] = r
        return out

    arms = {"a_host_windows": arm_a, "b_device_windows": arm_b}
    results, ok = [], True
    qv = None
    for p in [float(x) for x in args.fractions.split(",")]:
        for kind in ("Index", "MultiIndex"):
            cap = args.chunks * (args.rounds + 1) + 64
            ix = {k: (Index(cfg.hidden, cap, device=devices[0]) if kind == "Index" else MultiIndex(cfg.hidden, cap, devices=devices))
                  for k in arms}
            wall = {k: [] for k in arms}
            lat = {k: [] for k in arms}
            win_tokens = chunks = 0
            last = None
            for r in range(args.rounds + 1):                                   # round 0 warms both arms up
                texts = texts_for(p, 1000 * r + int(p * 100))
                ids = np.arange(r * args.chunks, (r + 1) * args.chunks, dtype=np.int64)
                if r:
                    tok, cu, ct = tk.encode_windows(texts, cfg.max_pos)
                    win_tokens += int(cu[-1])
                    chunks += len(texts)
                    last = (texts, ids, tok, cu, ct)
                for key, fn in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
                    if qv is None:
                        qv = to_bf16_bits(te.encode(texts[2:10]))
                    done = threading.Event()

                    def run():
                        try:
                            fn(ix[key], texts, ids)
                        finally:
                            done.set()
                    th = threading.Thread(target=run)
                    t0 = time.perf_counter()
                    th.start()
                    while not done.is_set():
                        q0 = time.perf_counter()
                        ix[key].search(qv, 10)
                        if r:
                            lat[key].append(time.perf_counter() - q0)
                    th.join()
                    if r:
                        wall[key].append(time.perf_counter() - t0)
            # check (b) against the oracle on the last round; compare (a) for information
            texts, ids, tok, cu, ct = last
            vecs = enc.encode([tok[cu[i]:cu[i + 1]] for i in range(len(cu) - 1)])
            want = to_bf16_bits(fold_texts(vecs, ct, cfg.normalize))
            rb, ra = rows_of(ix["b_device_windows"]), rows_of(ix["a_host_windows"])
            got_b = np.stack([rb[int(i)] for i in ids])
            got_a = np.stack([ra[int(i)] for i in ids])
            parity = bool(np.array_equal(got_b, want))
            ok &= parity
            same = np.all(got_a == got_b, axis=1)
            ulps = np.abs(got_a.view(np.int16).astype(np.int32) - got_b.view(np.int16).astype(np.int32)).max()
            res = {"p": p, "index": kind, "devices": devices if kind == "MultiIndex" else devices[:1], "chunks": chunks,
                   "window_tokens": win_tokens, "over_long": int(np.sum(np.diff(ct) > 1) * args.rounds),
                   "b_equals_oracle": parity, "a_b_identical_rows": round(float(same.mean()), 4),
                   "a_b_max_bf16_ulps": int(ulps)}
            for key in arms:
                t = float(np.sum(wall[key]))
                flop = 2.0 * win_tokens * (4.0 * cfg.hidden ** 2 + 2.0 * cfg.hidden * cfg.inter) * cfg.layers
                res[key] = {"s": round(t, 3), "chunks_per_s": round(chunks / t, 1), "tokens_per_s": round(win_tokens / t, 1),
                            "gemm_tflop_per_s": round(flop / t / 1e12, 1), "query_p50_ms": pct(lat[key], 50),
                            "query_p99_ms": pct(lat[key], 99), "queries": len(lat[key])}
            results.append(res)
            for x in ix.values():
                x.close()
    out = {"tool": "long_text_bench", "gpus": [dict(zip(("card", "power_limit", "max_sm_clock"), c)) for c in card()],
           "model": "bge-base dims, random-init (seed 7)", "max_tokens": args.max_tokens, "rounds": args.rounds,
           "huge_tokens": args.huge, "results": results, "parity": bool(ok)}
    print(json.dumps(out))
    if not ok:
        raise SystemExit("parity failed: TextEncoder.encode_append's rows differ from the window-mean oracle")


if __name__ == "__main__":
    main()

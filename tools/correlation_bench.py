"""Alert correlation's title similarity: the reference's call pattern against one device call per alert and per storm.
Prints one JSON line.

Workload: bge-base dimensions with random-init weights (seed 7), a synthetic vocabulary whose pieces "w<id>" are one
token each (as bench.py's text leg builds it), alert and incident titles of 6 .. 16 words, 20 candidates per alert
drawn from a pool of ``--incidents`` open incidents (so titles repeat across alerts, as in a storm), one service each.
Every 10th candidate has a blank title or one longer than the position table: ``embed`` answers None for it and its
title is scored by Jaccard on every arm.

Arms (SimilarityStrategy over encoder.EmbeddingClient, aurora_b200/correlation.py):
  (a) ``score`` per candidate: two ``embed`` calls (one aur_encode_texts forward each) and a Python cosine, as
      AlertCorrelator._score_candidate runs it today;
  (b) ``score_many`` per alert: one ``similarities`` call (one aur_encode_pair_cosines call);
  (c) ``score_alerts`` over storms of 1, 16 and 256 alerts: one call per storm.
Per arm: ms per alert, alerts/s, library calls and kernel launches per alert (forward launches counted per workspace
batch, plus the gather launch).  Parity: the largest |score difference| of (b) and (c) against (a) over the alerts (a)
ran (<= 1e-12), and every fallback candidate's score equal to (a)'s.  The card's name, power limit and SM clock are read
in the same run.  Needs a GPU: there is no CPU path."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--alerts-a", type=int, default=16, help="alerts through arm (a), the reference pattern (slow)")
    ap.add_argument("--alerts-b", type=int, default=64, help="alerts through arm (b)")
    ap.add_argument("--storms", default="1,16,256", help="storm sizes of arm (c)")
    ap.add_argument("--incidents", type=int, default=200, help="open incidents the candidates are drawn from")
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of arms (b) and (c)")
    ap.add_argument("--max-tokens", type=int, default=32768, help="encoder workspace (tokens)")
    ap.add_argument("--max-seqs", type=int, default=2048, help="encoder workspace (sequences)")
    args = ap.parse_args()

    from aurora_b200 import _native as N
    from aurora_b200 import encoder as E
    from aurora_b200.correlation import SimilarityStrategy
    from aurora_b200.wordpiece import NativeTokenizer
    from oracle import bert_encoder as B

    if N.load().aur_device_count() == 0:
        raise SystemExit("correlation_bench needs a CUDA device (aurora_b200 has no CPU path)")
    cfg = E.EncoderConfig()
    enc = E.Encoder(cfg, max_tokens=args.max_tokens, max_seqs=args.max_seqs)
    enc.load_weights(B.init_weights(B.BGE_BASE, seed=7, bf16=True))
    pieces = [f"w{i}" for i in range(cfg.vocab)]
    for i, p in ((0, "[PAD]"), (100, "[UNK]"), (101, "[CLS]"), (102, "[SEP]"), (103, "[MASK]")):
        pieces[i] = p
    tk = NativeTokenizer(pieces)
    # the whole text, not cut at max_pos: embed (and similarities) answer None for a longer one
    client = E.EmbeddingClient(enc, lambda text: tk.encode(text, int(tk.lengths([text], max_len=0x7FFFFFFF)[0])))
    E.configure_embedding_client(lambda: client)

    # count library calls and forward batches (each batch is one forward of `fwd` launches)
    count = {"calls": 0, "batches": 0, "gathers": 0}

    def batches(cu):
        n, toks, seqs = 0, 0, 0
        for L in np.diff(cu):
            if seqs == 0 or toks + L > args.max_tokens or seqs + 1 > args.max_seqs:
                n, toks, seqs = n + 1, 0, 0
            toks, seqs = toks + int(L), seqs + 1
        return n

    enc_texts, pair_cos = enc.encode_texts, enc.pair_cosines

    def counted_texts(tok, cu, ct, bf16=False):
        count["calls"] += 1
        count["batches"] += batches(cu)
        return enc_texts(tok, cu, ct, bf16)

    def counted_pairs(tok, cu, ct, pa, pb, clamp=True, vectors=False):
        count["calls"] += 1
        count["batches"] += batches(cu)
        count["gathers"] += int(len(pa) > 0)
        return pair_cos(tok, cu, ct, pa, pb, clamp=clamp, vectors=vectors)

    enc.encode_texts, enc.pair_cosines = counted_texts, counted_pairs
    enc.encode([[101, 2000, 102]])
    fwd = enc.stats()["launches"]

    rng = np.random.default_rng(7)

    def title():
        return " ".join(f"w{t}" for t in rng.integers(1000, cfg.vocab, int(rng.integers(6, 17))))

    incidents = [(title(), [f"svc-{rng.integers(0, 30)}"]) for _ in range(args.incidents)]
    for k in range(0, args.incidents, 10):                                      # embed answers None for these
        incidents[k] = ("   ", incidents[k][1]) if k % 20 == 0 else (" ".join(["w2000"] * 600), incidents[k][1])
    storms = [int(x) for x in args.storms.split(",")]
    n_alerts = max([args.alerts_a, args.alerts_b] + storms)
    alerts = [(title(), f"svc-{rng.integers(0, 30)}", [incidents[i] for i in rng.choice(args.incidents, 20, replace=False)])
              for _ in range(n_alerts)]
    fallback = [[not c[0].strip() or len(c[0].split()) > 500 for c in cands] for _, _, cands in alerts]
    strat = SimilarityStrategy()

    def run(fn, items, reps):
        for k in count:
            count[k] = 0
        t0 = time.perf_counter()
        for _ in range(reps):
            out = fn(items)
        return out, time.perf_counter() - t0, {k: v / reps for k, v in count.items()}

    arms = {
        "a_score_per_candidate": lambda items: [[strat.score(t, s, c[0], c[1]) for c in cands] for t, s, cands in items],
        "b_score_many_per_alert": lambda items: [strat.score_many(t, s, cands) for t, s, cands in items],
    }
    for m in storms:
        arms[f"c_score_alerts_storm_{m}"] = (lambda m: lambda items: sum((strat.score_alerts(items[i:i + m])
                                                                          for i in range(0, len(items), m)), []))(m)
    n_for = {"a_score_per_candidate": args.alerts_a, "b_score_many_per_alert": args.alerts_b}
    results, scores = {}, {}
    for key, fn in arms.items():
        n = n_for.get(key) or max(int(key.rsplit("_", 1)[1]), args.alerts_a)
        fn(alerts[:min(n, 2)])                                                 # warm-up
        reps = 1 if key.startswith("a_") else args.reps
        out, sec, cnt = run(fn, alerts[:n], reps)
        sec /= reps
        scores[key] = out
        results[key] = {"alerts": n, "reps": reps, "ms_per_alert": round(sec * 1e3 / n, 3), "alerts_per_s": round(n / sec, 1),
                        "calls_per_alert": round(cnt["calls"] / n, 3),
                        "launches_per_alert": round((cnt["batches"] * fwd + cnt["gathers"]) / n, 2)}
    ref = np.array(sum(scores["a_score_per_candidate"], []))
    fb = np.array(sum(fallback[:args.alerts_a], []))
    max_d, fallback_ok = 0.0, True
    for key, out in scores.items():
        got = np.array(sum(out[:args.alerts_a], []))
        d = float(np.max(np.abs(got - ref)))
        results[key]["max_abs_diff_vs_a"] = d
        max_d = max(max_d, d)
        fallback_ok &= bool(np.array_equal(got[fb], ref[fb]))
    parity = max_d <= 1e-12 and fallback_ok
    print(json.dumps({"tool": "correlation_bench", "gpus": [dict(zip(("card", "power_limit", "max_sm_clock"), c)) for c in card()],
                      "model": "bge-base dims, random-init (seed 7)", "forward_launches": fwd, "candidates_per_alert": 20,
                      "fallback_pairs_checked": int(fb.sum()), "results": results, "max_abs_diff": max_d,
                      "fallback_equal": fallback_ok, "parity": parity}))
    if not parity:
        raise SystemExit("parity failed: batched scores differ from the reference call pattern")


if __name__ == "__main__":
    main()

"""Per-query pre-filter lists (Index.search_lists) against the full-shard filtered paths, on the cfg2 corpus
(1M x 768 bf16, the seed bench.py uses).  Prints one JSON line.

Workloads:
  (a) one query, list of 100 / 1k / 10k / 100k / 1M rows: search_lists vs search_subset (mask + full scan);
  (b) 256 queries over 64 tenants of 2 000 rows each: search_lists with 64 lists vs aur_search with per-query tenant codes
      (64 scopes > 32, so the generic kernel today);
  (c) 256 queries sharing one 100k-row list: search_lists vs search_subset.
Per call: device ms (aur_stats.last_total_ms) and wall ms, medians of --calls calls after warm-up; gathered bytes from
shapes = listed rows x (dim * 2 + 8) per 64-query group, and their share of 3.35 TB/s over the device time; parity = the
ids of sampled queries bit-exact against oracle.cosine_topk over exactly the allowed rows.  The card's name and power
limit are read in the same run.  Needs a GPU: there is no CPU fallback."""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import _native as N                      # noqa: E402
from aurora_b200.engine import Index                      # noqa: E402
from oracle import cosine_topk as O                       # noqa: E402

HBM_BPS = 3.35e12
ROWS, DIM, SEED, QSEED, CHUNK, K = 1_000_000, 768, 1002, 2002, 125_000, 32
TENANTS, TENANT_MOD = 64, 500                              # tenant t = the ids with id % 500 == t: 2 000 rows each


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def timed(ix, fn, calls, warmup=3):
    for _ in range(warmup):
        fn()
    wall, dev = [], []
    for _ in range(calls):
        t0 = time.perf_counter()
        out = fn()
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(ix.stats()["last_total_ms"])
    return out, float(np.median(dev)), float(np.median(wall)), ix.stats()["last_kernel"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rows", type=int, default=ROWS)
    ap.add_argument("--sample", type=int, default=3, help="queries per workload checked against the oracle")
    args = ap.parse_args()
    if N.load().aur_device_count() == 0:
        raise SystemExit("list_bench needs a CUDA device (aurora_b200 has no CPU path)")
    import torch

    dev = torch.device("cuda:0")
    n = args.rows
    ix = Index(DIM, n + 64)
    host = []                                              # bf16 corpus on the host for the oracle
    for g, lo in enumerate(range(0, n, CHUNK)):
        m = min(CHUNK, n - lo)
        rows = torch.randn(m, DIM, generator=torch.Generator(device=dev).manual_seed(SEED + g), device=dev,
                           dtype=torch.float32).to(torch.bfloat16)
        ids = np.arange(lo, lo + m, dtype=np.int64)
        ix.add_dev(rows.data_ptr(), m, ids, user_codes=(ids % TENANT_MOD).astype(np.int32),
                   org_codes=np.full(m, -1, np.int32))
        host.append(rows.cpu())
        torch.cuda.synchronize()
    host = torch.cat(host)
    Qall = torch.randn(256, DIM, generator=torch.Generator(device=dev).manual_seed(QSEED), device=dev,
                       dtype=torch.float32).to(torch.bfloat16).cpu().view(torch.int16).numpy().view(np.uint16)
    Qf = O.round_to_bf16(torch.from_numpy(Qall.view(np.int16)).view(torch.bfloat16).float().numpy())
    rng = np.random.default_rng(7)
    parity = True

    def check(ids, qsel, allowed):
        nonlocal parity
        allowed = np.sort(np.asarray(allowed, dtype=np.int64))
        Csub = host[torch.from_numpy(allowed)].float().numpy()
        want, _ = O.cosine_topk(Qf[qsel], Csub, K, ids=allowed)
        ok = bool(np.array_equal(ids[: len(qsel)], want))
        parity &= ok
        return ok

    def gathered(list_rows, groups):
        return int(list_rows) * (DIM * 2 + 8) * int(groups)

    def row(name, ms_dev, ms_wall, kernel, nbytes=None):
        r = {"path": name, "device_ms": round(ms_dev, 4), "wall_ms": round(ms_wall, 4), "kernel": N.KERNEL_NAMES.get(kernel)}
        if nbytes is not None:
            r["gathered_bytes"] = nbytes
            r["hbm_share"] = round(nbytes / (ms_dev * 1e-3) / HBM_BPS, 4) if ms_dev > 0 else None
        return r

    out = {"tool": "list_bench", "rows": n, "dim": DIM, "k": K, "calls": args.calls}
    # (a) one query
    wa = []
    for size in (100, 1_000, 3_000, 10_000, 30_000, 100_000, 1_000_000):
        size = min(size, n)
        lst = rng.choice(n, size=size, replace=False).astype(np.int64)
        q = Qall[:1]
        (ids_l, sc_l), ld, lw, lk = timed(ix, lambda: ix.search_lists(q, K, [lst], np.zeros(1, np.int32)), args.calls)
        (ids_s, sc_s), sd, sw, sk = timed(ix, lambda: ix.search_subset(q, K, lst), args.calls)
        same = bool(np.array_equal(ids_l, ids_s) and np.array_equal(sc_l, sc_s))
        ok = check(ids_l, [0], lst)
        parity &= same
        wa.append({"list_rows": size, "lists": row("search_lists", ld, lw, lk, gathered(size, 1)),
                   "subset": row("search_subset", sd, sw, sk), "parity": ok and same})
    out["a_single_query"] = wa
    # (b) 64 tenants, 4 queries each
    q_list = np.repeat(np.arange(TENANTS, dtype=np.int32), 256 // TENANTS)
    all_ids = np.arange(n, dtype=np.int64)
    lists = [all_ids[all_ids % TENANT_MOD == t] for t in range(TENANTS)]
    (ids_l, sc_l), ld, lw, lk = timed(ix, lambda: ix.search_lists(Qall, K, lists, q_list), args.calls)
    (ids_c, sc_c), cd, cw, ck = timed(ix, lambda: ix.search(Qall, K, q_list.astype(np.int32), np.full(256, -1, np.int32)),
                                      args.calls)
    ok_b = all(check(ids_l[[q]], [q], lists[q_list[q]]) for q in rng.choice(256, args.sample, replace=False))
    same_b = bool(np.array_equal(ids_l, ids_c))
    parity &= same_b
    out["b_many_tenants"] = {"queries": 256, "lists": TENANTS, "list_rows": int(len(lists[0])),
                             "lists_path": row("search_lists", ld, lw, lk, gathered(sum(len(x) for x in lists), 1)),
                             "tenant_codes": row("search", cd, cw, ck), "parity": ok_b and same_b}
    # (c) one shared 100k list
    lst = rng.choice(n, size=min(100_000, n), replace=False).astype(np.int64)
    (ids_l, sc_l), ld, lw, lk = timed(ix, lambda: ix.search_lists(Qall, K, [lst], np.zeros(256, np.int32)), args.calls)
    (ids_s, sc_s), sd, sw, sk = timed(ix, lambda: ix.search_subset(Qall, K, lst), args.calls)
    ok_c = all(check(ids_l[[q]], [q], lst) for q in rng.choice(256, args.sample, replace=False))
    same_c = bool(np.array_equal(ids_l, ids_s) and np.array_equal(sc_l, sc_s))
    parity &= same_c
    out["c_shared_list"] = {"queries": 256, "list_rows": int(len(lst)),
                            "lists_path": row("search_lists", ld, lw, lk, gathered(len(lst), 4)),
                            "subset": row("search_subset", sd, sw, sk), "parity": ok_c and same_c}
    out["parity"] = parity
    out["card"], out["power_limit"] = card()
    print(json.dumps(out), flush=True)
    ix.close()
    if not parity:
        raise SystemExit(1)


if __name__ == "__main__":
    main()

"""Growth of a vector shard in place (aur_reserve) on bench.py's cfg2 shape.  Prints one JSON line with the card's name
and power limit read in the same run:

- growth: milliseconds aur_reserve takes per +1M rows of 768-dim bf16 (three growths of 1M rows each on a fresh shard);
- kernel: the cfg2 similarity kernel (1M x 768 bf16 rows from seed 1002, 256 queries from seed 2002, top-32) on a shard
  grown from 1,000 rows in 65,536-row steps against one opened at 1M, both in this process and timed alternately with
  CUDA events around `--launches` back-to-back aur_search_dev calls; their ids and scores must be identical;
- under growth: p50 / p99 host latency of aur_search at nq = 1 and nq = 256 with no writer, and while a writer thread
  only appends, only grows, or grows and appends, 65,536 rows at a time.

Needs a GPU: there is no CPU fallback."""

from __future__ import annotations

import argparse
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import _native as N                      # noqa: E402
from aurora_b200.engine import GROW_STEP, Index           # noqa: E402
from tools.int8_bench import card                         # noqa: E402

ROWS, DIM, NQ, K = 1_000_000, 768, 256, 32


def _fill(torch, ix_list, lo, hi, seed):
    dev = torch.device("cuda:0")
    for g, a in enumerate(range(lo, hi, GROW_STEP)):
        m = min(GROW_STEP, hi - a)
        rows = torch.randn(m, DIM, generator=torch.Generator(device=dev).manual_seed(seed + a), device=dev,
                           dtype=torch.float32).to(torch.bfloat16)
        torch.cuda.synchronize()                         # the shards' ingest streams do not wait for torch's stream
        for ix in ix_list:
            if ix.stats()["capacity"] < a + m:
                ix.reserve(a + GROW_STEP)
            ix.add_dev(rows.data_ptr(), m, np.arange(a, a + m, dtype=np.int64))
        torch.cuda.synchronize()


def growth_ms():
    with Index(DIM, 1000) as ix:
        out = []
        for step in range(1, 4):
            t0 = time.perf_counter()
            ix.reserve(step * ROWS)
            out.append((time.perf_counter() - t0) * 1e3)
    return out


def kernel_ms(torch, grown, opened, launches, rounds):
    dev = torch.device("cuda:0")
    q = torch.randn(NQ, DIM, generator=torch.Generator(device=dev).manual_seed(2002), device=dev,
                    dtype=torch.float32).to(torch.bfloat16)
    outs = {}
    for name, ix in (("grown", grown), ("opened", opened)):
        outs[name] = (torch.empty(NQ, K, dtype=torch.float32, device=dev), torch.empty(NQ, K, dtype=torch.int64, device=dev))
        for _ in range(5):
            ix.search_dev(q.data_ptr(), NQ, K, outs[name][0].data_ptr(), outs[name][1].data_ptr())
        ix.sync()
    times = {"grown": [], "opened": []}
    for _ in range(rounds):
        for name, ix in (("grown", grown), ("opened", opened)):
            s = torch.cuda.Stream()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s):
                e0.record(s)
                for _ in range(launches):
                    ix.search_dev(q.data_ptr(), NQ, K, outs[name][0].data_ptr(), outs[name][1].data_ptr(), stream=s.cuda_stream)
                e1.record(s)
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / launches)
    same = bool(torch.equal(outs["grown"][0], outs["opened"][0]) and torch.equal(outs["grown"][1], outs["opened"][1]))
    kern = N.KERNEL_NAMES.get(grown.stats()["last_kernel"])
    return {name: {"median_ms": round(float(np.median(v)), 4), "min_ms": round(float(np.min(v)), 4),
                   "max_ms": round(float(np.max(v)), 4)} for name, v in times.items()} | {"outputs_identical": same,
                                                                                            "kernel": kern}


def latency(torch, ix, calls, writer_rows):
    """Search latency with no writer, then with a writer that only appends (its capacity reserved beforehand), only
    grows (aur_reserve in 65,536-row steps, nothing appended) and grows and appends -- so that a tail can be told apart
    by its cause.  The writer appends one batch made on the GPU before any timing (the same rows under new ids), so it
    adds no torch work or device-wide synchronisation of its own to the window."""
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(7)
    q = rng.standard_normal((NQ, DIM)).astype(np.float32)
    batch = torch.randn(GROW_STEP, DIM, generator=torch.Generator(device=dev).manual_seed(9000), device=dev,
                        dtype=torch.float32).to(torch.bfloat16)
    torch.cuda.synchronize()
    res = {}
    for mode in ("idle", "append", "grow", "grow_append"):
        steps = writer_rows // GROW_STEP
        if mode == "append":
            ix.reserve(ix.stats()["rows"] + steps * GROW_STEP)
        stop, errs, done = threading.Event(), [], [0]

        def writer():
            try:
                for _ in range(steps):
                    if stop.is_set():
                        break
                    st = ix.stats()
                    if mode in ("grow", "grow_append"):
                        ix.reserve(max(st["rows"], st["capacity"]) + GROW_STEP)
                    if mode in ("append", "grow_append"):
                        a = st["rows"]
                        ix.add_dev(batch.data_ptr(), GROW_STEP, np.arange(a, a + GROW_STEP, dtype=np.int64))
                    done[0] += 1
            except Exception as e:   # noqa: BLE001
                errs.append(repr(e))

        th = threading.Thread(target=writer) if mode != "idle" else None
        if th:
            th.start()
        for nq in (1, NQ):
            lat = []
            for _ in range(calls):
                t0 = time.perf_counter()
                ix.search(q[:nq], K)
                lat.append((time.perf_counter() - t0) * 1e3)
            res[f"{mode}_nq{nq}"] = {"p50_ms": round(float(np.percentile(lat, 50)), 4),
                                     "p99_ms": round(float(np.percentile(lat, 99)), 4),
                                     "max_ms": round(float(np.max(lat)), 4)}
        stop.set()
        if th:
            th.join()
            res[f"{mode}_writer_steps"] = done[0]
        if errs:
            raise RuntimeError(errs[0])
    res["rows_after"] = int(ix.stats()["rows"])
    res["capacity_after"] = int(ix.stats()["capacity"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=300, help="searches per latency percentile")
    ap.add_argument("--writer-rows", type=int, default=1 << 21, help="rows a writer grows or appends per latency mode")
    args = ap.parse_args()
    import torch

    if N.load().aur_device_count() == 0:
        raise SystemExit("grow_bench needs a CUDA device (aurora_b200 has no CPU path)")
    name, power = card()
    out = {"tool": "grow_bench", "card": name, "power_limit": power, "rows": ROWS, "dim": DIM, "nq": NQ, "k": K}
    out["reserve_ms_per_1M_rows"] = [round(v, 3) for v in growth_ms()]
    grown, opened = Index(DIM, 1000), Index(DIM, ROWS)
    _fill(torch, [grown, opened], 0, ROWS, 1002)
    assert grown.stats()["rows"] == opened.stats()["rows"] == ROWS
    out["grown_capacity"] = int(grown.stats()["capacity"])
    out["kernel"] = kernel_ms(torch, grown, opened, args.launches, args.rounds)
    opened.close()
    out["latency"] = latency(torch, grown, args.calls, args.writer_rows)
    grown.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

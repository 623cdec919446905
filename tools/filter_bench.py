"""Metadata pre-filters evaluated on the device (Index.search_filtered) against the host-resolved path the retriever takes
without them (the Python predicate over the org's rows, then Index.search_lists / search_subset with the allowed ids), on
the cfg2 corpus (1M x 768 bf16, the seed bench.py uses), k = 32.  Prints one JSON line.

Workloads: orgs of 1k / 10k / 100k / 1M rows, half of each org's rows under a "discovery:" document id, the
prediscovery filter `org_id == o AND document_id LIKE "discovery:*"` (rca_prompt_builder.py:286-298), one query and 256
queries.  Both paths pick list kernels or the masked scan by the retriever's rule (allowed rows <= 0.5 % of the shard),
so they run the same similarity kernels.  Per call: device ms (aur_stats.last_total_ms; the device path's includes its
filter kernels) and wall ms (host path: predicate + id resolution + search; device path: program compile + search),
medians after warm-up.  parity = ids and float32 scores bit-identical between the paths, and the 1k org's answer equal to
oracle.cosine_topk over its matching rows.  The card's name and power limit are read in the same run.  Needs a GPU."""

from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aurora_b200 import _native as N                      # noqa: E402
from aurora_b200.engine import Index                      # noqa: E402
from aurora_b200.filters import AttrColumn, Filter, compile_program   # noqa: E402
from oracle import cosine_topk as O                       # noqa: E402
from tools.list_bench import CHUNK, DIM, K, QSEED, ROWS, SEED, card   # noqa: E402

LIST_MAX_FRACTION = 0.005                                  # retriever._LIST_MAX_FRACTION
ORGS = (1_000, 10_000, 100_000)                            # disjoint orgs at the front of the shard; the 1M org is "tier"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rows", type=int, default=ROWS)
    args = ap.parse_args()
    if N.load().aur_device_count() == 0:
        raise SystemExit("filter_bench needs a CUDA device (aurora_b200 has no CPU path)")
    import torch

    dev = torch.device("cuda:0")
    n = args.rows
    ix = Index(DIM, n + 64)
    host = []
    for g, lo in enumerate(range(0, n, CHUNK)):
        m = min(CHUNK, n - lo)
        rows = torch.randn(m, DIM, generator=torch.Generator(device=dev).manual_seed(SEED + g), device=dev,
                           dtype=torch.float32).to(torch.bfloat16)
        ix.add_dev(rows.data_ptr(), m, np.arange(lo, lo + m, dtype=np.int64))
        host.append(rows.cpu())
        torch.cuda.synchronize()
    host = torch.cat(host)
    Qall = torch.randn(256, DIM, generator=torch.Generator(device=dev).manual_seed(QSEED), device=dev,
                       dtype=torch.float32).to(torch.bfloat16).cpu().view(torch.int16).numpy().view(np.uint16)
    Qf = O.round_to_bf16(torch.from_numpy(Qall.view(np.int16)).view(torch.bfloat16).float().numpy())

    # the metadata table and its columns, as retriever.KnowledgeBase keeps them
    bounds = np.cumsum((0,) + ORGS)
    props, pools = [], {}
    for i in range(n):
        o = int(np.searchsorted(bounds, i, side="right")) - 1
        p = {"document_id": f"discovery:{i}" if i % 2 else f"doc:{i}", "tier": "all"}
        if o < len(ORGS):
            p["org_id"] = f"org{ORGS[o]}"
            pools.setdefault(p["org_id"], []).append(i)
        props.append(p)
    pools["all"] = list(range(n))
    cols = {nm: AttrColumn(nm, 2 + j) for j, nm in enumerate(("org_id", "document_id", "tier"))}
    ids_all = np.arange(n, dtype=np.int64)
    for c in cols.values():
        ix.set_attrs(c.col, ids_all, np.array([c.code(p) for p in props], np.int32))
    max_list = int(LIST_MAX_FRACTION * n)

    def timed(fn, calls):
        fn()
        fn()
        wall, devms = [], []
        for _ in range(calls):
            t0 = time.perf_counter()
            out = fn()
            wall.append((time.perf_counter() - t0) * 1e3)
            devms.append(ix.stats()["last_total_ms"])
        return out, round(float(np.median(devms)), 4), round(float(np.median(wall)), 4), N.KERNEL_NAMES[ix.stats()["last_kernel"]]

    parity = True
    work = []
    for size in ORGS + (n,):
        if size > n:
            continue
        if size == n:
            f, pool = Filter.by_property("tier").equal("all"), pools["all"]
        else:
            f, pool = Filter.by_property("org_id").equal(f"org{size}"), pools[f"org{size}"]
        f = f & Filter.by_property("document_id").like("discovery:*")
        for nq in (1, 256):
            Q = Qall[:nq]

            def host_path():
                allowed = np.asarray([rid for rid in pool if f.matches(props[rid])], dtype=np.int64)
                if len(allowed) <= max_list:
                    return ix.search_lists(Q, K, [allowed], np.zeros(nq, np.int32)), len(allowed)
                return ix.search_subset(Q, K, allowed), len(allowed)

            def device_path():
                ids_, sc_, m, _ = ix.search_filtered(Q, K, [compile_program(f, cols)], max_list_rows=max_list)
                return (ids_, sc_), int(m[0])

            calls = args.calls if size <= 100_000 else max(3, args.calls // 3)
            ((h_ids, h_sc), h_m), hd, hw, hk = timed(host_path, calls)
            ((d_ids, d_sc), d_m), dd, dw, dk = timed(device_path, args.calls)
            ok = bool(h_m == d_m and np.array_equal(h_ids, d_ids) and np.array_equal(h_sc.view(np.uint32), d_sc.view(np.uint32)))
            if size == ORGS[0]:
                allowed = np.asarray([rid for rid in pool if f.matches(props[rid])], dtype=np.int64)
                want, _ = O.cosine_topk(Qf[:nq], host[torch.from_numpy(allowed)].float().numpy(), K, ids=allowed)
                ok &= bool(np.array_equal(d_ids, want))
            parity &= ok
            work.append({"org_rows": size, "matched": d_m, "queries": nq,
                         "host_resolved": {"device_ms": hd, "wall_ms": hw, "kernel": hk},
                         "device_filter": {"device_ms": dd, "wall_ms": dw, "kernel": dk}, "parity": ok})
    out = {"tool": "filter_bench", "rows": n, "dim": DIM, "k": K, "calls": args.calls, "max_list_rows": max_list,
           "workloads": work, "parity": parity}
    out["card"], out["power_limit"] = card()
    print(json.dumps(out), flush=True)
    ix.close()
    if not parity:
        raise SystemExit(1)


if __name__ == "__main__":
    main()

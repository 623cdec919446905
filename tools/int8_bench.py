"""int8 shards (AUR_I8) against bf16 shards on bench.py's cfg2 shape: 1M x 768 rows from seed 1002, 256 queries from
seed 2002, top-32 (and, with --cfg4, cfg4's per-GPU shape: 1.25M x 1024 rows from seed 1004, 1024 queries from seed
2004, top-100).  Prints one JSON line.

The same bf16 rows go into a bf16 shard and an int8 shard; the two are timed alternately in one run through
aur_search_dev on the same device queries.  Per format: median kernel ms (aur_stats.last_kernel_ms: the similarity
kernels of the first block of queries), median step ms (host clock around the call and a synchronise) and q/s, the
kernel that served it, algorithmic bytes of one scan (rows x dim x bytes per element) and their share of 3.35 TB/s over
the kernel time, the tensor share (MMA operations over the kernel time against 989 TFLOP/s bf16 / 1,979 TOPS int8, the int8
kernel counted with its two s8 MMAs per product), and the shard's row bytes.  Parity: the int8 shard's ids and scores bit-exact against its bf16 twin (a
bf16 shard fed the int8 rows) for every query, and ids bit-exact against oracle.cosine_topk over the int8 rows for a
sample.  recall@k of the int8 answers against the bf16 shard's answers is information, not a check.  The card's name
and power limit are read in the same run.  Needs a GPU: there is no CPU fallback."""

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
from aurora_b200.engine import DeviceBuffer, Index        # noqa: E402
from oracle import cosine_topk as O                       # noqa: E402
from oracle import quantize as Qz                         # noqa: E402

HBM_BPS = 3.35e12
BF16_OPS, S8_OPS = 989e12, 1979e12     # H100 SXM data sheet, dense, 700 W
CHUNK = 125_000
SHAPES = {"cfg2": dict(rows=1_000_000, dim=768, nq=256, k=32, seed=1002, qseed=2002),
          "cfg4_per_gpu": dict(rows=1_250_000, dim=1024, nq=1024, k=100, seed=1004, qseed=2004)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def run_shape(name, cfg, calls, sample):
    import torch

    dev = torch.device("cuda:0")
    n, d, nq, k = cfg["rows"], cfg["dim"], cfg["nq"], cfg["k"]
    bf, i8, twin = Index(d, n + 64), Index(d, n + 64, dtype="int8"), Index(d, n + 64)
    for g, lo in enumerate(range(0, n, CHUNK)):
        m = min(CHUNK, n - lo)
        rows = torch.randn(m, d, generator=torch.Generator(device=dev).manual_seed(cfg["seed"] + g), device=dev,
                           dtype=torch.float32).to(torch.bfloat16)
        ids = np.arange(lo, lo + m, dtype=np.int64)
        bf.add_dev(rows.data_ptr(), m, ids)
        i8.add_dev(rows.data_ptr(), m, ids)
        torch.cuda.synchronize()
    q8, _ = i8.read_rows(0, n)
    for lo in range(0, n, CHUNK):
        twin.add(Qz.int8_to_bf16_bits(q8[lo:lo + CHUNK]), np.arange(lo, min(n, lo + CHUNK), dtype=np.int64))
    q = torch.randn(nq, d, generator=torch.Generator(device=dev).manual_seed(cfg["qseed"]), device=dev,
                    dtype=torch.float32).to(torch.bfloat16)
    qbits = q.cpu().view(torch.int16).numpy().view(np.uint16)
    ds, di = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8)

    def call(ix):
        t0 = time.perf_counter()
        ix.search_dev(q.data_ptr(), nq, k, ds.ptr, di.ptr)
        ix.sync()
        return (time.perf_counter() - t0) * 1e3, ix.stats()

    for ix in (bf, i8):
        for _ in range(3):
            call(ix)
    res = {"bf16": ([], []), "int8": ([], [])}
    kern = {}
    for _ in range(calls):                                 # alternate the two formats
        for key, ix in (("bf16", bf), ("int8", i8)):
            wall, st = call(ix)
            res[key][0].append(st["last_kernel_ms"])
            res[key][1].append(wall)
            kern[key] = N.KERNEL_NAMES.get(st["last_kernel"])
    out = {"shape": name, "rows": n, "dim": d, "nq": nq, "k": k, "calls": calls}
    for key, elt, mmas, peak in (("bf16", 2, 1, BF16_OPS), ("int8", 1, 2, S8_OPS)):
        kms, wms = float(np.median(res[key][0])), float(np.median(res[key][1]))
        scan = n * d * elt
        ops = 2.0 * nq * n * d * mmas          # the int8 kernel runs two s8 MMAs (hi and lo query halves) per product
        # last_kernel_ms covers the first block of queries (up to 512 on the cluster kernel): shares of a larger batch are
        # taken over the step time
        t_ms, basis = (kms, "kernel") if nq <= 512 else (wms, "step")
        out[key] = {"kernel": kern[key], "kernel_ms": round(kms, 4), "step_ms": round(wms, 4),
                    "qps": round(nq / (wms * 1e-3), 1), "scan_bytes": scan,
                    "share_basis": basis,
                    "hbm_share": round(scan * (1 if nq <= 512 else -(-nq // 512)) / (t_ms * 1e-3) / HBM_BPS, 4),
                    "mma_ops": ops, "tensor_share": round(ops / (t_ms * 1e-3) / peak, 4),
                    "shard_row_bytes": scan}
    a_ids, a_sc = i8.search(qbits, k)
    t_ids, t_sc = twin.search(qbits, k)
    b_ids, _ = bf.search(qbits, k)
    twin_ok = bool(np.array_equal(a_ids, t_ids) and np.array_equal(a_sc.view(np.int32), t_sc.view(np.int32)))
    rng = np.random.default_rng(5)
    sel = np.sort(rng.choice(nq, sample, replace=False))
    Qf = Qz.bf16_bits_to_f64(qbits[sel]).astype(np.float32)
    want, _ = O.cosine_topk(Qf, q8.astype(np.float32), k)
    oracle_ok = bool(np.array_equal(a_ids[sel], want))
    recall = float(np.mean([len(np.intersect1d(a_ids[i], b_ids[i])) / k for i in range(nq)]))
    out["parity"] = {"ids_scores_exact_vs_bf16_twin": twin_ok, "ids_exact_vs_oracle_sample": oracle_ok,
                     "oracle_sample": int(sample)}
    out["recall_at_k_vs_bf16"] = round(recall, 4)
    for ix in (bf, i8, twin):
        ix.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--sample", type=int, default=4, help="queries checked against the CPU oracle per shape")
    ap.add_argument("--cfg4", action="store_true", help="also cfg4's per-GPU shape (dim 1024, 1024 queries, top-100)")
    args = ap.parse_args()
    if N.load().aur_device_count() == 0:
        raise SystemExit("int8_bench needs a CUDA device (aurora_b200 has no CPU path)")
    name, power = card()
    out = {"tool": "int8_bench", "card": name, "power_limit": power,
           "shapes": [run_shape(s, SHAPES[s], args.calls, args.sample) for s in (["cfg2", "cfg4_per_gpu"] if args.cfg4 else ["cfg2"])]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Timing decomposition of simtopk_tc_kernel with the bring-up switches (dbg_flags, internal.h): same box,
same corpus, one process -- what each part of the pipeline costs when the others are switched off.

  python tools/decompose.py [n_rows] [out.json] [--flags 0,1,3] [--configs tile:stages:qregs,...]

--flags keeps only those dbg_flags values; --configs repeats the table under several kernel configurations
(aur_set_option tc_tile : tc_stages : tc_qregs, default 0:0:-1 = what a search picks by itself), e.g. 128:2:0,128:3:0 for
the slope of kernel time against ring depth.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits  # noqa: E402

VARIANTS = [
    (0, "full kernel"),
    (16, "no per-tile threshold read"),
    (32, "no inverse-norm prefetch"),
    (48, "neither"),
    (8, "scale + maxima, no threshold test / park / publish"),
    (8 | 16 | 32, "scale + maxima only, no global loads"),
    (4, "accumulator read, not examined"),
    (1, "accumulator neither read nor examined (TMA + MMA)"),
    (2, "no MMAs (TMA + epilogue)"),
    (1 | 2, "TMA only"),
    (0, "full kernel (again)"),
]


def sm_clock():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        return pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM), pynvml.nvmlDeviceGetPowerUsage(h) / 1000.0
    except Exception:
        return None, None


def _opt(args, name, default):
    if name not in args:
        return default
    i = args.index(name)
    v = args[i + 1]
    del args[i:i + 2]
    return v


def main():
    keep = [int(f) for f in _opt(sys.argv, "--flags", "").split(",") if f]
    configs = [tuple(int(x) for x in c.split(":")) for c in _opt(sys.argv, "--configs", "0:0:-1").split(",")]
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    out = sys.argv[2] if len(sys.argv) > 2 else "gpurun_out/decompose.json"
    variants = [v for v in VARIANTS if not keep or v[0] in keep]
    d, nq, k = 768, 256, 32
    rng = np.random.default_rng(1002)
    block = to_bf16_bits(rng.standard_normal((50_000, d)).astype(np.float32))
    q = to_bf16_bits(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
    res = []
    with Index(d, n) as ix:
        for lo in range(0, n, 50_000):
            m = min(50_000, n - lo)
            ix.add(np.roll(block[:m], lo // 50_000, axis=1), np.arange(lo, lo + m, dtype=np.int64))
        dq = DeviceBuffer(q.nbytes).upload(q)
        ds = DeviceBuffer(nq * k * 4)
        di = DeviceBuffer(nq * k * 8)
        for (tile, stages, qregs), (flags, name) in ((c, v) for c in configs for v in variants):
            for key, val in ((b"tc_tile", tile), (b"tc_stages", stages), (b"tc_qregs", qregs), (b"dbg_flags", flags)):
                N.check(ix._lib.aur_set_option(ix._h, key, val))
            for _ in range(150):                       # back to back: the clock settles where the power cap puts it
                ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr)
            clk, pw = sm_clock()
            ix.sync()
            ks = []
            for _ in range(30):
                ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr)
                ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr)
                ix.sync()
                ks.append(ix.stats()["last_kernel_ms"])
            r = {"tc_tile": tile, "tc_stages": stages, "tc_qregs": qregs, "tile_n": ix.stats()["last_tile_n"], "flags": flags, "what": name, "kernel_ms": float(np.median(ks)), "kernel_ms_min": float(np.min(ks)),
                 "sm_mhz_under_load": clk, "power_w": pw}
            res.append(r)
            print(f"tile {tile:3d} stages {stages:2d} qregs {qregs:2d}  flags {flags:3d}  {r['kernel_ms']:.4f} ms (min {r['kernel_ms_min']:.4f})  sm {clk} MHz  {pw} W   {name}", flush=True)
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    json.dump({"rows": n, "dim": d, "nq": nq, "k": k, "variants": res}, open(out, "w"), indent=1)


if __name__ == "__main__":
    main()

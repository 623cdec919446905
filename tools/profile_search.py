#!/usr/bin/env python
"""Tiny driver for ncu: build the cfg2 corpus (1M x 768 bf16) and run a few searches.

  [AUR_DIM=1024] python tools/profile_search.py [tc2|tc1|simt|auto] [n_rows] [nq] [k] [reps]
numpy + ctypes only.
"""

from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits  # noqa: E402


def main():
    kern = {"tc2": N.KERNEL_TC2, "tc1": N.KERNEL_TC1, "simt": N.KERNEL_SIMT, "auto": N.KERNEL_AUTO}[
        sys.argv[1] if len(sys.argv) > 1 else "tc2"]
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
    nq = int(sys.argv[3]) if len(sys.argv) > 3 else 256
    k = int(sys.argv[4]) if len(sys.argv) > 4 else 32
    reps = int(sys.argv[5]) if len(sys.argv) > 5 else 5
    d = int(os.environ.get("AUR_DIM", "768"))
    rng = np.random.default_rng(1002)
    block = to_bf16_bits(rng.standard_normal((min(n, 50_000), d)).astype(np.float32))
    q = to_bf16_bits(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
    with Index(d, n) as ix:
        for lo in range(0, n, block.shape[0]):
            m = min(block.shape[0], n - lo)
            # rotate the block so rows differ across chunks without regenerating randn
            ix.add(np.roll(block[:m], lo // block.shape[0], axis=1), np.arange(lo, lo + m, dtype=np.int64))
        ix.set_kernel(kern)
        flags = int(os.environ.get("AUR_DBG_FLAGS", "0"))
        if flags:
            N.check(ix._lib.aur_set_option(ix._h, b"dbg_flags", flags))
        dq = DeviceBuffer(q.nbytes).upload(q)
        ds = DeviceBuffer(nq * k * 4)
        di = DeviceBuffer(nq * k * 8)
        for _ in range(reps):
            ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr)
            ix.sync()
            st = ix.stats()
            print(f"kernel {st['last_kernel_ms']:.3f} ms  total {st['last_total_ms']:.3f} ms  launches {st['last_launches']}")


if __name__ == "__main__":
    main()

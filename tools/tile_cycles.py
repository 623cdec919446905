#!/usr/bin/env python
"""Per-tile cycles of simtopk_tc_kernel from its bring-up counters (a library built with AUR_TC_PROFILE=1, dbg_flags 64):
the MMA warpgroup's cycles over its tile count, and how much of them it spent waiting for TMA (tm_full) and for the
epilogue (tm_empty); the producer's wait for free ring stages (tp_wait); the SM clock from the globaltimer.  1M x 768
corpus, 128 queries on CTA pairs (the bring-up entry point's largest batch).

  AURORA_B200_LIB=lib_prof.so python tools/tile_cycles.py [tc_tile: 0 | 64 | 128] [n_rows] [tc_stages] [tc_qregs]
prints one JSON line.  tc_stages (0 = the deepest ring that fits) and tc_qregs (-1 = auto, 0 = the whole query block in
shared memory) are set only when given, so a library without those options can be measured too."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits  # noqa: E402

Q = N.TC_QUERY_ROWS
MAX_CTAS = 1024


def main():
    tile = int(sys.argv[1]) if len(sys.argv) > 1 else 0
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
    d, nq = 768, 2 * Q
    rng = np.random.default_rng(1002)
    block = to_bf16_bits(rng.standard_normal((50_000, d)).astype(np.float32))
    q = to_bf16_bits(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
    with Index(d, n) as ix:
        for lo in range(0, n, 50_000):
            m = min(50_000, n - lo)
            ix.add(np.roll(block[:m], lo // 50_000, axis=1), np.arange(lo, lo + m, dtype=np.int64))
        N.check(ix._lib.aur_set_option(ix._h, b"dbg_flags", 64))
        if tile:
            N.check(ix._lib.aur_set_option(ix._h, b"tc_tile", tile))
        for key, arg in ((b"tc_stages", 3), (b"tc_qregs", 4)):
            if len(sys.argv) > arg:
                N.check(ix._lib.aur_set_option(ix._h, key, int(sys.argv[arg])))
        dq = DeviceBuffer(q.nbytes).upload(q)
        dout = DeviceBuffer(MAX_CTAS * Q * 64 * 4)
        for _ in range(20):
            n_ctas = ix.debug_tc_scores(dq.ptr, nq, 2, dout.ptr)
        ix.sync()
        tile_n = tile or 64    # the bring-up entry point's default width
        out = dout.download(np.empty((MAX_CTAS, Q, 64), dtype=np.float32))[:n_ctas]
    tiles = -(-(-(-n // tile_n)) // (n_ctas // 2))        # tiles per CTA pair (one tile set per pair)
    mm, pp = out[:, 0, 32:35].astype(np.float64), out[:, 0, 36:39].astype(np.float64)
    total, full, empty = mm[:, 2].mean(), mm[:, 1].mean(), mm[:, 0].mean()
    mhz = pp[:, 1].mean() / max(pp[:, 2].mean(), 1) * 1e3
    r = {"tile_n": tile_n, "tc_stages": int(sys.argv[3]) if len(sys.argv) > 3 else 0,
         "tc_qregs": int(sys.argv[4]) if len(sys.argv) > 4 else -1, "tiles_per_cta": tiles, "mma_cycles": total, "cycles_per_tile": total / tiles,
         "cycles_per_64_rows": total / tiles * 64 / tile_n, "tm_full_share": full / total, "tm_empty_share": empty / total,
         "tp_wait_share": pp[:, 0].mean() / max(pp[:, 1].mean(), 1), "sm_mhz": mhz,
         "us_per_64_rows": total / tiles * 64 / tile_n / mhz}
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))


if __name__ == "__main__":
    main()

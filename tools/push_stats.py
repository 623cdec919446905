#!/usr/bin/env python
"""Bring-up: how many candidates each epilogue thread pushed (dbg_flags 64)."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits
Q = N.TC_QUERY_ROWS                  # queries per CTA = epilogue threads
MAX_CTAS = 1024                      # buffer sized for more CTAs than any GPU has SMs; the call returns the real count
n, d, nq = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000, 768, 2 * Q   # one query block per CTA of a pair
rng = np.random.default_rng(1002)
block = to_bf16_bits(rng.standard_normal((50_000, d)).astype(np.float32))
q = to_bf16_bits(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
with Index(d, n) as ix:
    for lo in range(0, n, 50_000):
        m = min(50_000, n - lo)
        ix.add(np.roll(block[:m], lo // 50_000, axis=1), np.arange(lo, lo + m, dtype=np.int64))
    N.check(ix._lib.aur_set_option(ix._h, b"dbg_flags", 64 | int(os.environ.get("AUR_DBG_FLAGS", "0"))))
    dq = DeviceBuffer(q.nbytes).upload(q)
    dout = DeviceBuffer(MAX_CTAS * Q * 64 * 4)
    for _ in range(3):
        n_ctas = ix.debug_tc_scores(dq.ptr, nq, 2, dout.ptr)
    out = dout.download(np.empty((MAX_CTAS, Q, 64), dtype=np.float32))[:n_ctas]
tiles = -(-(-(-n // 64)) // (n_ctas // 2))       # corpus tiles per CTA pair (one tile set per pair)
npush, nslow, tg, tl = (out[:, :, i] for i in range(4))
print(f"final list entries/thread mean {npush.mean():.1f} max {npush.max():.0f} p50 {np.median(npush):.0f}; "
      f"slow-chunk entries/thread mean {nslow.mean():.1f} max {nslow.max():.0f} (of {4 * tiles} chunks); "
      f"tau_glob mean {tg.mean():.3f} tau_local mean {tl.mean():.3f}")

tw, ts, tx, tl, tt = (out[:, :, 8 + i] for i in range(5))
print(f"cycles/thread: total {tt.mean():.0f} wait_full {tw.mean():.0f} ({100*tw.mean()/tt.mean():.0f}%) "
      f"slow {ts.mean():.0f} ({100*ts.mean()/tt.mean():.0f}%) xchg {tx.mean():.0f} ({100*tx.mean()/tt.mean():.0f}%) "
      f"ld_scores {tl.mean():.0f} ({100*tl.mean()/tt.mean():.0f}%)  slow max {ts.max():.0f}")
mm = out[:, 0, 32:35]
print(f"MMA warpgroup cycles: total {mm[:,2].mean():.0f} wait_score_buffer {mm[:,0].mean():.0f} ({100*mm[:,0].mean()/mm[:,2].mean():.0f}%) "
      f"wait_smem_full {mm[:,1].mean():.0f} ({100*mm[:,1].mean()/mm[:,2].mean():.0f}%)")
pp = out[:, 0, 36:39]
print(f"TMA producer cycles: total {pp[:,1].mean():.0f} wait_smem_empty {pp[:,0].mean():.0f} ({100*pp[:,0].mean()/max(pp[:,1].mean(),1):.0f}%); "
      f"streaming phase {pp[:,2].mean()/1e3:.1f} us -> SM clock {pp[:,1].mean()/max(pp[:,2].mean(),1)*1e3:.0f} MHz")
ts = out[:, :, 9]; ns = out[:, :, 1]
flat = np.argsort(-ts.ravel())[:12]
for f in flat:
    cta, r = divmod(int(f), Q)
    print(f"  cta {cta} r {r} warp {r//32}: t_slow {ts[cta, r]:.0f} nslow {ns[cta, r]:.0f} tau_end {out[cta, r, 2]:.3f} nfill {out[cta, r, 0]:.0f} total {out[cta, r, 12]:.0f} wait {out[cta, r, 8]:.0f}")
w = ts.reshape(n_ctas, Q // 32, 32).max(axis=2)
print("per-warp slow cycles: mean %.0f p50 %.0f p90 %.0f p99 %.0f max %.0f" % (w.mean(), np.median(w), np.percentile(w, 90), np.percentile(w, 99), w.max()))
print("nslow per thread: p50 %.0f p90 %.0f p99 %.0f max %.0f" % (np.median(ns), np.percentile(ns, 90), np.percentile(ns, 99), ns.max()))

tt = out[:, :, 12].mean()
for name, idx in (("chunks it<8", 13), ("wait_full", 8), ("ld_scores", 11), ("fast", 14), ("chunks it>=8", 15), ("publish", 16)):
    print(f"  {name:18s} {out[:, :, idx].mean():10.0f} cycles ({100 * out[:, :, idx].mean() / tt:4.1f}%)  per tile {out[:, :, idx].mean() / tiles:.0f}")

print(f"  q-load {out[:, :, 18].mean():.0f} cycles; bootstrap (incl. first MMA tile) {out[:, :, 17].mean():.0f} (max {out[:, :, 17].max():.0f}); tail {out[:, :, 19].mean():.0f}")

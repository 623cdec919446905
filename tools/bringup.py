#!/usr/bin/env python
"""GPU bring-up ladder.  Each stage runs in its own process under a timeout so a hung
kernel (mbarrier protocol bug) costs seconds, not the box.

  python tools/bringup.py            # run every stage, print a PASS/FAIL table
  python tools/bringup.py --stage <name>   # run one stage in-process

Only numpy + ctypes (no torch import): start-up is fast on a fresh box.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from aurora_b200 import _native as N  # noqa: E402
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits  # noqa: E402

from oracle import cosine_topk as O  # noqa: E402
from tests import bounds as BD  # noqa: E402

QROWS = N.TC_QUERY_ROWS
MAX_CTAS = 1024      # debug-score buffers are sized for more CTAs than any GPU has SMs; the call returns the real count


def _data(n, d, nq, seed=0, planted=True):
    rng = np.random.default_rng(seed)
    Cm = O.round_to_bf16(rng.standard_normal((n, d)).astype(np.float32))
    Qm = O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))
    if planted and n >= 8 * nq:
        for i in range(nq):
            rows = rng.choice(n, size=4, replace=False)
            Cm[rows] = O.round_to_bf16((Qm[i][None, :] + 0.3 * rng.standard_normal((4, d))).astype(np.float32))
    return Cm, Qm


def _compare(ids, sc, oids, osc, tag):
    ok_ids = np.array_equal(ids, oids)
    finite = np.isfinite(osc)
    dmax = float(np.max(np.abs(sc[finite] - osc[finite]))) if finite.any() else 0.0
    nbad = int((ids != oids).sum())
    print(f"[{tag}] ids_equal={ok_ids} mismatches={nbad}/{ids.size} max|dscore|={dmax:.3e}")
    if not ok_ids:
        bad = np.argwhere(ids != oids)[:5]
        for q, j in bad:
            print(f"   q={q} rank={j}: got id {ids[q, j]} ({sc[q, j]:.6f}) want {oids[q, j]} ({osc[q, j]:.6f})")
    return ok_ids and dmax <= 1e-3


def stage_simt_small():
    ok = True
    for (n, d, nq, k, dtype) in [(1000, 384, 1, 5, "f32"), (5000, 768, 33, 32, "bf16"), (700, 100, 7, 10, "f32"),
                                  (3, 64, 2, 5, "bf16")]:
        Cm, Qm = _data(n, d, nq, seed=n)
        if dtype == "f32":
            rng = np.random.default_rng(n + 1)
            Cm = rng.standard_normal((n, d)).astype(np.float32)
            Qm = rng.standard_normal((nq, d)).astype(np.float32)
        with Index(d, max(n, 64), dtype=dtype) as ix:
            ix.set_kernel(N.KERNEL_SIMT)
            ix.add(Cm, np.arange(n, dtype=np.int64) * 3 + 7)
            ids, sc = ix.search(Qm, k)
        oids, osc = O.cosine_topk(Qm, Cm, k, ids=np.arange(n, dtype=np.int64) * 3 + 7)
        ok &= _compare(ids, sc, oids, osc, f"simt n={n} d={d} nq={nq} k={k} {dtype}")
    return ok


def stage_simt_filter_delete():
    n, d, nq, k = 4000, 128, 9, 8
    Cm, Qm = _data(n, d, nq, seed=5)
    rng = np.random.default_rng(9)
    ru = rng.integers(0, 5, n).astype(np.int32)
    ro = rng.integers(-1, 3, n).astype(np.int32)
    qu = rng.integers(0, 5, nq).astype(np.int32)
    qo = rng.integers(-1, 3, nq).astype(np.int32)
    ids0 = np.arange(n, dtype=np.int64)
    live = np.ones(n, dtype=bool)
    with Index(d, n + 100) as ix:
        ix.set_kernel(N.KERNEL_SIMT)
        ix.add(Cm, ids0, ru, ro)
        dead = rng.choice(n, size=500, replace=False)
        assert ix.remove(dead) == 500
        live[dead] = False
        ids, sc = ix.search(Qm, k, qu, qo)
        st = ix.stats()
    oids, osc = O.cosine_topk(Qm, Cm, k, ids=ids0, live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo)
    ok = _compare(ids, sc, oids, osc, "simt filter+delete")
    print("   stats", st)
    return ok and st["live"] == n - 500


def _tc_scores(cta_group):
    # the debug entry takes one query block per CTA of a pair: 2 x QROWS queries; every CTA returns the first tile
    # of its tile set, [QROWS queries x 64 rows]
    n, d, nq = 200 * 64 + 37, 768, 2 * QROWS
    Cm, Qm = _data(n, d, nq, seed=11, planted=False)
    with Index(d, n) as ix:
        ix.add(Cm, np.arange(n, dtype=np.int64))
        dq = DeviceBuffer(nq * d * 2).upload(to_bf16_bits(Qm))
        cap = MAX_CTAS * QROWS * 64
        dout = DeviceBuffer(cap * 4).upload(np.full(cap, -7.0, dtype=np.float32))
        got_ctas = ix.debug_tc_scores(dq.ptr, nq, cta_group, dout.ptr)
        out = dout.download(np.empty((MAX_CTAS, QROWS, 64), dtype=np.float32))[:got_ctas]
    print(f"   kernel returned, n_ctas={got_ctas}")
    S, bound = BD.sim_reference(Qm, Cm)
    worst = 0.0
    nbad = 0
    for cta in range(got_ctas):
        qblock, lst = BD.tc_debug_tile(cta, nq)
        row0 = lst * 64
        rows = np.arange(row0, row0 + 64)
        valid = rows < n
        want = S[qblock * QROWS:(qblock + 1) * QROWS][:, rows[valid]]
        got = out[cta][:, valid]
        e = BD.ratio(got, want, bound[qblock * QROWS:(qblock + 1) * QROWS][:, rows[valid]])
        if e > 1.0:
            nbad += 1
            if nbad <= 4:
                print(f"   cta {cta} (qblock {qblock}, tile {lst}) max err/bound {e:.3f}; got[0,:4]={got[0, :4]} want[0,:4]={want[0, :4]}")
        worst = max(worst, e)
    print(f"[tc scores cta_group={cta_group}] bad_ctas={nbad}/{got_ctas} max(err / bound)={worst:.3f}")
    return nbad == 0


def stage_tc1_scores():
    return _tc_scores(1)


def stage_tc2_scores():
    return _tc_scores(2)


def _tc_search(kernel, n, nq, k, d=768):
    Cm, Qm = _data(n, d, nq, seed=n % 1000 + nq)
    ids0 = np.arange(n, dtype=np.int64)
    with Index(d, n) as ix:
        ix.add(Cm, ids0)
        ix.set_kernel(kernel)
        t0 = time.time()
        ids, sc = ix.search(Qm, k)
        t1 = time.time()
        st = ix.stats()
    oids, osc = O.cosine_topk(Qm, Cm, k)
    ok = _compare(ids, sc, oids, osc, f"{N.KERNEL_NAMES[kernel]} n={n} nq={nq} k={k} d={d}")
    print(f"   host wall {1e3 * (t1 - t0):.2f} ms, kernel {st['last_kernel_ms']:.3f} ms, total dev {st['last_total_ms']:.3f} ms, launches {st['last_launches']}")
    return ok


def stage_tc1_search():
    return _tc_search(N.KERNEL_TC1, 30000, 256, 32) and _tc_search(N.KERNEL_TC1, 9000, 100, 10, d=384)


def stage_tc2_search():
    return _tc_search(N.KERNEL_TC2, 30000, 256, 32) and _tc_search(N.KERNEL_TC2, 50001, 200, 100, d=512)


def stage_tc_big():
    """1M x 768: tensor-core paths against each other and the SIMT path (no CPU oracle at this size)."""
    n, d, nq, k = 1_000_000, 768, 256, 32
    rng = np.random.default_rng(1002)
    bits = np.empty((n, d), dtype=np.uint16)
    for lo in range(0, n, 100_000):
        bits[lo:lo + 100_000] = to_bf16_bits(rng.standard_normal((100_000, d)).astype(np.float32))
    Qm = O.round_to_bf16(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
    res = {}
    with Index(d, n) as ix:
        for lo in range(0, n, 250_000):
            ix.add(bits[lo:lo + 250_000], np.arange(lo, lo + 250_000, dtype=np.int64))
        for kern in (N.KERNEL_TC2, N.KERNEL_TC1, N.KERNEL_SIMT):
            ix.set_kernel(kern)
            for rep in range(3):
                ids, sc = ix.search(Qm, k)
            st = ix.stats()
            res[kern] = (ids, sc)
            print(f"[big {N.KERNEL_NAMES[kern]}] kernel {st['last_kernel_ms']:.3f} ms total {st['last_total_ms']:.3f} ms "
                  f"launches {st['last_launches']} -> {1.5365e9 / (st['last_kernel_ms'] * 1e-3) / 1e9:.0f} GB/s algorithmic")
    ok = True
    for kern in (N.KERNEL_TC2, N.KERNEL_TC1):
        same = np.array_equal(res[kern][0], res[N.KERNEL_SIMT][0])
        dm = float(np.max(np.abs(res[kern][1] - res[N.KERNEL_SIMT][1])))
        print(f"[big] {N.KERNEL_NAMES[kern]} vs simt: ids_equal={same} max|ds|={dm:.2e}")
        ok &= same and dm < 1e-6
    # oracle on a subsample of queries
    sub = [0, 17, 255]
    Cf = O.bf16_bits_to_f32(bits)
    oids, osc = O.cosine_topk(Qm[sub], Cf, k)
    ok &= _compare(res[N.KERNEL_TC2][0][sub], res[N.KERNEL_TC2][1][sub], oids, osc, "big tc2 vs oracle (3 queries)")
    return ok


STAGES = {
    "simt_small": (stage_simt_small, 180),
    "simt_filter_delete": (stage_simt_filter_delete, 120),
    "tc1_scores": (stage_tc1_scores, 120),
    "tc2_scores": (stage_tc2_scores, 120),
    "tc1_search": (stage_tc1_search, 180),
    "tc2_search": (stage_tc2_search, 180),
    "tc_big": (stage_tc_big, 600),
}


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--stage":
        ok = STAGES[sys.argv[2]][0]()
        print("STAGE", sys.argv[2], "PASS" if ok else "FAIL")
        sys.exit(0 if ok else 1)
    wanted = sys.argv[1:] or list(STAGES)
    results = {}
    for name in wanted:
        fn, tmo = STAGES[name]
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--stage", name], timeout=tmo, capture_output=True, text=True)
            out = p.stdout + p.stderr
            results[name] = "PASS" if p.returncode == 0 else f"FAIL(rc={p.returncode})"
        except subprocess.TimeoutExpired as e:
            out = ((e.stdout or b"").decode() if isinstance(e.stdout, bytes) else (e.stdout or "")) + "\n<<TIMEOUT>>"
            results[name] = "TIMEOUT"
        print(f"===== {name}: {results[name]} ({time.time() - t0:.1f}s)")
        print(out[-6000:])
        sys.stdout.flush()
    print("===== SUMMARY")
    for k, v in results.items():
        print(f"  {k:22s} {v}")


if __name__ == "__main__":
    main()

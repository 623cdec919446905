"""Kernel outputs held to what they must be exactly or within a per-element bound (tests/bounds.py): the similarity
kernel's raw score tiles against fp64, and the order of tied rows -- bit-identical chunks are common in a knowledge
base (boilerplate paragraphs) -- through the tensor-core, generic and sharded paths.  Run on an H100 with -m gpu."""

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index, MultiIndex, to_bf16_bits
from oracle import cosine_topk as O
from tests import bounds as BD

pytestmark = pytest.mark.gpu
QROWS = N.TC_QUERY_ROWS
SENTINEL = -7.0


def _bf16(x):
    return O.round_to_bf16(np.asarray(x, dtype=np.float32))


# ------------------------------------------------------------------------------ raw similarity score tiles
@pytest.mark.parametrize("nq", [1, 64, 65, 128])
@pytest.mark.parametrize("d", [64, 128, 192, 576, 768, 1024])
@pytest.mark.parametrize("cta_group", [1, 2])
def test_tc_raw_scores_against_fp64(cta_group, d, nq):
    """Every CTA returns the first [64 x 64] tile of its tile set.  41 tiles (the last one partial) for more tile sets
    than that: some CTAs own no tile and must leave the buffer alone."""
    rng = np.random.default_rng(d + nq + cta_group)
    n = 40 * 64 + 37
    C = _bf16(rng.standard_normal((n, d)))
    Q = _bf16(rng.standard_normal((nq, d)))
    C[[7, 64 * 5 + 3, n - 1]] = 0.0                                   # zero rows: score exactly 0
    copies = [3, 10, 64 * 2 + 9, 64 * 33 + 63, n - 2]                 # one row within a tile, across tiles and CTAs
    C[copies] = C[3]
    dead = np.array([11, 64 * 7], dtype=np.int64)
    n_tiles = (n + 63) // 64
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.remove(dead)
        ix.set_kernel(N.KERNEL_TC1 if cta_group == 1 else N.KERNEL_TC2)
        before = ix.search(Q, 10)
        dq = DeviceBuffer(Q.size * 2).upload(to_bf16_bits(Q))
        cap = 1024 * QROWS * 64
        dout = DeviceBuffer(cap * 4).upload(np.full(cap, SENTINEL, dtype=np.float32))
        n_ctas = ix.debug_tc_scores(dq.ptr, nq, cta_group, dout.ptr)
        out = dout.download(np.empty((1024, QROWS, 64), dtype=np.float32))[:n_ctas]
        after = ix.search(Q, 10)                                    # the debug call leaves no candidates behind
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])

    ref, bound = BD.sim_reference(Q, C)
    got = np.full((nq, n), np.nan)
    seen = np.zeros(n_tiles, dtype=bool)
    for cta in range(n_ctas):
        qb, tile = BD.tc_debug_tile(cta, nq)
        if tile >= n_tiles:
            assert (out[cta] == SENTINEL).all(), f"CTA {cta} owns no tile but wrote its buffer"
            continue
        q0, q1 = qb * QROWS, min(nq, (qb + 1) * QROWS)
        if q1 <= q0:
            continue
        seen[tile] = True
        rows = tile * 64 + np.arange(64)
        past = rows >= n
        assert np.isnan(out[cta][:q1 - q0, past]).all(), "rows past n must be NaN"
        got[q0:q1, rows[~past]] = out[cta][:q1 - q0, ~past]
    assert seen.all()
    assert np.isnan(got[:, dead]).all(), "tombstones must be NaN"
    live = np.ones(n, dtype=bool); live[dead] = False
    assert (got[:, [7, 64 * 5 + 3, n - 1]] == 0.0).all()
    for c in copies[1:]:
        assert np.array_equal(got[:, c], got[:, copies[0]]), f"row copy at {c} scores differently"
    BD.assert_within(f"tc scores cta_group={cta_group} d={d} nq={nq}", got[:, live], ref[:, live], bound[:, live])


# ------------------------------------------------------------------------------------------- ties
KERNELS = [N.KERNEL_TC1, N.KERNEL_TC2, N.KERNEL_SIMT]


def _tie_data(n=3000, d=128, seed=0):
    """60 bit-identical rows (500..559) that are every query's best match, among random rows."""
    rng = np.random.default_rng(seed)
    C = _bf16(rng.standard_normal((n, d)))
    Q = _bf16(rng.standard_normal((3, d)))
    C[500:560] = _bf16(Q[0] * 0.5 + Q[1] * 0.25 + Q[2] * 0.25)
    return C, Q, rng


def _check_exact(got, C, Q, k, ids, live=None):
    want_ids, want_sc = O.cosine_topk(Q, C, k, ids=ids, live=live)
    assert np.array_equal(got[0], want_ids), f"got {got[0][:, :12].tolist()} want {want_ids[:, :12].tolist()}"
    assert np.abs(got[1] - want_sc).max() <= 1e-6


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("case", ["ids_in_row_order", "shuffled_ids", "low_id_upserted_after_group"])
def test_tied_rows_keep_the_lowest_ids(kernel, case):
    """A group of tied rows larger than k + slack is cut by every selection stage; the survivors must be the lowest
    ids, in id order, whatever rows they sit in."""
    n, d, k = 3000, 128, 10
    C, Q, rng = _tie_data(n, d)
    ids = np.arange(n, dtype=np.int64) if case == "ids_in_row_order" else rng.permutation(10 * n)[:n].astype(np.int64) + 10
    live = None
    if case == "low_id_upserted_after_group":
        ids[10] = 3                                  # an unrelated row holds the lowest id ...
    with Index(d, n + 64) as ix:
        ix.add(C, ids)
        ix.set_kernel(kernel)
        if case == "low_id_upserted_after_group":   # ... and is upserted with the tied vector: its old row becomes a
            ix.add(C[500:501], np.array([3], dtype=np.int64))   # tombstone, the new row lands behind the group
            C, ids = np.concatenate([C, C[500:501]]), np.concatenate([ids, [3]])
            live = np.ones(n + 1, dtype=bool)
            live[10] = False
        got = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == kernel
    _check_exact(got, C, Q, k, ids, live)
    if case == "low_id_upserted_after_group":
        assert got[0][0, 0] == 3                     # query 0's best match is the tied vector


@pytest.mark.parametrize("kernel", KERNELS)
def test_tied_rows_with_k128_over_many_lists(kernel):
    """k = 128 over 70 000 rows: the generic kernel's 35 segment lists of k + slack keys exceed one 4096-key sort, so
    they are folded by the list reduction before the final sort; a tied group of 200 rows crosses every cut."""
    n, d, k = 70000, 64, 128
    rng = np.random.default_rng(11)
    C = _bf16(rng.standard_normal((n, d)))
    Q = _bf16(rng.standard_normal((2, d)))
    C[rng.choice(n, size=200, replace=False)] = _bf16(Q[0] * 0.5 + Q[1] * 0.5)
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    with Index(d, n) as ix:
        ix.add(C, ids)
        ix.set_kernel(kernel)
        got = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == kernel
        if kernel == N.KERNEL_SIMT:
            assert ix.stats()["last_launches"] == 8         # 3 x (scores + select) per 32 768 rows, one reduction, the final sort
    _check_exact(got, C, Q, k, ids)


@pytest.mark.parametrize("kernel", KERNELS)
def test_tied_rows_across_three_shards(kernel):
    n, d, k = 3000, 128, 10
    C, Q, rng = _tie_data(n, d, seed=1)
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    with MultiIndex(d, n, devices=[0, 0, 0]) as mi:
        for s in mi.shards:
            s.set_kernel(kernel)
        mi.add(C, ids)
        assert len({int(i) % 3 for i in ids[500:560]}) == 3
        got = mi.search(Q, k)
    _check_exact(got, C, Q, k, ids)


@pytest.mark.parametrize("kernel", KERNELS)
def test_near_tie_group_straddling_k_comes_out_in_exact_order(kernel):
    """Six rows one bf16 ulp apart from a base row, each in a component where the query is tiny, so their scores
    differ in the last bits only; the group straddles position k and is smaller than the slack, so the exact re-rank
    must order it."""
    n, d, k = 4000, 128, 10
    rng = np.random.default_rng(5)
    C = _bf16(rng.standard_normal((n, d)))
    q = rng.standard_normal(d)
    q[:6] = 1e-4
    Q = _bf16(q[None, :])
    base = _bf16(0.5 * Q[0] + 0.3 * rng.standard_normal(d))
    rows = rng.choice(n, size=13, replace=False)
    for i, r in enumerate(rows[:7]):                                 # seven clearly better rows
        C[r] = _bf16(Q[0] + 0.05 * (i + 1) * rng.standard_normal(d))
    for i, r in enumerate(rows[7:]):                                 # the near-tie group: ranks 7 .. 12
        bits = to_bf16_bits(base[None, :])[0].copy()
        bits[i] += 1
        C[r] = O.bf16_bits_to_f32(bits)
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    with Index(d, n) as ix:
        ix.add(C, ids)
        ix.set_kernel(kernel)
        got = ix.search(Q, k)
    want = O.cosine_topk(Q, C, k, ids=ids)
    assert set(want[0][0, 7:].tolist()) <= set(ids[rows[7:]].tolist())
    _check_exact(got, C, Q, k, ids)

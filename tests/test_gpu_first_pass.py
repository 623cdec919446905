"""Every first-pass similarity score, element by element, against an fp64 reference (tests/bounds.py).

A search keeps k + 8 candidates of a first pass in fp32 and orders them by an exact fp64 re-rank.  The re-rank hides a
first pass that is wrong by much more than its rounding until near-duplicates sit at the cut, so the first pass of
every kernel is checked here on its own, through debug entry points that launch it as a search does: the tensor-core
kernel's whole first tile per CTA (64- and 128-row tiles, query k-blocks in registers or shared memory, single CTAs and
pairs, bf16 and int8 rows), the list kernel and the generic kernel as dense [nq, rows] matrices.  Each case prints
max(err / bound).  Run on an H100 with -m gpu."""

import ctypes

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits
from oracle import cosine_topk as O
from tests import bounds as BD

pytestmark = pytest.mark.gpu
QROWS = N.TC_QUERY_ROWS
SENTINEL = -7.0
MAX_CTAS = 1024


def _bf16(x):
    return O.round_to_bf16(np.asarray(x, dtype=np.float32))


def _opt(ix, key, value):
    N.check(ix._lib.aur_set_option(ix._h, key, int(value)))


# ------------------------------------------------------------------------------------------ tensor-core tiles
N_TC = 32 * 128 + 37                 # the last tile partial at either width; no more tiles than tile sets (132 SMs)
TC_ZERO = [7, 64 * 5 + 3, N_TC - 1]
TC_COPIES = [3, 10, 64 * 2 + 9, 128 * 20 + 100, 64 * 33 + 63, N_TC - 2]   # within a tile, across tiles, halves and CTAs
TC_DEAD = [11, 64 * 7, 128 * 9 + 127]


def _tc_corpus(d, seed):
    rng = np.random.default_rng(seed)
    C = _bf16(rng.standard_normal((N_TC, d)))
    C[TC_ZERO] = 0.0
    C[TC_COPIES] = C[TC_COPIES[0]]
    return C, rng


def _tc_dump(ix, dq, nq, cta_group, tile, qregs):
    """One debug launch with the index's tc_tile / tc_qregs set: (scores [n_ctas, 64, tile_n], tile_n)."""
    _opt(ix, b"tc_tile", tile)
    _opt(ix, b"tc_qregs", qregs)
    cap = MAX_CTAS * QROWS * 128
    dout = DeviceBuffer(cap * 4).upload(np.full(cap, SENTINEL, dtype=np.float32))
    n_ctas, tile_n = ix.debug_tc_tile(dq.ptr, nq, cta_group, dout.ptr, cap)
    assert tile_n == (tile or 64)
    out = dout.download(np.empty(cap, dtype=np.float32))[:n_ctas * QROWS * tile_n].reshape(n_ctas, QROWS, tile_n)
    assert (dout.download(np.empty(cap, dtype=np.float32))[n_ctas * QROWS * tile_n:] == SENTINEL).all()
    return out, tile_n


def _tc_dense(out, tile_n, nq, n):
    """The dump as [nq, n] (every row is the first tile of exactly one tile set), with its layout rules checked: CTAs
    that own no tile leave their buffer alone, rows past n are NaN."""
    got = np.full((nq, n), np.nan)
    seen = np.zeros(-(-n // tile_n), dtype=bool)
    for cta in range(out.shape[0]):
        qb, rows = BD.tc_debug_rows(cta, nq, tile_n)
        if rows[0] >= n:
            assert (out[cta] == SENTINEL).all(), f"CTA {cta} owns no tile but wrote its buffer"
            continue
        q0, q1 = qb * QROWS, min(nq, (qb + 1) * QROWS)
        if q1 <= q0:
            continue
        seen[rows[0] // tile_n] = True
        past = rows >= n
        assert np.isnan(out[cta][:q1 - q0, past]).all(), "rows past n must be NaN"
        got[q0:q1, rows[~past]] = out[cta][:q1 - q0, ~past]
    assert seen.all()
    return got


def _check_rules(got, live):
    assert np.isnan(got[:, TC_DEAD]).all(), "tombstones must be NaN"
    assert np.isfinite(got[:, live]).all()
    assert (got[:, TC_ZERO] == 0.0).all()
    for c in TC_COPIES[1:]:
        assert np.array_equal(got[:, c], got[:, TC_COPIES[0]]), f"row copy at {c} scores differently"


def _same(tag, a, b):
    same = np.array_equal(a, b, equal_nan=True)
    print(f"{tag}: {'bit-identical' if same else f'differ in {int((a != b).sum())} scores, max {np.nanmax(np.abs(a - b)):.3g}'}")
    return same


@pytest.mark.parametrize("nq", [1, 64, 65, 128])
@pytest.mark.parametrize("d", [320, 384, 448, 768, 1024])
def test_tc_bf16_first_tile_every_width_and_operand(d, nq):
    """64- and 128-row tiles, the 128-row tile with its first query k-blocks in registers (tc_qregs auto: 6 from dim 384)
    and all in shared memory, single CTAs and pairs.  Every score within BD.sim_reference; the register and
    shared-memory operands bit-identical, as the kernel documents (same operands, same order)."""
    C, rng = _tc_corpus(d, d)
    Q = _bf16(rng.standard_normal((nq, d)))
    live = np.ones(N_TC, dtype=bool)
    live[TC_DEAD] = False
    ref, bound = BD.sim_reference(Q, C)
    dumps = {}
    with Index(d, N_TC + 100) as ix:
        ix.add(C, np.arange(N_TC, dtype=np.int64))
        ix.remove(np.array(TC_DEAD, dtype=np.int64))
        dq = DeviceBuffer(Q.size * 2).upload(to_bf16_bits(Q))
        for cta_group in (1, 2):
            for tile, qregs in ((0, -1), (128, 0), (128, -1)):
                out, tile_n = _tc_dump(ix, dq, nq, cta_group, tile, qregs)
                got = _tc_dense(out, tile_n, nq, N_TC)
                _check_rules(got, live)
                tag = f"tc bf16 d={d} nq={nq} cta_group={cta_group} tile={tile_n} tc_qregs={qregs}"
                BD.assert_within(tag, got[:, live], ref[:, live], bound[:, live])
                dumps[cta_group, tile_n, qregs] = got
    for g in (1, 2):
        assert _same(f"d={d} nq={nq} cta_group={g}: 128-row tiles, query k-blocks in registers vs shared memory",
                     dumps[g, 128, -1], dumps[g, 128, 0])
        _same(f"d={d} nq={nq} cta_group={g}: 64- vs 128-row tiles", dumps[g, 64, -1], dumps[g, 128, 0])
    for t in (64, 128):
        _same(f"d={d} nq={nq} tile={t}: cta_group 1 vs 2", dumps[1, t, -1], dumps[2, t, -1])


def _int8_queries(d, rng):
    """65 queries (two query blocks): a dominant component, a zero query, negative values whose 16-bit image lies on and
    next to multiples of 256 and of 256 +- 128 (where hi = (q16 + 128) >> 8 changes), then random ones."""
    Q = rng.standard_normal((65, d))
    Q[0] = 1e-3 * Q[0]
    Q[0, 5] = 3.0
    Q[1] = 0.0
    m = rng.integers(1, 127, size=d)
    off = rng.choice([-129, -128, -127, -1, 0, 1, 127, 128, 129], size=d)
    Q[2] = -(256.0 * m + off) / 32512.0
    Q[2, 0] = -1.0                                   # amax = 1: q16 = rint(32512 q)
    Q[3] = -Q[2]
    return _bf16(Q)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("d", [384, 768, 1024])
def test_tc_int8_first_tile_exact(d, tile, cta_group):
    """The int8 first pass is integer arithmetic up to two fp32 roundings, so the dump must equal BD.int8_tc_reference
    bit for bit (0 ulps; the inverse norm is reproduced exactly).  Divided by the query image's scale it must also lie
    within amax_q / 65024 per dimension of the fp64 cosine over the stored rows (BD.int8_cosine_reference)."""
    C, rng = _tc_corpus(d, 100 + d)
    Q = _int8_queries(d, rng)
    nq = Q.shape[0]
    live = np.ones(N_TC, dtype=bool)
    live[TC_DEAD] = False
    with Index(d, N_TC + 100, dtype="int8") as ix:
        ix.add(C, np.arange(N_TC, dtype=np.int64))
        ix.remove(np.array(TC_DEAD, dtype=np.int64))
        R = ix.export()[0]
        dq = DeviceBuffer(Q.size * 2).upload(to_bf16_bits(Q))
        out, tile_n = _tc_dump(ix, dq, nq, cta_group, tile, -1)
    got = _tc_dense(out, tile_n, nq, N_TC)
    _check_rules(got, live)
    q_bits = to_bf16_bits(Q)
    want = BD.int8_tc_reference(q_bits, R)
    g32, w32 = got[:, live].astype(np.float32), want[:, live]
    ulps = np.abs(g32.view(np.int32).astype(np.int64) - w32.view(np.int32).astype(np.int64))
    print(f"tc int8 d={d} tile={tile_n} cta_group={cta_group}: max |dump - exact| = {int(ulps.max())} ulps")
    assert np.array_equal(g32, w32), f"{int((g32 != w32).sum())} scores differ from the exact int8 first pass"
    assert (got[1, live] == 0.0).all()               # the zero query
    ref, bound, scale = BD.int8_cosine_reference(q_bits, R)
    BD.assert_within(f"tc int8 d={d} tile={tile_n} cta_group={cta_group} vs fp64 cosine",
                     got[:, live] * scale[:, None], ref[:, live], bound[:, live])


# ---------------------------------------------------------------------------------------------- list kernel
LIST_LENS = [1, 63, 64, 65, 2047, 2048, 2049, 4097]   # one 64-row tile, tile edges, segment edges, three segments
LIST_QUERIES = [1, 15, 16, 17, 64, 65]                # m_tiles 1 .. 4, and two groups
N_LIST = 6000


def _list_case(d, seed):
    """Rows, dead rows, lists (drawn from one pool, so they share rows; unsorted, with a repeat) and q_list."""
    rng = np.random.default_rng(seed)
    C = _bf16(rng.standard_normal((N_LIST, d)))
    C[17] = 0.0
    dead = rng.choice(N_LIST, size=40, replace=False)
    lists = []
    for ln in LIST_LENS:
        rows = rng.choice(N_LIST, size=ln, replace=False)
        lists.append(np.concatenate([rows, rows[:1]]) if ln > 1 else rows)
    lists[3][:8] = lists[4][:8]                                        # shared rows
    counts = [LIST_QUERIES[i % len(LIST_QUERIES)] for i in range(len(lists))]
    q_list = rng.permutation(np.repeat(np.arange(len(lists)), counts)).astype(np.int32)
    return C, dead, lists, q_list, rng


def _list_expect_mask(lists, q_list, dead):
    m = np.zeros((len(q_list), N_LIST), dtype=bool)
    for q, l in enumerate(q_list):
        m[q, lists[l]] = True
    m[:, dead] = False
    return m


@pytest.mark.parametrize("d", [8, 56, 64, 72, 200, 1536])
def test_list_scores_against_fp64(d):
    """list_scores_kernel as aur_search_lists launches it: every query against every live row of its list within
    BD.sim_reference, NaN for tombstones and everywhere the list does not reach."""
    C, dead, lists, q_list, rng = _list_case(d, 300 + d)
    Q = _bf16(rng.standard_normal((len(q_list), d)))
    with Index(d, N_LIST + 64) as ix:
        ix.add(C, np.arange(N_LIST, dtype=np.int64))
        ix.remove(dead)
        got = ix.debug_list_scores(Q, lists, q_list)
    m = _list_expect_mask(lists, q_list, dead)
    assert got.shape == (len(q_list), N_LIST)
    assert np.isnan(got[~m]).all(), "a score where the query's list does not reach, or for a tombstone"
    assert np.isfinite(got[m]).all(), "a listed live row without a score"
    ref, bound = BD.sim_reference(Q, C)
    BD.assert_within(f"list scores d={d} nq={len(q_list)}", got[m], ref[m], bound[m])
    for l in range(len(lists)):
        print(f"  list {l}: {len(np.unique(lists[l]))} rows, {int((q_list == l).sum())} queries")


@pytest.mark.parametrize("d", [64, 1536])
def test_list_scores_int8_rows_bit_identical_to_bf16_twin(d):
    """int8 rows enter the ring as the bf16 values they are: the same scores, bit for bit, as a bf16 shard fed the
    stored int8 rows; and within BD.sim_reference over those rows."""
    C, dead, lists, q_list, rng = _list_case(d, 400 + d)
    Q = _bf16(rng.standard_normal((len(q_list), d)))
    with Index(d, N_LIST + 64, dtype="int8") as ix:
        ix.add(C, np.arange(N_LIST, dtype=np.int64))
        ix.remove(dead)
        R = ix.export()[0]
        got8 = ix.debug_list_scores(Q, lists, q_list)
    with Index(d, N_LIST + 64) as tw:
        tw.add(R.astype(np.float32), np.arange(N_LIST, dtype=np.int64))
        tw.remove(dead)
        got16 = tw.debug_list_scores(Q, lists, q_list)
    assert np.array_equal(got8, got16, equal_nan=True)
    m = _list_expect_mask(lists, q_list, dead)
    ref, bound = BD.sim_reference(Q, R)
    BD.assert_within(f"list scores int8 d={d}", got8[m], ref[m], bound[m])


# -------------------------------------------------------------------------------------------- generic kernel
N_SIMT = 16 * 2048 + 3 * 64 + 37       # a second chunk (row0 > 0) ending in a partial 64-row block
SIMT_NQ = [1, 63, 64, 65, 130]


@pytest.mark.parametrize("dtype,d", [("f32", 1), ("f32", 3), ("f32", 15), ("f32", 17), ("f32", 100), ("f32", 1025),
                                     ("bf16", 8), ("bf16", 24), ("bf16", 64), ("bf16", 200),
                                     ("int8", 16), ("int8", 48)])
def test_simt_scores_against_fp64(dtype, d):
    """simt_scores_kernel over n_rows below the capacity, as a search chunks it: every score within
    BD.sim_reference (bf16 and int8 rows: exact products) or BD.sim_reference_f32; -inf for tombstones and, with the
    batch's one tenant scope (nq = 65), for the rows it may not see."""
    rng = np.random.default_rng(500 + d)
    C = rng.standard_normal((N_SIMT, d)).astype(np.float32)
    Q = rng.standard_normal((max(SIMT_NQ), d)).astype(np.float32)
    if dtype != "f32":
        C, Q = _bf16(C), _bf16(Q)
    C[[5, N_SIMT - 1]] = 0.0
    user = rng.integers(0, 3, size=N_SIMT).astype(np.int32)
    dead = rng.choice(N_SIMT, size=50, replace=False)
    with Index(d, N_SIMT + 1000, dtype=dtype) as ix:
        ix.add(C, np.arange(N_SIMT, dtype=np.int64), user_codes=user)
        ix.remove(dead)
        rows = ix.export()[0] if dtype == "int8" else C
        ref, bound = (BD.sim_reference_f32 if dtype == "f32" else BD.sim_reference)(Q, rows)
        for nq in SIMT_NQ:
            scoped = nq == 65
            qu = np.full(nq, 1, np.int32) if scoped else None
            got = ix.debug_simt_scores(Q[:nq], q_user=qu)
            hidden = np.zeros(N_SIMT, dtype=bool)
            hidden[dead] = True
            if scoped:
                hidden |= user != 1
            assert got.shape == (nq, N_SIMT)
            assert (got[:, hidden] == -np.inf).all(), "tombstones and rows outside the scope must be -inf"
            assert np.isfinite(got[:, ~hidden]).all(), "a visible row without a score"
            BD.assert_within(f"simt {dtype} d={d} nq={nq}{' scoped' if scoped else ''}", got[:, ~hidden],
                             ref[:nq, ~hidden], bound[:nq, ~hidden])


def test_debug_dumps_refuse_a_short_buffer():
    """The capacity of the output is checked before anything runs: a buffer sized for 64-row tiles is too small for a
    128-row dump, and the dense dumps need nq x rows floats."""
    d = 128
    C = _bf16(np.random.default_rng(1).standard_normal((300, d)))
    with Index(d, 400) as ix:
        ix.add(C, np.arange(300, dtype=np.int64))
        dq = DeviceBuffer(2 * d * 2).upload(to_bf16_bits(C[:2]))
        _opt(ix, b"tc_tile", 128)
        cap = MAX_CTAS * QROWS * 64
        out = DeviceBuffer(cap * 4).upload(np.full(cap, SENTINEL, dtype=np.float32))
        n_ctas = ix.debug_tc_tile(dq.ptr, 2, 1, out.ptr, cap)[0]
        with pytest.raises(N.AuroraError) as e:
            ix.debug_tc_tile(dq.ptr, 2, 1, out.ptr, n_ctas * QROWS * 128 - 1)
        assert e.value.code == N.AUR_ERR_INVALID
        q = to_bf16_bits(C[:2])
        host = np.full(2 * 300, SENTINEL, np.float32)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)   # noqa: E731
        assert ix._lib.aur_debug_simt_scores(ix._h, p(q), 2, None, None, p(host), host.size - 1, None) == N.AUR_ERR_INVALID
        lists, offs, ql = np.arange(300, dtype=np.int64), np.array([0, 300], np.int64), np.zeros(2, np.int32)
        assert ix._lib.aur_debug_list_scores(ix._h, p(q), 2, p(lists), p(offs), 1, p(ql), p(host), host.size - 1,
                                             None) == N.AUR_ERR_INVALID
        assert (host == SENTINEL).all()

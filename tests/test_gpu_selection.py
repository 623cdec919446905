"""The selection stages between the raw similarity scores and the exact fp64 re-rank, at their capacity and boundary
edges: the generic path's 2048-row segments, 32 768-row chunks and list folds, the re-rank's multi-round sort, scalar
gather and wide-shared-memory launch, the tensor-core kernel's partial tiles and padding, the 32-scope limit of the
per-query tenant masks, one search context reused across shapes, and the threshold exchange after a bring-up launch
and across the launch counter's wrap.  Every answer is held to the oracle exactly (tests/gpu_exact.py): ids bit for
bit, fp64 scores within dim * 2^-52 * 4.  Run on an H100 with -m gpu."""

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index, to_bf16_bits
from oracle import cosine_topk as O
from tests.gpu_exact import check_exact, check_host_exact, dev_search

pytestmark = pytest.mark.gpu
SLACK = 8                       # kSlack (csrc/internal.h): candidates kept beyond k for the exact re-rank
SEG, CHUNK, SORT_CAP = 2048, 32768, 4096   # kSimtSeg, the generic path's score chunk, kSortCap
TC = [N.KERNEL_TC1, N.KERNEL_TC2]
ALL = [N.KERNEL_TC1, N.KERNEL_TC2, N.KERNEL_SIMT]


def _bf16(x):
    return O.round_to_bf16(np.asarray(x, dtype=np.float32))


def _rows(n, d, seed, dtype="bf16"):
    x = np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)
    return _bf16(x) if dtype == "bf16" else x


def _near(q, cos, rng):
    """A row whose cosine with q is about `cos` (a component orthogonal to q mixed in)."""
    v = rng.standard_normal(q.shape[0])
    v -= q * (v @ q) / (q @ q)
    v *= np.linalg.norm(q) / np.linalg.norm(v)
    return cos * q + np.sqrt(1.0 - cos * cos) * v


def simt_launches(n_rows, k):
    """Kernels of one generic-path search of <= 1024 queries, as search_enqueue (csrc/capi.cu) enqueues them: scores +
    select per 32 768-row chunk, one list reduction per fold while n_lists * (k + slack) > 4096, the exact re-rank."""
    ksel = k + SLACK
    launches = 2 * -(-n_rows // CHUNK)
    n_lists, folds = -(-n_rows // SEG), 0
    while n_lists * ksel > SORT_CAP:
        n_lists = -(-n_lists // (SORT_CAP // ksel))
        folds += 1
    return launches + folds + 1, folds


def test_generic_path_launch_count_formula():
    assert simt_launches(928 * SEG, 128) == (119, 2)            # 928 lists -> 31 -> 2
    assert simt_launches(316 * SEG - 1000, 5) == (42, 1)        # 316 lists of 13 keys -> 2
    assert simt_launches(70000, 128) == (8, 1)


# ------------------------------------------------------------------------------ generic path: boundaries
@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_simt_best_rows_on_segment_and_chunk_boundaries(dtype):
    """The best rows sit on both sides of a segment boundary (2047 | 2048), of a chunk boundary (32767 | 32768) and in
    the last row, which is alone in its chunk and its list.  Each query ranks them in a different order."""
    n, d, nq, k = 65537, 64, 5, 8
    rng = np.random.default_rng(1)
    C = _rows(n, d, 2, dtype)
    Q = _rows(nq, d, 3, dtype).astype(np.float64)
    spots = np.array([2047, 2048, 32767, 32768, n - 1])
    for j in range(nq):                                          # query j's rows: the spots shifted by j (the last one by 0)
        at = np.array([2047 - j, 2048 + j, 32767 - j, 32768 + j, n - 1 - j])
        for r, (row, cos) in enumerate(zip(at, 0.98 - 0.02 * ((np.arange(5) + j) % 5))):
            C[row] = _near(Q[j], cos, rng)
    C = _bf16(C) if dtype == "bf16" else C.astype(np.float32)
    Q = _bf16(Q) if dtype == "bf16" else Q.astype(np.float32)
    ids = np.arange(n, dtype=np.int64) * 5 + 1
    with Index(d, n, dtype=dtype) as ix:
        ix.add(C, ids)
        ix.set_kernel(N.KERNEL_SIMT)
        got = dev_search(ix, Q, k)
        assert ix.stats()["last_launches"] == simt_launches(n, k)[0]
    want = check_exact(got, Q, C, k, ids=ids)
    assert set(want[0][0, :5].tolist()) == set((spots * 5 + 1).tolist())


@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_simt_best_rows_crowded_into_one_segment(dtype):
    """k + slack + 3 best rows: all but the k-th sit in ONE 2048-row segment, whose list keeps only k + slack of
    them; the k-th best is alone in another segment and must still make the cut."""
    n, d, k = 4 * SEG + 100, 256, 16
    rng = np.random.default_rng(4)
    C = _rows(n, d, 5, dtype)
    q = rng.standard_normal(d)
    Q = (_bf16 if dtype == "bf16" else np.float32)(q[None, :])
    planted = np.concatenate([SEG + 7 + 11 * np.arange(k - 1), [3 * SEG + 1000], SEG + 7 + 11 * np.arange(k - 1, k + SLACK + 2)])
    for r, row in enumerate(planted):
        C[row] = _near(q, 0.95 - 0.01 * r, rng)
    C = _bf16(C) if dtype == "bf16" else C.astype(np.float32)
    with Index(d, n, dtype=dtype) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.set_kernel(N.KERNEL_SIMT)
        got = dev_search(ix, Q, k)
    want = check_exact(got, Q, C, k)
    assert want[0][0].tolist() == planted[:k].tolist()                # the planted order is the true order
    assert len(set(planted.tolist()) - {planted[k - 1]}) == k + SLACK + 2


@pytest.mark.parametrize("n,k,folds", [(928 * SEG, 128, 2), (316 * SEG - 1000, 5, 1)])
def test_simt_list_folds(n, k, folds):
    """928 lists of k + slack = 136 keys fold twice (to 31 groups of 30, then to 2) before the final sort; 316 lists of
    13 keys fold once (groups of 315).  The reduction ping-pongs between two buffers."""
    d, nq = 8, 3
    C = _rows(n, d, n)
    Q = _rows(nq, d, n + 1)
    ids = np.random.default_rng(n).permutation(2 * n)[:n].astype(np.int64)
    with Index(d, n) as ix:
        ix.add(C, ids)
        ix.set_kernel(N.KERNEL_SIMT)
        got = dev_search(ix, Q, k)
        want_launches, want_folds = simt_launches(n, k)
        assert want_folds == folds
        assert ix.stats()["last_launches"] == want_launches
    check_exact(got, Q, C, k, ids=ids)


@pytest.mark.parametrize("kernel", ALL)
@pytest.mark.parametrize("case", ["three_rows_k5", "all_tombstoned", "tenant_of_four_k16"])
def test_fewer_visible_rows_than_k(kernel, case):
    """Fewer visible rows than k (and than k + slack): the answer is padded with (-1, -inf) exactly where the
    oracle pads."""
    d = 64
    rng = np.random.default_rng(7)
    if case == "three_rows_k5":
        n, k, nq = 3, 5, 4
    else:
        n, k, nq = 3000, 16 if case == "tenant_of_four_k16" else 5, 4
    C = _rows(n, d, 8)
    Q = _rows(nq, d, 9)
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    users = np.where(np.isin(np.arange(n), [5, 900, 2047, 2999]), 7, rng.integers(0, 5, n)).astype(np.int32)
    live = np.ones(n, dtype=bool)
    with Index(d, max(n, 64)) as ix:
        ix.add(C, ids, users, np.full(n, -1, np.int32))
        if case == "all_tombstoned":
            assert ix.remove(ids) == n
            live[:] = False
        ix.set_kernel(kernel)
        if case == "tenant_of_four_k16":
            qu, qo = np.full(nq, 7, np.int32), np.full(nq, -1, np.int32)
            got = ix.search(Q, k, qu, qo)                      # one scope for the batch: folds into the row scale
            assert ix.stats()["last_kernel"] == kernel
            want = check_host_exact(got, Q, C, k, ids=ids, row_user=users, row_org=np.full(n, -1), q_user=qu, q_org=qo)
            if kernel == N.KERNEL_SIMT:                         # per-query codes through the device entry point
                check_exact(dev_search(ix, Q, k, q_user=qu, q_org=qo), Q, C, k, ids=ids, row_user=users,
                            row_org=np.full(n, -1), q_user=qu, q_org=qo)
            assert (want[0][:, :4] >= 0).all() and (want[0][:, 4:] == -1).all()
        else:
            got = dev_search(ix, Q, k)
            assert ix.stats()["last_kernel"] == kernel
            want = check_exact(got, Q, C, k, ids=ids, live=live)
            assert (want[0] >= 0).sum() == (0 if case == "all_tombstoned" else nq * n)


@pytest.mark.parametrize("d", [1, 3, 100, 1025])
def test_bf16_index_refuses_dims_that_are_not_a_multiple_of_8(d):
    with pytest.raises(N.AuroraError) as e:
        Index(d, 64)
    assert e.value.code == N.AUR_ERR_INVALID


@pytest.mark.parametrize("dtype,d", [
    ("bf16", 1032), ("bf16", 1536), ("bf16", 3072), ("bf16", 16384),     # > 1024: the re-rank's scalar gather
    ("f32", 1), ("f32", 3), ("f32", 5), ("f32", 100),                    # f32 dim % 4 != 0: scalar gather
    ("f32", 768), ("f32", 1536),                                          # f32 > 512: scalar gather
])
def test_rerank_scalar_gather_and_wide_dims(dtype, d):
    """Dims only the generic path serves, gathered element by element in the re-rank; at 16384 the query beside the
    sort buffer needs the shared-memory opt-in above 48 KB.  k = 40 over 7000 rows also leaves 4 lists of 48 keys.
    At dim 1 every nonzero row scores exactly +1 or -1, a tie group the approximate scores split by rounding noise
    (wider than the slack, which the selection does not promise to cut exactly), so that corpus holds fewer rows than
    k + slack and the exact re-rank alone orders them."""
    n, nq, k = (20 if d == 1 else 7000), 6, 40
    C = _rows(n, d, d, dtype)
    Q = _rows(nq, d, d + 1, dtype)
    rng = np.random.default_rng(d)
    for i in range(nq if d > 1 else 0):
        C[rng.integers(0, n, 3)] = Q[i] + 0.2 * rng.standard_normal((3, d)).astype(np.float32)
    C = _bf16(C) if dtype == "bf16" else C
    with Index(d, n, dtype=dtype) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        got = dev_search(ix, Q, k)
        assert ix.stats()["last_kernel"] == N.KERNEL_SIMT
    check_exact(got, Q, C, k)


@pytest.mark.parametrize("kernel", ALL)
@pytest.mark.parametrize("query", ["zero", "anti_correlated"])
def test_degenerate_queries(kernel, query):
    """A zero query scores 0 against every row: the answer is the k lowest visible ids.  A query anti-correlated with
    an all-positive corpus scores below 0 everywhere: the answer runs from the least negative score."""
    n, d, k = 5000, 256, 32
    rng = np.random.default_rng(12)
    C = _bf16(np.abs(rng.standard_normal((n, d))) + 0.05)
    if query == "zero":
        Q = np.zeros((3, d), np.float32)
    else:
        Q = _bf16(-(np.abs(rng.standard_normal((3, d))) + 0.05))
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    dead = ids[np.argsort(ids)[[0, 5]]]                            # two of the lowest ids are deleted
    live = ~np.isin(ids, dead)
    with Index(d, n) as ix:
        ix.add(C, ids)
        ix.remove(dead)
        ix.set_kernel(kernel)
        got = dev_search(ix, Q, k)
        assert ix.stats()["last_kernel"] == kernel
    want = check_exact(got, Q, C, k, ids=ids, live=live)
    if query == "zero":
        assert (want[0] == np.sort(ids[live])[:k][None, :]).all() and (got[2] == 0.0).all()
    else:
        assert (got[2] < 0).all() and (np.diff(got[2], axis=1) <= 0).all()


# ------------------------------------------------------------------------------ tensor-core path: edges
@pytest.mark.parametrize("kernel", TC)
@pytest.mark.parametrize("n,nq,k", [(64 * 200 + 1, 130, 32), (64 * 41 + 1, 1, 1)])
def test_tc_short_and_partial_tiles(kernel, n, nq, k):
    """64 t + 1 rows with every query's best row alone in the last, partial tile (corpora shorter than one tile are
    shapes of test_tcgen05_parity)."""
    d = 256
    rng = np.random.default_rng(n)
    C = _rows(n, d, n + 1)
    C[n - 1] = _bf16(rng.standard_normal(d))
    Q = _bf16(C[n - 1][None, :] + 0.3 * rng.standard_normal((nq, d)))      # cosine ~0.96 with the last row
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.set_kernel(kernel)
        got = dev_search(ix, Q, k)
        assert ix.stats()["last_kernel"] == kernel
    want = check_exact(got, Q, C, k)
    assert (want[0][:, 0] == n - 1).all()


@pytest.mark.parametrize("kernel", TC)
def test_tc_uniform_scope_with_fewer_visible_rows_than_k(kernel):
    n, d, nq, k = 20000, 256, 70, 32
    rng = np.random.default_rng(3)
    C = _rows(n, d, 4)
    Q = _rows(nq, d, 5)
    users = np.zeros(n, np.int32)
    users[rng.choice(n, 20, replace=False)] = 9
    qu, qo = np.full(nq, 9, np.int32), np.full(nq, -1, np.int32)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), users, np.full(n, -1, np.int32))
        ix.set_kernel(kernel)
        got = ix.search(Q, k, qu, qo)
        assert ix.stats()["last_kernel"] == kernel
    want = check_host_exact(got, Q, C, k, row_user=users, row_org=np.full(n, -1), q_user=qu, q_org=qo)
    assert (want[0][:, :20] >= 0).all() and (want[0][:, 20:] == -1).all()


def _sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc_lists(kernel, nq_launch, k, sm_count):
    """Candidate lists per query of one tensor-core launch (run_tc_block, csrc/capi.cu; one epilogue group)."""
    ksel = k + SLACK
    if kernel == N.KERNEL_TC1 or nq_launch <= 64:
        return (sm_count & ~1) // (2 if nq_launch > 64 else 1)
    pairs = sm_count // 2
    n_super = -(-nq_launch // 128)
    while n_super > 1 and -(-ksel // (pairs // n_super)) > 4:
        n_super -= 1
    return pairs // n_super


@pytest.mark.parametrize("kernel,k,nq", [(N.KERNEL_TC1, 128, 100), (N.KERNEL_TC2, 128, 100), (N.KERNEL_TC1, 32, 64)])
def test_tc_tie_group_overflows_the_sort_buffer(kernel, k, nq):
    """20 000 bit-identical rows are every query's best: every CTA's list fills with tied keys, the compacted row of a
    query holds n_lists * (k + slack) > 4096 keys, and the re-rank sorts it in several rounds.  The lowest ids come
    out, in id order."""
    n, d = 50000, 256
    rng = np.random.default_rng(k + nq)
    C = _rows(n, d, 21)
    group = rng.choice(n, 20000, replace=False)
    C[group] = _bf16(rng.standard_normal(d))
    Q = _bf16(C[group[0]][None, :] + 0.4 * rng.standard_normal((nq, d)))
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    with Index(d, n) as ix:
        ix.add(C, ids)
        ix.set_kernel(kernel)
        got = dev_search(ix, Q, k)
        st = ix.stats()
    assert st["last_kernel"] == kernel
    n_keys = tc_lists(kernel, nq, k, _sm_count()) * (k + SLACK)
    assert n_keys > SORT_CAP
    assert st["last_candidates_max"] > SORT_CAP, st                   # the multi-round sort really ran
    assert st["last_candidates_max"] <= n_keys
    check_exact(got, Q, C, k, ids=ids)
    assert (got[0] == np.sort(ids[group])[:k][None, :]).all()


@pytest.mark.parametrize("n_scopes,kernel", [(32, N.KERNEL_TC2), (33, N.KERNEL_SIMT)])
def test_32_scopes_ride_the_tensor_core_kernel_33_do_not(n_scopes, kernel):
    """Per-query tenant scopes become one bit per distinct scope of the batch: 32 fit (bit 31 in use), 33 fall back to
    the generic kernel.  Query i carries scope i % n_scopes, so the last scope's queries are the batch's last ones."""
    n, d, nq, k = 30000, 256, 99, 16
    rng = np.random.default_rng(n_scopes)
    C = _rows(n, d, 31)
    Q = _rows(nq, d, 32)
    users = rng.integers(0, 40, n).astype(np.int32)
    orgs = rng.integers(-1, 4, n).astype(np.int32)
    qu = (np.arange(nq) % n_scopes).astype(np.int32)
    qo = np.where(qu % 3 == 0, qu % 4, -1).astype(np.int32)
    assert len(set(zip(qu.tolist(), qo.tolist()))) == n_scopes
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), users, orgs)
        got = ix.search(Q, k, qu, qo)
        assert ix.stats()["last_kernel"] == kernel
    check_host_exact(got, Q, C, k, row_user=users, row_org=orgs, q_user=qu, q_org=qo)


# ------------------------------------------------------------------------------ one context, many shapes
def _reuse_steps():
    """Each step: (name, fn(ix, state) -> None).  Device searches run on the index's own stream (one bound context),
    host searches on the pool context; both see every shape, and the debug launch shares the bound context."""
    d = 256

    def plain(kernel, k, nq, seed):
        def run(ix, s):
            Q = _rows(nq, d, seed)
            ix.set_kernel(kernel)
            got = dev_search(ix, Q, k)
            assert ix.stats()["last_kernel"] == kernel
            check_exact(got, Q, s["C"], k, ids=s["ids"], live=s["live"])
            host = ix.search(Q, k)
            assert np.array_equal(host[0], got[0]) and np.array_equal(host[1], got[1])
        return run

    def scoped(ix, s):
        Q = _rows(70, d, 41)
        qu = (np.arange(70) % 20).astype(np.int32)
        qo = np.full(70, -1, np.int32)
        ix.set_kernel(N.KERNEL_AUTO)
        got = ix.search(Q, 32, qu, qo)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        check_host_exact(got, Q, s["C"], 32, ids=s["ids"], live=s["live"], row_user=s["users"],
                         row_org=np.full(len(s["C"]), -1), q_user=qu, q_org=qo)

    def subset(ix, s):
        Q = _rows(9, d, 42)
        allow = s["ids"][::7]
        ix.set_kernel(N.KERNEL_AUTO)
        got = ix.search_subset(Q, 12, allow)
        check_host_exact(got, Q, s["C"], 12, ids=s["ids"], live=s["live"] & np.isin(s["ids"], allow))

    def uniform(ix, s):
        Q = _rows(40, d, 43)
        qu, qo = np.full(40, 3, np.int32), np.full(40, -1, np.int32)
        ix.set_kernel(N.KERNEL_AUTO)
        got = ix.search(Q, 10, qu, qo)
        check_host_exact(got, Q, s["C"], 10, ids=s["ids"], live=s["live"], row_user=s["users"],
                         row_org=np.full(len(s["C"]), -1), q_user=qu, q_org=qo)

    def debug(ix, s):
        Q = _rows(100, d, 44)
        dq = DeviceBuffer(Q.size * 2).upload(to_bf16_bits(Q))
        dout = DeviceBuffer(1024 * 64 * 64 * 4)
        assert ix.debug_tc_scores(dq.ptr, 100, 2, dout.ptr) > 0
        ix.sync()

    def mutate_then_search(ix, s):
        rng = np.random.default_rng(45)
        new = _rows(500, d, 46)
        new_ids = np.concatenate([s["ids"][:100], 10**7 + np.arange(400)]).astype(np.int64)   # 100 upserts, 400 new rows
        new_users = rng.integers(0, 20, 500).astype(np.int32)
        ix.add(new, new_ids, new_users, np.full(500, -1, np.int32))
        s["live"][:100] = False
        gone = s["ids"][1000:1300]
        assert ix.remove(gone) == 300
        s["live"][1000:1300] = False
        s["C"] = np.concatenate([s["C"], new]); s["ids"] = np.concatenate([s["ids"], new_ids])
        s["users"] = np.concatenate([s["users"], new_users]); s["live"] = np.concatenate([s["live"], np.ones(500, bool)])
        plain(N.KERNEL_TC2, 128, 300, 40)(ix, s)

    return [
        ("tc2_k128_nq300", plain(N.KERNEL_TC2, 128, 300, 40)),
        ("simt_k5_nq1", plain(N.KERNEL_SIMT, 5, 1, 47)),
        ("tc2_20_scopes", scoped),
        ("subset", subset),
        ("tc1_k1_nq1025", plain(N.KERNEL_TC1, 1, 1025, 48)),
        ("uniform_scope", uniform),
        ("debug_tc_scores", debug),
        ("tc2_k128_nq300_again", plain(N.KERNEL_TC2, 128, 300, 40)),
        ("add_remove_then_search", mutate_then_search),
    ]


@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_one_index_many_shapes_in_sequence(order):
    """Stale candidate counts, candidate slots, masked inverse norms or scope masks left by one search must not leak
    into the next, whatever shape, kernel and scope kind follows."""
    n, d = 30000, 256
    rng = np.random.default_rng(50)
    s = {"C": _rows(n, d, 51), "ids": rng.permutation(10 * n)[:n].astype(np.int64),
         "users": rng.integers(0, 20, n).astype(np.int32), "live": np.ones(n, dtype=bool)}
    steps = _reuse_steps()
    if order == "reverse":
        steps = steps[::-1]
    with Index(d, n + 1000) as ix:
        ix.add(s["C"], s["ids"], s["users"], np.full(n, -1, np.int32))
        for name, fn in steps:
            try:
                fn(ix, s)
            except AssertionError as e:
                raise AssertionError(f"step {name}: {e}") from e


# ------------------------------------------------------------------------------ the threshold exchange stays alive
EX_N, EX_D, EX_NQ, EX_K = 200_000, 768, 256, 32


@pytest.fixture(scope="module")
def exchange_data():
    C = _rows(EX_N, EX_D, 60)
    Q = _rows(EX_NQ, EX_D, 61)
    return C, Q, O.cosine_topk(Q, C, EX_K, return_f64=True)


def _dead_exchange_keys(kernel):
    """Keys per query the re-rank reads when no threshold is ever certified: every list full."""
    nq_launch = EX_NQ if kernel == N.KERNEL_TC2 else 128
    return tc_lists(kernel, nq_launch, EX_K, _sm_count()) * (EX_K + SLACK)


def _exchange_search(ix, C, Q, want):
    got = dev_search(ix, Q, EX_K)
    check_exact(got, Q, C, EX_K, want=want)
    st = ix.stats()
    return st["last_candidates"] / EX_NQ, st["last_candidates_max"]


@pytest.mark.parametrize("kernel", TC)
def test_threshold_exchange_survives_a_debug_launch(kernel, exchange_data):
    """aur_debug_tc_scores tags its exchange entries from a range searches never use.  A later search on the same
    context must still certify thresholds: its re-rank reads about as many keys as on a fresh index, far fewer than
    the n_lists * (k + slack) it reads when the exchange is dead."""
    C, Q, want = exchange_data
    dead = _dead_exchange_keys(kernel)
    with Index(EX_D, EX_N) as ix:
        ix.add(C, np.arange(EX_N, dtype=np.int64))
        ix.set_kernel(kernel)
        fresh_mean, fresh_max = _exchange_search(ix, C, Q, want)
        dq = DeviceBuffer(128 * EX_D * 2).upload(to_bf16_bits(Q[:128]))
        dout = DeviceBuffer(1024 * 64 * 64 * 4)
        ix.debug_tc_scores(dq.ptr, 128, 1 if kernel == N.KERNEL_TC1 else 2, dout.ptr)
        ix.sync()
        after = [_exchange_search(ix, C, Q, want) for _ in range(3)]
    print(f"kernel {N.KERNEL_NAMES[kernel]}: dead exchange {dead} keys/query; fresh mean {fresh_mean:.1f} max {fresh_max}; "
          f"after debug launch " + ", ".join(f"mean {m:.1f} max {x}" for m, x in after))
    assert fresh_max < dead / 2
    for mean, mx in after:
        assert mx < dead / 2, (mean, mx, dead)


@pytest.mark.parametrize("kernel", TC)
def test_threshold_exchange_survives_the_epoch_wrap(kernel, exchange_data):
    """The launch counter starts 16 launches before it wraps back to 1: the entries the last launches before the wrap
    left behind carry larger tags than the first ones after it, and must not block them."""
    C, Q, want = exchange_data
    dead = _dead_exchange_keys(kernel)
    launches_per_search = 1 if kernel == N.KERNEL_TC2 else 2
    with Index(EX_D, EX_N) as ix:
        ix.add(C, np.arange(EX_N, dtype=np.int64))
        ix.set_kernel(kernel)
        N.check(ix._lib.aur_set_option(ix._h, b"dbg_epoch", 0x7FFFFFFF - 15))
        with pytest.raises(N.AuroraError):
            N.check(ix._lib.aur_set_option(ix._h, b"dbg_epoch", 0x80000000))   # the bring-up launches' range
        counts = [_exchange_search(ix, C, Q, want) for _ in range(32 // launches_per_search)]
    print(f"kernel {N.KERNEL_NAMES[kernel]}: dead exchange {dead} keys/query; across the wrap (mean, max): {counts}")
    for mean, mx in counts:
        assert mx < dead / 2, (counts, dead)

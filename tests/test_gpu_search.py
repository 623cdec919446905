"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same
seeded inputs -- ids bit-exact, scores within 1e-3 (BASELINE.json north_star tolerance; in
practice they agree to fp32 rounding because the final ranking is an fp64 re-score).
Run on an H100:  python -m pytest tests -m gpu"""

import json
import os

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import DeviceBuffer, Index, MultiIndex, cosine_pairs, merge_topk_dev, merge_topk_packed_dev, to_bf16_bits
from oracle import cosine_topk as O
from tests.gpu_exact import check_exact, dev_search

pytestmark = pytest.mark.gpu
TOL = 1e-3
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cosine_ref.json")


def _data(n, d, nq, seed, bf16=True, planted=4):
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    if planted and n >= 8 * nq:
        for i in range(nq):
            rows = rng.choice(n, size=planted, replace=False)
            C[rows] = Q[i][None, :] + 0.3 * rng.standard_normal((planted, d)).astype(np.float32)
    if bf16:
        C, Q = O.round_to_bf16(C), O.round_to_bf16(Q)
    return C, Q


def _check(ids, sc, oids, osc):
    assert np.array_equal(ids, oids), f"{int((ids != oids).sum())} id mismatches"
    fin = np.isfinite(osc)
    assert np.array_equal(np.isfinite(sc), fin)
    if fin.any():
        assert float(np.max(np.abs(sc[fin] - osc[fin]))) <= TOL


def test_library_loaded_and_device_present():
    assert N.load().aur_device_count() >= 1


# ------------------------------------------------------------------ BASELINE config 1 (fp32)
def test_cfg1_fp32_matches_reference_golden():
    g = json.load(open(GOLDEN))["cfg1"]
    C = np.random.default_rng(g["corpus_seed"]).standard_normal((g["N"], g["D"])).astype(np.float32)
    Q = np.random.default_rng(g["query_seed"]).standard_normal((1, g["D"])).astype(np.float32)
    with Index(g["D"], g["N"], dtype="f32") as ix:
        ix.add(C, np.arange(g["N"], dtype=np.int64))
        ids, sc = ix.search(Q, g["k"])
        assert ix.stats()["last_kernel"] == N.KERNEL_SIMT
    assert ids[0].tolist() == g["raw_ids"]                         # produced by the real reference function
    assert np.allclose(sc[0], g["raw_scores"], atol=1e-6)


# ------------------------------------------------------------------ generic (SIMT) path
@pytest.mark.parametrize("n,d,nq,k,dtype", [
    (1000, 384, 1, 5, "f32"), (5000, 768, 33, 32, "bf16"), (700, 100, 7, 10, "f32"), (3, 64, 2, 5, "bf16"),
    (4097, 200, 65, 128, "bf16"), (2048, 8, 3, 1, "bf16"),
    (3, 5, 2, 5, "f32"), (2049, 1536, 4, 16, "bf16"),      # fewer rows than k; the re-rank's scalar gather
])
def test_simt_parity(n, d, nq, k, dtype):
    C, Q = _data(n, d, nq, seed=n + d, bf16=(dtype == "bf16"))
    ext = np.arange(n, dtype=np.int64) * 3 + 7
    want = O.cosine_topk(Q, C, k, ids=ext, return_f64=True)
    with Index(d, max(n, 64), dtype=dtype) as ix:
        ix.set_kernel(N.KERNEL_SIMT)
        ix.add(C, ext)
        ids, sc = ix.search(Q, k)
        check_exact(dev_search(ix, Q, k), Q, C, k, want=want)
    _check(ids, sc, *want[:2])


def test_simt_tenant_filter_and_tombstones():
    n, d, nq, k = 4000, 128, 9, 8
    C, Q = _data(n, d, nq, seed=5)
    rng = np.random.default_rng(9)
    ru, ro = rng.integers(0, 5, n).astype(np.int32), rng.integers(-1, 3, n).astype(np.int32)
    qu, qo = rng.integers(0, 5, nq).astype(np.int32), rng.integers(-1, 3, nq).astype(np.int32)
    live = np.ones(n, dtype=bool)
    with Index(d, n + 100) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), ru, ro)
        dead = rng.choice(n, size=500, replace=False)
        assert ix.remove(dead) == 500
        assert ix.remove(dead[:10]) == 0
        live[dead] = False
        ix.set_kernel(N.KERNEL_SIMT)                            # the generic kernel's own per-query filter
        ids, sc = ix.search(Q, k, qu, qo)
        st = ix.stats()
        ix.set_kernel(N.KERNEL_AUTO)                            # same batch in AUTO: <= 32 scopes -> tensor path, row bit masks
        ids_tc, sc_tc = ix.search(Q, k, qu, qo)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        assert np.array_equal(ids_tc, ids) and np.array_equal(sc_tc, sc)
    assert st["last_kernel"] == N.KERNEL_SIMT and st["live"] == n - 500 and st["rows"] == n
    _check(ids, sc, *O.cosine_topk(Q, C, k, live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo))


@pytest.mark.parametrize("with_org", [False, True])
def test_uniform_tenant_scope_is_served_by_the_tcgen05_kernel(with_org):
    """The reference asks one tenant's question at a time (user_id == u OR org_id == o,
    weaviate_client.py:244-249): with one scope for the whole batch the filter folds into the row scale
    and the tensor-core kernel serves it; a batch mixing up to 32 scopes (the daemon's coalesced requests) rides on the
    same kernel through per-row bit masks; beyond that the generic kernel takes over."""
    n, d, nq, k = 30000, 768, 70, 16
    C, Q = _data(n, d, nq, seed=99)
    rng = np.random.default_rng(5)
    ru = rng.integers(0, 40, n).astype(np.int32)
    ro = rng.integers(-1, 6, n).astype(np.int32)
    live = np.ones(n, dtype=bool)
    qu = np.full(nq, 7, np.int32)
    qo = np.full(nq, 3 if with_org else -1, np.int32)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64), ru, ro)
        gone = np.nonzero(ru == 7)[0][:5].astype(np.int64)           # tombstones inside the tenant's rows
        ix.remove(gone); live[gone] = False
        ids, sc = ix.search(Q, k, qu, qo)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        _check(ids, sc, *O.cosine_topk(Q, C, k, live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo))
        vis = (ru[ids[ids >= 0]] == 7) | ((qo[0] >= 0) & (ro[ids[ids >= 0]] == qo[0]))
        assert vis.all()
        qu2 = qu.copy(); qu2[1] = 8                                    # two different scopes in one batch: row bit masks
        ids2, sc2 = ix.search(Q, k, qu2, qo)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        _check(ids2, sc2, *O.cosine_topk(Q, C, k, live=live, row_user=ru, row_org=ro, q_user=qu2, q_org=qo))
        rng2 = np.random.default_rng(77)                               # a coalesced batch: 20 tenants' questions at once
        qu3 = rng2.integers(0, 20, nq).astype(np.int32); qo3 = (qu3 % 7 - 1).astype(np.int32)   # 20 distinct (user, org) scopes
        ids3, sc3 = ix.search(Q, k, qu3, qo3)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
        _check(ids3, sc3, *O.cosine_topk(Q, C, k, live=live, row_user=ru, row_org=ro, q_user=qu3, q_org=qo3))
        qu4 = np.arange(nq, dtype=np.int32) % 40                       # more than 32 distinct scopes: generic kernel
        ids4, sc4 = ix.search(Q, k, qu4, np.full(nq, -1, np.int32))
        assert ix.stats()["last_kernel"] == N.KERNEL_SIMT
        _check(ids4, sc4, *O.cosine_topk(Q, C, k, live=live, row_user=ru, row_org=ro, q_user=qu4, q_org=np.full(nq, -1, np.int32)))
        none = ix.search(Q, k, np.full(nq, 1234, np.int32), np.full(nq, -1, np.int32))   # a tenant with no rows
        assert (none[0] == -1).all()


# ------------------------------------------------------------------ tensor-core path
@pytest.mark.parametrize("kernel", [N.KERNEL_TC1, N.KERNEL_TC2])
@pytest.mark.parametrize("n,d,nq,k", [
    (30000, 768, 256, 32), (9000, 384, 100, 10), (50001, 512, 200, 100), (20000, 768, 300, 5),
    (777, 64, 1, 1), (12345, 256, 129, 128), (64, 768, 256, 32), (5000, 768, 128, 64),
    # dims up to 1024: the whole query block stays in shared memory beside the TMA ring
    (20000, 1024, 256, 32), (9000, 1024, 300, 64), (7000, 896, 130, 10), (4000, 832, 64, 5),
    # corpora shorter than one tile (fewer rows than k: padding)
    (1, 256, 3, 5), (63, 128, 70, 32),
])
def test_tcgen05_parity(kernel, n, d, nq, k):
    C, Q = _data(n, d, nq, seed=n % 1000 + nq + d)
    want = O.cosine_topk(Q, C, k, return_f64=True)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.set_kernel(kernel)
        ids, sc = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == kernel
        check_exact(dev_search(ix, Q, k), Q, C, k, want=want)
    _check(ids, sc, *want[:2])


@pytest.mark.parametrize("n,d,nq,k", [
    (40000, 768, 1024, 32), (30000, 768, 600, 10), (25000, 1024, 1024, 100), (60000, 768, 512, 32), (3000, 768, 900, 64),
    (20000, 768, 257, 128), (9000, 512, 1024, 5), (70000, 768, 2100, 16),
])
def test_query_super_blocks(n, d, nq, k):
    """More than 256 queries per launch: up to four CTA pairs ("query super-blocks") walk the same corpus tiles side by
    side (the corpus crosses HBM once per 256 x S queries, the siblings hit L2).  Fewer tile sets scan the corpus then, so
    every CTA vouches for 2-4 rows in the threshold exchange (best four chunk maxima); batches past 1024 queries and
    large k (fewer super-blocks per launch) split into several launches."""
    C, Q = _data(n, d, nq, seed=n % 977 + nq + k, planted=3)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ids, sc = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
    _check(ids, sc, *O.cosine_topk(Q, C, k))


@pytest.mark.parametrize("kernel", [N.KERNEL_TC1, N.KERNEL_TC2])
@pytest.mark.parametrize("tiles_per_pair", [1, 2, 5])
def test_one_strong_row_per_tile_large_k(kernel, tiles_per_pair):
    """Adversarial for the threshold exchange with two published values per CTA (k + slack > 74 CTA pairs,
    i.e. k >= 67): every 64-row tile holds exactly one row close to the query and 63 unrelated ones, so a
    CTA that counted its best row twice would certify a threshold only ~half of the claimed rows reach and
    the tail of the top-128 would be dropped.  Also the shape a tenant mask produces (about one visible
    row per tile)."""
    d, nq, k = 768, 6, 128
    n = 74 * 64 * tiles_per_pair
    rng = np.random.default_rng(tiles_per_pair)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    for t in range(n // 64):
        for i in range(nq):
            C[t * 64 + (7 * i + t) % 64] = Q[i] * (1.0 + 0.01 * i) + 0.05 * rng.standard_normal(d).astype(np.float32)
    C, Q = O.round_to_bf16(C), O.round_to_bf16(Q)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ix.set_kernel(kernel)
        ids, sc = ix.search(Q, k)
    assert (ids >= 0).all()
    _check(ids, sc, *O.cosine_topk(Q, C, k))


def test_large_k_at_dim_1024_falls_back_in_auto_mode():
    """dim 1024 with k = 128: the lists (k + slack per query) plus the shared-memory part of
    the queries leave no room for a TMA ring, so AUTO serves it with the generic kernel and an explicit
    tensor-core request is refused."""
    n, d, nq, k = 6000, 1024, 70, 128
    C, Q = _data(n, d, nq, seed=5)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ids, sc = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == N.KERNEL_SIMT
        ix.set_kernel(N.KERNEL_TC2)
        with pytest.raises(N.AuroraError) as e:
            ix.search(Q, k)
        assert e.value.code == N.AUR_ERR_UNSUPPORTED
    _check(ids, sc, *O.cosine_topk(Q, C, k))


@pytest.mark.parametrize("nq", [70, 300, 512])
def test_cfg4_shape_class_dim1024_top100_on_tcgen05(nq):
    """BASELINE config 4's shape class (dim 1024, top-100): served by CTA pairs; a short tail block of the
    batch runs as a pair with a padding query block because single-CTA stages no longer fit."""
    n, d, k = 9000, 1024, 100
    C, Q = _data(n, d, nq, seed=nq + 1)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ids, sc = ix.search(Q, k)
        assert ix.stats()["last_kernel"] == N.KERNEL_TC2
    _check(ids, sc, *O.cosine_topk(Q, C, k))


@pytest.mark.parametrize("kernel", [N.KERNEL_TC1, N.KERNEL_TC2])
def test_tcgen05_duplicates_zero_rows_tombstones_upserts(kernel):
    n, d, nq, k = 20000, 768, 256, 32
    C, Q = _data(n, d, nq, seed=77)
    C[1000:1040] = C[999]                       # 41 bit-identical rows: ties broken by id
    C[5000:5010] = 0.0                          # zero-norm rows score 0.0
    C[7] = Q[3]                                 # exact match: cosine 1
    ids0 = np.arange(n, dtype=np.int64)
    live = np.ones(n, dtype=bool)
    with Index(d, n + 64) as ix:
        ix.add(C, ids0)
        gone = np.array([7, 1003, 15000], dtype=np.int64)
        assert ix.remove(gone) == 3
        live[gone] = False
        ix.set_kernel(kernel)
        ids, sc = ix.search(Q, k)
        _check(ids, sc, *O.cosine_topk(Q, C, k, ids=ids0, live=live))
        # upsert: id 42 gets a new vector; the old row must never come back
        newv = O.round_to_bf16((Q[5] * 2.0)[None, :])
        ix.add(newv, np.array([42], dtype=np.int64))
        ids, sc = ix.search(Q, k)
    C2 = np.concatenate([C, newv])
    ids2 = np.concatenate([ids0, [42]])
    live2 = np.concatenate([live, [True]])
    live2[42] = False
    _check(ids, sc, *O.cosine_topk(Q, C2, k, ids=ids2, live=live2))
    assert ids[5, 0] == 42 and abs(sc[5, 0] - 1.0) < 1e-6


def test_auto_kernel_selection_and_device_entry_point():
    n, d, nq, k = 10000, 768, 256, 32
    C, Q = _data(n, d, nq, seed=3)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        ids, sc = ix.search(Q, k)
        st = ix.stats()
        assert st["last_kernel"] == N.KERNEL_TC2 and st["last_launches"] >= 2
        dq = DeviceBuffer(nq * d * 2).upload(to_bf16_bits(Q))
        ds, di, d64 = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8), DeviceBuffer(nq * k * 8)
        ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr, d64.ptr)
        ix.sync()
        sc_d = ds.download(np.empty((nq, k), np.float32))
        ids_d = di.download(np.empty((nq, k), np.int64))
        s64 = d64.download(np.empty((nq, k), np.float64))
    assert np.array_equal(ids, ids_d) and np.array_equal(sc, sc_d)
    assert np.array_equal(s64.astype(np.float32), sc_d)
    assert np.all(np.diff(s64, axis=1) <= 0)                   # sorted best-first
    _check(ids, sc, *O.cosine_topk(Q, C, k))


def test_unsupported_shapes_fail_loudly():
    with Index(100, 256, dtype="f32") as ix:
        ix.add(np.ones((4, 100), np.float32), np.arange(4, dtype=np.int64))
        ix.set_kernel(N.KERNEL_TC2)
        with pytest.raises(N.AuroraError) as e:
            ix.search(np.ones((1, 100), np.float32), 2)
        assert e.value.code == N.AUR_ERR_UNSUPPORTED
        ix.set_kernel(N.KERNEL_AUTO)
        with pytest.raises(N.AuroraError):
            ix.search(np.ones((1, 100), np.float32), 1000)       # k > 128
    with Index(64, 8) as ix:
        with pytest.raises(N.AuroraError) as e:
            ix.add(np.ones((9, 64), np.float32), np.arange(9, dtype=np.int64))
        assert e.value.code == N.AUR_ERR_NOMEM


# ------------------------------------------------------------------ row-sharded corpus: exact cross-shard merge
def test_two_shards_merge_equals_single_index():
    n, d, nq, k, G = 40000, 768, 256, 32, 2
    C, Q = _data(n, d, nq, seed=21)
    C[100] = C[30000]                                          # a tie across shards
    full_ids, full_sc = O.cosine_topk(Q, C, k)
    qbits = to_bf16_bits(Q)
    per = n // G
    s64 = np.empty((G, nq, k), np.float64)
    sid = np.empty((G, nq, k), np.int64)
    for g in range(G):
        with Index(d, per) as ix:
            ix.add(C[g * per:(g + 1) * per], np.arange(g * per, (g + 1) * per, dtype=np.int64))
            dq = DeviceBuffer(qbits.nbytes).upload(qbits)
            ds, di, d64 = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8), DeviceBuffer(nq * k * 8)
            ix.search_dev(dq.ptr, nq, k, ds.ptr, di.ptr, d64.ptr)
            ix.sync()
            s64[g] = d64.download(np.empty((nq, k), np.float64))
            sid[g] = di.download(np.empty((nq, k), np.int64))
    din_s, din_i = DeviceBuffer(s64.nbytes).upload(s64), DeviceBuffer(sid.nbytes).upload(sid)
    dos, doi = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8)
    merge_topk_dev(0, din_s.ptr, din_i.ptr, G, nq, k, dos.ptr, doi.ptr)
    ids = doi.download(np.empty((nq, k), np.int64))
    sc = dos.download(np.empty((nq, k), np.float32))
    _check(ids, sc, full_ids, full_sc)
    # the packed layout used by the single all-gather: [shard][plane 0 = fp64 keys | plane 1 = ids]
    packed = np.empty((G, 2, nq, k), np.int64)
    packed[:, 0] = s64.view(np.int64)
    packed[:, 1] = sid
    dpk = DeviceBuffer(packed.nbytes).upload(packed)
    dos2, doi2 = DeviceBuffer(nq * k * 4), DeviceBuffer(nq * k * 8)
    merge_topk_packed_dev(0, dpk.ptr, G, nq, k, dos2.ptr, doi2.ptr)
    assert np.array_equal(doi2.download(np.empty((nq, k), np.int64)), ids)
    assert np.array_equal(dos2.download(np.empty((nq, k), np.float32)), sc)


# ------------------------------------------------------------------ in-repo cosine (a7)
def test_cosine_pairs_matches_reference_golden():
    g = json.load(open(GOLDEN))
    by_dim = {}
    for e in g["random_pairs"]:
        by_dim.setdefault(len(e["a"]), []).append(e)
    for dim, es in by_dim.items():
        a = np.array([e["a"] for e in es], dtype=np.float32)
        b = np.array([e["b"] for e in es], dtype=np.float32)
        raw = cosine_pairs(a, b)
        clamped = cosine_pairs(a, b, clamp=True)
        assert np.allclose(raw, [e["raw"] for e in es], atol=1e-9)
        assert np.allclose(clamped, [e["clamped"] for e in es], atol=1e-9)


# ------------------------------------------------------------------ BASELINE config 2 at full size: properties
def test_cfg2_full_size_properties():
    """1M x 768 bf16, 256 queries, top-32: planted neighbours are found, the tensor-core
    variants agree with each other bit for bit, a repeated search is identical, and a
    subsample of queries matches the oracle."""
    n, d, nq, k, P = 1_000_000, 768, 256, 32, 8
    rng = np.random.default_rng(1002)
    Qf = O.round_to_bf16(np.random.default_rng(2002).standard_normal((nq, d)).astype(np.float32))
    bits = np.empty((n, d), dtype=np.uint16)
    for lo in range(0, n, 100_000):
        bits[lo:lo + 100_000] = to_bf16_bits(rng.standard_normal((100_000, d)).astype(np.float32))
    prng = np.random.default_rng(3002)
    planted = prng.choice(n, size=(nq, P), replace=False)
    for i in range(nq):
        noise = prng.standard_normal((P, d)).astype(np.float32) * (0.1 * (1 + np.arange(P))[:, None])
        bits[planted[i]] = to_bf16_bits(Qf[i][None, :] + noise)     # increasing noise => known order
    with Index(d, n) as ix:
        for lo in range(0, n, 250_000):
            ix.add(bits[lo:lo + 250_000], np.arange(lo, lo + 250_000, dtype=np.int64))
        res = {}
        for kern in (N.KERNEL_TC2, N.KERNEL_TC1):
            ix.set_kernel(kern)
            res[kern] = ix.search(Qf, k)
        again = ix.search(Qf, k)
    ids, sc = res[N.KERNEL_TC2]
    assert np.array_equal(np.sort(ids[:, :P], axis=1), np.sort(planted, axis=1))   # the planted rows lead
    assert np.array_equal(ids[:, 0], planted[:, 0])                  # least-noisy copy first
    assert np.all(np.diff(sc, axis=1) <= 0)
    assert np.array_equal(res[N.KERNEL_TC1][0], ids) and np.array_equal(res[N.KERNEL_TC1][1], sc)
    assert np.array_equal(again[0], res[N.KERNEL_TC1][0])
    sub = [0, 100, 255]
    oids, osc = O.cosine_topk(Qf[sub], O.bf16_bits_to_f32(bits), k)
    _check(ids[sub], sc[sub], oids, osc)


def test_export_save_load_roundtrip(tmp_path):
    """aur_export / Index.save / Index.load: the restored shard answers exactly like the original,
    tombstones are compacted away."""
    n, d, nq, k = 3000, 128, 16, 10
    C, Q = _data(n, d, nq, seed=77)
    ids = np.arange(100, 100 + n, dtype=np.int64)
    user = (np.arange(n) % 3).astype(np.int32)
    org = np.full(n, -1, np.int32)
    with Index(d, 4096) as ix:
        ix.add(C, ids, user, org)
        ix.remove(ids[::7])
        rows, eid, eu, eo, live = ix.export()
        assert rows.shape == (n, d) and np.array_equal(eid, ids) and np.array_equal(eu, user)
        assert np.array_equal(live, ~np.isin(ids, ids[::7]))
        assert np.array_equal(rows, to_bf16_bits(C))
        want = ix.search(Q, k)
        ix.save(str(tmp_path / "shard"))
    with Index.load(str(tmp_path / "shard")) as ix2:
        st = ix2.stats()
        assert st["rows"] == st["live"] == int(live.sum())
        got = ix2.search(Q, k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("nq", [1, 130, 200])
def test_partial_query_blocks_stay_correct_over_many_launches(nq):
    """A batch that does not fill its last 128-query block leaves padding rows in the kernel; they must not
    accumulate candidates across launches (their counters are never reset by the finalize step)."""
    n, d, k = 30000, 768, 32
    C, Q = _data(n, d, nq, seed=nq)
    want = O.cosine_topk(Q, C, k)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        for kern in (N.KERNEL_TC2, N.KERNEL_TC1):
            ix.set_kernel(kern)
            for _ in range(40):
                ids, sc = ix.search(Q, k)
            _check(ids, sc, *want)


def test_sharded_searcher_single_rank_on_gpu():
    """aurora_b200.sharded.make_gpu_searcher (the wiring bench.py's N > 1 path uses) at world size 1:
    local search + device merge must reproduce Index.search."""
    torch = pytest.importorskip("torch")
    from aurora_b200.sharded import make_gpu_searcher

    n, d, nq, k = 20000, 768, 64, 16
    C, Q = _data(n, d, nq, seed=3)
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        want_ids, want_sc = ix.search(Q, k)
        q_dev = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).cuda()
        ids, sc = make_gpu_searcher(ix, world=1, device=0).search(q_dev, k)
        torch.cuda.synchronize()
    assert np.array_equal(ids.cpu().numpy(), want_ids)
    assert np.array_equal(sc.cpu().numpy(), want_sc)


def test_concurrent_ingest_and_search_threads():
    """BASELINE config 5's access pattern in miniature: one thread appends chunk batches while three others search
    (the reference is hit from gunicorn threads and Celery workers at once).  The shard publishes its row count
    only after a batch has landed and a search scans exactly the prefix published when it was enqueued, so EVERY
    answer must equal the oracle's top-k of exactly the prefix the call reports (aur_search_ex) -- ids bit-exact."""
    import threading

    d, k, batches, per = 768, 8, 24, 512
    rng = np.random.default_rng(11)
    Q = O.round_to_bf16(rng.standard_normal((32, d)).astype(np.float32))
    blocks = [O.round_to_bf16(rng.standard_normal((per, d)).astype(np.float32)) for _ in range(batches)]
    blocks[5][7] = Q[3]                                    # exact match appears with batch 5 (id 5*512+7)
    C = np.concatenate(blocks)
    errors, done, answers = [], threading.Event(), []
    with Index(d, batches * per) as ix:
        def writer():
            try:
                for b, blk in enumerate(blocks):
                    ix.add(blk, np.arange(b * per, (b + 1) * per, dtype=np.int64))
            except Exception as e:      # pragma: no cover
                errors.append(e)
            finally:
                done.set()

        def reader(slot):
            try:
                mine = []
                while not done.is_set() or len(mine) < 2:
                    ids, sc, snap = ix.search_snapshot(Q, k)
                    assert snap % per == 0 and 0 <= snap <= batches * per       # only whole, landed batches are visible
                    mine.append((snap, ids, sc))
                answers.append(mine)
            except Exception as e:      # pragma: no cover
                errors.append(e)

        ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader, args=(i,)) for i in range(3)]
        [t.start() for t in ts]; [t.join() for t in ts]
        assert not errors, errors[0]
        ids, sc = ix.search(Q, k)
    _check(ids, sc, *O.cosine_topk(Q, C, k))
    seen = set()
    oracle = {}
    for mine in answers:
        snaps = [s_ for s_, _, _ in mine]
        assert snaps == sorted(snaps)                                         # a thread never sees the shard shrink
        for snap, ids_t, sc_t in mine:
            seen.add(snap)
            if snap not in oracle:
                if snap == 0:
                    oracle[0] = (np.full((32, k), -1, np.int64), np.full((32, k), -np.inf, np.float32))
                else:
                    oracle[snap] = O.cosine_topk(Q, C[:snap], k)
            _check(ids_t, sc_t, *oracle[snap])
    assert len(seen) >= 2                                                      # readers really overlapped the writer


def test_search_subset_is_a_pre_filter():
    """aur_search_subset: a resolved metadata filter (ids) restricts the scan itself -- the allowed rows are found even
    when thousands of better-scoring rows exist outside the list.  tensor-core and generic kernels, with tombstones."""
    n, d, nq, k = 40000, 768, 5, 10
    C, Q = _data(n, d, nq, seed=21)
    rng = np.random.default_rng(3)
    ext = np.arange(n, dtype=np.int64) * 2 + 1
    allow_rows = np.sort(rng.choice(n, size=300, replace=False))
    live = np.zeros(n, dtype=bool); live[allow_rows] = True
    with Index(d, n) as ix:
        ix.add(C, ext)
        dead = allow_rows[:7]
        ix.remove(ext[dead]); live[dead] = False
        unknown = np.array([10**12, 4], dtype=np.int64)                          # ids that do not exist are ignored
        for kern in (N.KERNEL_AUTO, N.KERNEL_SIMT):
            ix.set_kernel(kern)
            ids, sc = ix.search_subset(Q, k, np.concatenate([ext[allow_rows], unknown]))
            _check(ids, sc, *O.cosine_topk(Q, C, k, ids=ext, live=live))
        ix.set_kernel(N.KERNEL_AUTO)
        assert ix.stats()["last_kernel"] in (N.KERNEL_SIMT, N.KERNEL_TC2)
        few, _ = ix.search_subset(Q, k, ext[allow_rows[7:10]])
        assert (few[:, :3] >= 0).all() and (few[:, 3:] == -1).all()
        none, _ = ix.search_subset(Q, k, np.zeros(0, dtype=np.int64))
        assert (none == -1).all()
        ids_all, sc_all = ix.search(Q, k)                                        # the mask does not leak into plain searches
        live_all = np.ones(n, dtype=bool); live_all[dead] = False
        _check(ids_all, sc_all, *O.cosine_topk(Q, C, k, ids=ext, live=live_all))


@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_compaction_reclaims_tombstones(dtype):
    """Upserts and deletes leave dead rows behind (the prediscovery job re-inserts its chunks periodically,
    weaviate_client.py:374-394); aur_compact moves the live rows down so the shard never fills up with them."""
    n, d, nq, k = 9000, 256, 9, 12
    C, Q = _data(n, d, nq, seed=8, bf16=(dtype == "bf16"))
    rng = np.random.default_rng(4)
    with Index(d, n, dtype=dtype) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        dead = rng.choice(n, size=3000, replace=False)
        assert ix.remove(dead) == 3000
        with pytest.raises(N.AuroraError):                                        # full: 9000 + 1 > capacity
            ix.add(C[:1], np.array([n + 5], dtype=np.int64))
        live = np.ones(n, dtype=bool); live[dead] = False
        before = ix.search(Q, k)
        assert ix.compact() == 3000
        st = ix.stats()
        assert st["rows"] == n - 3000 and st["live"] == n - 3000
        after = ix.search(Q, k)
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        _check(*after, *O.cosine_topk(Q, C, k, live=live))
        assert ix.compact() == 0
        # the freed space is usable again, ids keep resolving (upsert of a moved row, delete of another)
        ix.add(C[dead[:100]], dead[:100].astype(np.int64))
        live[dead[:100]] = True
        survivor = int(np.nonzero(live)[0][-1])
        ix.add(Q[:1], np.array([survivor], dtype=np.int64))                       # replaces that id's vector with query 0
        C2 = C.copy(); C2[survivor] = Q[0]
        ids2, sc2 = ix.search(Q, k)
        assert ids2[0, 0] == survivor
        rows, ids_e, _, _, live_e = ix.export()
        order = {int(i): r for r, i in enumerate(ids_e) if live_e[r]}
        assert len(order) == int(live.sum())
    ref_ids, ref_sc = O.cosine_topk(Q, C2, k, live=live)
    _check(ids2, sc2, ref_ids, ref_sc)


# ------------------------------------------------------------------ one owner process, several shards
def test_multi_index_one_process_many_shards():
    """engine.MultiIndex: one shard per GPU of the box (three shards on the one GPU when there is only one), searched from
    one host thread each and merged on the host -- against the oracle over the whole corpus, with tenant scopes,
    upserts, deletes, a subset pre-filter and concurrent callers."""
    import threading

    n_dev = N.load().aur_device_count()
    devices = list(range(n_dev)) if n_dev > 1 else [0, 0, 0]
    n, d, nq, k = 60000, 768, 40, 16
    C, Q = _data(n, d, nq, seed=321)
    rng = np.random.default_rng(8)
    ids = (rng.permutation(4 * n)[:n]).astype(np.int64)
    ru, ro = rng.integers(0, 6, n).astype(np.int32), rng.integers(-1, 3, n).astype(np.int32)
    live = np.ones(n, dtype=bool)
    with MultiIndex(d, n + 1000, devices=devices) as mi:
        mi.add(C[:35000], ids[:35000], ru[:35000], ro[:35000])
        mi.add(C[35000:], ids[35000:], ru[35000:], ro[35000:])
        st = mi.stats()
        assert st["rows"] == n and st["shards"] == len(devices) and min(st["rows_per_shard"]) > n // len(devices) * 0.9
        got = mi.search(Q, k)
        _check(*got, *O.cosine_topk(Q, C, k, ids=ids))
        gone = ids[11:9000:13]
        assert mi.remove(gone) == len(gone)
        live[11:9000:13] = False
        C2 = C.copy(); C2[20000:20050] = O.round_to_bf16(C[20000:20050] * 0.25 + 0.5)        # upsert 50 rows
        mi.add(C2[20000:20050], ids[20000:20050], ru[20000:20050], ro[20000:20050])
        qu = np.full(nq, 3, np.int32); qo = np.full(nq, 1, np.int32)
        _check(*mi.search(Q, k, qu, qo), *O.cosine_topk(Q, C2, k, ids=ids, live=live, row_user=ru, row_org=ro, q_user=qu, q_org=qo))
        allow = ids[rng.permutation(n)[:5000]]
        sub_live = live & np.isin(ids, allow)
        _check(*mi.search_subset(Q, k, allow), *O.cosine_topk(Q, C2, k, ids=ids, live=sub_live))
        want = O.cosine_topk(Q, C2, k, ids=ids, live=live)
        errs = []

        def caller():
            try:
                for _ in range(5):
                    _check(*mi.search(Q, k), *want)
            except Exception as e:       # pragma: no cover
                errs.append(e)
        ts = [threading.Thread(target=caller) for _ in range(4)]
        [t.start() for t in ts]; [t.join() for t in ts]
        assert not errs, errs[0]
        assert mi.compact() == int((~live).sum()) + 50
        _check(*mi.search(Q, k), *want)


def test_results_written_straight_into_pinned_host_buffers():
    """aur_search, aur_search_ex, aur_search_subset and aur_search_lists with page-locked result buffers: the re-rank
    kernel writes through the UVA mapping (no device-to-host copies); same answer as with pageable buffers, including a
    multi-pass batch (> 1024 queries) and the generic kernel."""
    import ctypes as C
    from aurora_b200.engine import lists_csr
    torch = pytest.importorskip("torch")

    def vp(a):
        return C.c_void_p(a.ctypes.data)

    n, d, k = 30000, 768, 24
    for nq, kernel in ((70, N.KERNEL_AUTO), (1300, N.KERNEL_AUTO), (9, N.KERNEL_SIMT)):
        C_, Q = _data(n, d, nq, seed=nq)
        rng = np.random.default_rng(nq)
        allow = np.ascontiguousarray(rng.choice(n, size=n // 3, replace=False).astype(np.int64))
        lists = [rng.choice(n, size=m, replace=False) for m in (50, 3000, 9000)]
        q_list = np.ascontiguousarray(rng.integers(0, len(lists), size=nq), dtype=np.int32)
        flat, offsets = lists_csr(lists)
        with Index(d, n) as ix:
            ix.add(C_, np.arange(n, dtype=np.int64))
            ix.set_kernel(kernel)
            want_ids, want_sc = ix.search(Q, k)                       # numpy (pageable) buffers
            want = {"search": (want_ids, want_sc), "search_ex": (want_ids, want_sc),
                    "subset": ix.search_subset(Q, k, allow), "lists": ix.search_lists(Q, k, lists, q_list)}
            q = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).pin_memory()
            qp = C.c_void_p(q.data_ptr())
            snap = C.c_int64(-1)
            calls = {
                "search": lambda s, i: ix._lib.aur_search(ix._h, qp, nq, k, None, None, s, i),
                "search_ex": lambda s, i: ix._lib.aur_search_ex(ix._h, qp, nq, k, None, None, s, i, C.byref(snap)),
                "subset": lambda s, i: ix._lib.aur_search_subset(ix._h, qp, nq, k, vp(allow), allow.shape[0], s, i),
                "lists": lambda s, i: ix._lib.aur_search_lists(ix._h, qp, nq, k, vp(flat), vp(offsets), len(lists),
                                                               vp(q_list), s, i, C.byref(snap)),
            }
            for name, call in calls.items():
                h_sc = torch.full((nq, k), float("nan"), dtype=torch.float32).pin_memory()
                h_id = torch.full((nq, k), -7, dtype=torch.int64).pin_memory()
                snap.value = -1
                N.check(call(C.c_void_p(h_sc.data_ptr()), C.c_void_p(h_id.data_ptr())))
                w_ids, w_sc = want[name]
                assert np.array_equal(h_id.numpy(), w_ids) and np.array_equal(h_sc.numpy(), w_sc), name
                if name in ("search_ex", "lists"):
                    assert snap.value == n, name
        _check(want_ids, want_sc, *O.cosine_topk(Q, C_, k))

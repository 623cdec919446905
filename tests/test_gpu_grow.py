"""aur_reserve / aur_kw_reserve: a vector shard and a keyword store grow in place while they serve.  A shard grown step
by step from 1,000 rows answers every kind of search byte for byte as its twin opened at the final capacity, with the
same adds, upserts, deletes and attribute codes; a grown keyword store scores bit for bit as one opened large; searches
running while a writer grows and appends answer exactly over the prefix they report; a device search enqueued before a
growth and a CUDA graph captured before it still answer over what they saw; a knowledge base opened at 512 chunks
ingests 5,000 and answers as one opened at 8,192."""

from __future__ import annotations

import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index, KeywordIndex, KeywordVocab, MultiIndex, MultiKeywordIndex, hybrid_search, to_bf16_bits
from aurora_b200.filters import Filter
from oracle import cosine_topk as O
from tests.test_gpu_delete_filtered import Table, _props

pytestmark = pytest.mark.gpu

F = Filter.by_property
STEPS = (1_000, 4_000, 20_000, 70_000, 140_000, 200_000)   # capacities the grown shard passes through (2 MiB granules
                                                           # hold 1,365 rows of 768 bf16, 2,730 int8, 5,461 of 96 f32)
UPSERTS, REMOVES = 200, 100


def _opt(ix, key, v):
    N.check(ix._lib.aur_set_option(ix._h, key, int(v)))


def _grow_twins(dtype, dim, seed=0):
    """(A grown through STEPS, B opened at STEPS[-1], the shared Table, query rows, rng) after identical writes."""
    rng = np.random.default_rng(seed)
    n = STEPS[-1]
    Cm = O.round_to_bf16(rng.standard_normal((n, dim)).astype(np.float32))
    ext = rng.permutation(4 * n)[:n].astype(np.int64) * 3 + 7
    user = rng.integers(40, size=n).astype(np.int32)
    org = rng.integers(-1, 6, size=n).astype(np.int32)
    props = _props(rng, n)
    A, B = Index(dim, STEPS[0], dtype=dtype), Index(dim, n, dtype=dtype)
    t = Table()
    rows, new = 0, 0                                     # rows appended, new ids used
    for i, cap in enumerate(STEPS):
        if i:
            A.reserve(cap)
            assert A.stats()["capacity"] == cap and A.capacity == cap
        ups = UPSERTS if i else 0
        m = cap - rows - ups
        sl = slice(new, new + m)
        coded = i <= 1                                   # rows of the first two steps get attribute codes, later ones none
        for ix in (A, B):
            ix.add(Cm[sl], ext[sl], user[sl], org[sl])
        t.rows += props[sl] if coded else [{}] * m
        if coded:
            for c in t.cols.values():
                codes = np.array([c.code(p) for p in props[sl]], np.int32)
                for ix in (A, B):
                    ix.set_attrs(c.col, ext[sl], codes)
        if ups:                                          # upserts: new vectors for old ids, appended behind
            old = rng.choice(new, size=ups, replace=False)
            vec = O.round_to_bf16(rng.standard_normal((ups, dim)).astype(np.float32))
            for ix in (A, B):
                ix.add(vec, ext[old], user[old], org[old])
            t.rows += [{}] * ups
        new += m
        rows = cap
        gone = ext[rng.choice(new, size=REMOVES, replace=False)]
        assert A.remove(gone) == B.remove(gone)
        assert A.stats()["rows"] == B.stats()["rows"] == cap
    Q = O.round_to_bf16(rng.standard_normal((300, dim)).astype(np.float32))
    Q[:50] = Cm[rng.choice(n, size=50, replace=False)]   # exact matches: ties with upserted / removed rows included
    return A, B, t, Q, rng, ext[:new]


def _same(a, b, what):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), what


def _answers(ix, t, Q, rng_seed, dtype, ids_pool):
    """Every search kind's (ids, scores, ...) on ix, in a fixed order."""
    rng = np.random.default_rng(rng_seed)
    nq, k = 64, 32
    q = Q[:nq]
    out = []
    kernels = [N.KERNEL_AUTO, N.KERNEL_SIMT] + ([N.KERNEL_TC1, N.KERNEL_TC2] if dtype != "f32" else [])
    one = np.full(nq, 3, np.int32), np.full(nq, 2, np.int32)
    few = rng.integers(20, size=nq).astype(np.int32), np.full(nq, -1, np.int32)         # <= 32 scopes: row masks
    many_u = np.arange(300, dtype=np.int32) % 40                                          # 40 scopes: generic kernel
    for kern in kernels:
        for tile in ((64, 128) if kern in (N.KERNEL_TC1, N.KERNEL_TC2) else (0,)):
            ix.set_kernel(kern)
            _opt(ix, b"tc_tile", tile)
            out.append((kern, tile, ix.search(q, k)))
            out.append((kern, tile, "one", ix.search(q, k, *one)))
            out.append((kern, tile, "few", ix.search(q, k, *few)))
            if kern in (N.KERNEL_AUTO, N.KERNEL_SIMT):
                out.append((kern, tile, "many", ix.search(Q, k, many_u)))
    ix.set_kernel(N.KERNEL_AUTO)
    _opt(ix, b"tc_tile", 0)
    allow = rng.choice(ids_pool, size=5000, replace=False)
    out.append(("subset", ix.search_subset(q, k, allow)))
    if dtype != "f32":
        lists = [rng.choice(ids_pool, size=s, replace=False) for s in (10, 3000, 20000)]
        out.append(("lists", ix.search_lists(q, k, lists, rng.integers(3, size=nq).astype(np.int32))))
        progs = [t.program(F("n").less_than(40)), t.program(F("org_id").equal("o3") | F("document_id").like("doc:1*"))]
        qp = (np.arange(nq) % 2).astype(np.int32)
        for mlr in (0, 10 ** 9):                          # masked scan, list side
            r = ix.search_filtered(q, k, progs, qp, max_list_rows=mlr)
            out.append(("filtered", mlr, r[0], r[1], r[2]))
        for e in (F("n").greater_than(50), F("org_id").not_equal("o1")):
            out.append(("count", ix.count_filtered(t.program(e))))
    rows, ids, user, org, live = ix.export()
    out.append(("export", rows, ids, user, org, live))
    out.append(("read_rows",) + tuple(ix.read_rows(1234, 4321)))
    return out


def _flat(v):
    if isinstance(v, (tuple, list)):
        return [a for x in v for a in _flat(x)]
    return [np.asarray(v)]


def _compare(A, B, t, Q, dtype, ids_pool, seed):
    a, b = _answers(A, t, Q, seed, dtype, ids_pool), _answers(B, t, Q, seed, dtype, ids_pool)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        _same(_flat(x), _flat(y), repr(x[:2])[:80])


@pytest.mark.parametrize("dtype,dim", [("bf16", 768), ("int8", 768), ("f32", 96)])
def test_grown_shard_answers_as_one_opened_large(dtype, dim):
    A, B, t, Q, rng, pool = _grow_twins(dtype, dim)
    with A, B:
        _compare(A, B, t, Q, dtype, pool, seed=1)
        # a column first set after the growths: allocated at the grown capacity, every other row absent
        for ix in (A, B):
            ix.set_attrs(5, pool[:777], np.arange(777, dtype=np.int32) % 9)
        if dtype != "f32":
            t5 = Table()
            from aurora_b200.filters import AttrColumn
            t5.cols = {"w": AttrColumn("w", 5)}
            for v in range(9):
                t5.cols["w"].code({"w": v})
            prog = t5.program(F("w").less_than(4))
            assert A.count_filtered(prog) == B.count_filtered(prog) > 0
            e = F("n").less_than(10)
            gone = [A.remove_filtered(t.program(e)), B.remove_filtered(t.program(e))]
            assert len(gone[0]) > 0
            _same(gone[:1], gone[1:], "remove_filtered")
            _compare(A, B, t, Q, dtype, pool, seed=2)
        assert A.compact() == B.compact() > 0
        _compare(A, B, t, Q, dtype, pool, seed=3)


def _kw_docs(rng, n, vocab=400):
    lens = rng.integers(1, 30, size=n)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(lens)
    terms = np.concatenate([np.sort(rng.choice(vocab, size=l, replace=False)) for l in lens]).astype(np.int32)
    tfs = rng.integers(1, 4, size=off[-1]).astype(np.int32)
    return terms, tfs, off


def _kw_add(stores, rng, ids, vocab=400):
    terms, tfs, off = _kw_docs(rng, len(ids), vocab)
    for s in stores:
        s.add(ids, terms, tfs, off, (ids % 7).astype(np.int32), None)


def test_grown_keyword_store_scores_as_one_opened_large():
    """BM25 bit for bit: a term-major index built before growth, appends after it, text appends (from another GPU when
    there are two), hybrid queries against a grown shard and the multi-store search over grown stores."""
    rng = np.random.default_rng(5)
    steps = (500, 3_000, 40_000, 100_000)
    A, B = KeywordIndex(steps[0]), KeywordIndex(steps[-1])
    q_rng = np.random.default_rng(6)
    qt, _, qo = _kw_docs(q_rng, 64)
    nxt = 0
    for i, cap in enumerate(steps):
        if i:
            A.reserve(cap)
            assert A.stats()["capacity"] == cap
        m = cap - A.stats()["docs"] - (50 if i else 0)
        _kw_add((A, B), rng, np.arange(nxt, nxt + m, dtype=np.int64))
        if i:
            _kw_add((A, B), rng, rng.choice(nxt, size=50, replace=False).astype(np.int64))   # upserts
        nxt += m
        if i == 1:
            A.reindex(); B.reindex()                          # a term-major index built before the next growth
        A.remove(np.arange(i, nxt, 97)); B.remove(np.arange(i, nxt, 97))
        ra, rb = A.search(qt, qo, 20), B.search(qt, qo, 20)
        _same(ra[:2], rb[:2], f"kw step {i}")
    # text appends into a grown store, from another GPU's vocabulary when the machine has two
    vocab = KeywordVocab(0)
    words = [f"w{j}" for j in range(60)]
    texts = [" ".join(rng.choice(words, size=int(rng.integers(1, 12)))) for _ in range(2000)]
    dev = 1 if N.load().aur_device_count() >= 2 else 0
    A2, B2 = KeywordIndex(1000, device=dev), KeywordIndex(4000, device=dev)
    A2.reserve(4000)
    for st in (A2, B2):
        st.add_text(vocab, np.arange(2000, dtype=np.int64), texts)
    known = vocab.read(0)
    qw = np.array(sorted(known.index(w) for w in words[:5]), np.int32)
    qwo = np.array([0, len(qw)], np.int64)
    _same(A2.search(qw, qwo, 30)[:2], B2.search(qw, qwo, 30)[:2], "add_text")
    for x in (A2, B2, vocab):
        x.close()
    # hybrid against a grown keyword store and a grown shard
    dim = 128
    Cm = O.round_to_bf16(rng.standard_normal((nxt, dim)).astype(np.float32))
    with Index(dim, 1000) as ia, Index(dim, nxt) as ib:
        ia.reserve(nxt)
        for ix in (ia, ib):
            ix.add(Cm, np.arange(nxt, dtype=np.int64))
        Q = O.round_to_bf16(rng.standard_normal((64, dim)).astype(np.float32))
        ha = hybrid_search(ia, A, Q, 40, qt, qo, 0.6)
        hb = hybrid_search(ib, B, Q, 40, qt, qo, 0.6)
        _same(ha[:3], hb[:3], "hybrid")
    A.close(); B.close()
    # the multi-store search over grown stores
    ma, mb = MultiKeywordIndex(600, devices=[0, 0]), MultiKeywordIndex(20_000, devices=[0, 0])
    ma.reserve(20_000)
    assert ma.stats()["capacity"] == mb.stats()["capacity"]
    _kw_add((ma, mb), rng, np.arange(15_000, dtype=np.int64))
    _same(ma.search(qt, qo, 25)[:2], mb.search(qt, qo, 25)[:2], "multi")
    ma.close(); mb.close()


def test_growth_under_load():
    """One writer grows and appends while three threads search: every answer is the oracle's top-k over exactly the
    prefix it reports, and reported capacity and prefix never decrease."""
    d, k, per, batches = 768, 8, 2048, 24
    rng = np.random.default_rng(11)
    Q = O.round_to_bf16(rng.standard_normal((16, d)).astype(np.float32))
    blocks = [O.round_to_bf16(rng.standard_normal((per, d)).astype(np.float32)) for _ in range(batches)]
    blocks[9][5] = Q[2]
    Cm = np.concatenate(blocks)
    errors, done, answers = [], threading.Event(), []
    with Index(d, per) as ix:
        def writer():
            try:
                for b, blk in enumerate(blocks):
                    ix.reserve((b + 1) * per)
                    ix.add(blk, np.arange(b * per, (b + 1) * per, dtype=np.int64))
            except Exception as e:      # pragma: no cover
                errors.append(e)
            finally:
                done.set()

        def reader():
            try:
                mine, caps = [], []
                while not done.is_set() or len(mine) < 2:
                    caps.append(ix.stats()["capacity"])
                    ids, sc, snap = ix.search_snapshot(Q, k)
                    assert snap % per == 0 and snap <= ix.stats()["capacity"]
                    mine.append((snap, ids, sc))
                assert caps == sorted(caps)
                answers.append(mine)
            except Exception as e:      # pragma: no cover
                errors.append(e)

        ts = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
        [x.start() for x in ts]; [x.join() for x in ts]
        assert not errors, errors[0]
    oracle, seen = {}, set()
    for mine in answers:
        snaps = [s_ for s_, _, _ in mine]
        assert snaps == sorted(snaps)
        for snap, ids, sc in mine:
            seen.add(snap)
            if snap not in oracle:
                oracle[snap] = (O.cosine_topk(Q, Cm[:snap], k) if snap else
                                (np.full((16, k), -1, np.int64), np.full((16, k), -np.inf, np.float32)))
            assert np.array_equal(ids, oracle[snap][0])
            fin = np.isfinite(oracle[snap][1])
            assert np.array_equal(np.isfinite(sc), fin) and np.all(np.abs(sc[fin] - oracle[snap][1][fin]) <= 2e-3)
    assert len(seen) >= 2


def test_device_search_and_captured_graph_across_growth():
    """An aur_search_dev enqueued on a caller stream just before an aur_reserve from another thread answers right, and
    a search captured as a CUDA graph before growth replays afterwards with the answer it gave before."""
    torch = pytest.importorskip("torch")
    d, n, nq, k = 768, 60_000, 256, 32
    rng = np.random.default_rng(3)
    Cm = O.round_to_bf16(rng.standard_normal((2 * n, d)).astype(np.float32))
    Q = O.round_to_bf16(rng.standard_normal((nq, d)).astype(np.float32))
    Q[0] = Cm[n + 5]                                      # found only once the second half is in
    with Index(d, n) as ix:
        ix.add(Cm[:n], np.arange(n, dtype=np.int64))
        want = ix.search(Q, k)
        q_dev = torch.from_numpy(to_bf16_bits(Q).view(np.int16)).cuda()
        s = torch.cuda.Stream()
        sc = torch.empty((nq, k), dtype=torch.float32, device="cuda")
        ids = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        with torch.cuda.stream(s):
            for _ in range(3):
                ix.search_dev(q_dev.data_ptr(), nq, k, sc.data_ptr(), ids.data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
            ix.search_dev(q_dev.data_ptr(), nq, k, sc.data_ptr(), ids.data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        # enqueued, then a reserve from another thread while it may still run
        sc2 = torch.empty_like(sc); ids2 = torch.empty_like(ids)
        ix.search_dev(q_dev.data_ptr(), nq, k, sc2.data_ptr(), ids2.data_ptr(), stream=s.cuda_stream)
        th = threading.Thread(target=ix.reserve, args=(2 * n,))
        th.start(); th.join()
        s.synchronize()
        assert np.array_equal(ids2.cpu().numpy(), want[0]) and np.array_equal(sc2.cpu().numpy(), want[1])
        ix.add(Cm[n:], np.arange(n, 2 * n, dtype=np.int64))
        g.replay()
        s.synchronize()
        torch.cuda.synchronize()
        assert np.array_equal(ids.cpu().numpy(), want[0]) and np.array_equal(sc.cpu().numpy(), want[1])
        now = ix.search(Q, k)
        assert now[0][0, 0] == n + 5 and np.array_equal(now[0], O.cosine_topk(Q, Cm, k)[0])
        del g


def test_reserve_limits():
    with Index(256, 1000) as ix:
        rows = O.round_to_bf16(np.random.default_rng(0).standard_normal((1000, 256)).astype(np.float32))
        ix.add(rows[:600], np.arange(600, dtype=np.int64))
        before = ix.stats()
        ans = ix.search(rows[:8], 5)
        lib = ix._lib
        assert lib.aur_reserve(ix._h, 10) == N.AUR_OK and lib.aur_reserve(ix._h, 1000) == N.AUR_OK
        assert ix.stats()["capacity"] == 1000
        assert lib.aur_reserve(ix._h, 0x7FFFFFC1) == N.AUR_ERR_INVALID
        assert lib.aur_reserve(None, 5000) == N.AUR_ERR_INVALID
        assert lib.aur_reserve(ix._h, 0x7FFFFFC0) == N.AUR_ERR_NOMEM    # 2^31 rows of 512 B: more than the device holds
        after = ix.stats()
        assert (after["rows"], after["live"], after["capacity"]) == (before["rows"], before["live"], before["capacity"])
        _same(ix.search(rows[:8], 5), ans, "after NOMEM")
        ix.add(rows[600:], np.arange(600, 1000, dtype=np.int64))           # up to the old capacity
        with pytest.raises(RuntimeError):
            ix.add(rows[:1], np.array([5000], np.int64))
    kw = KeywordIndex(100)
    assert kw._lib.aur_kw_reserve(kw._h, 50) == N.AUR_OK and kw.stats()["capacity"] == 100
    assert kw._lib.aur_kw_reserve(kw._h, 0x7FFFFFC1) == N.AUR_ERR_INVALID
    assert kw._lib.aur_kw_reserve(None, 500) == N.AUR_ERR_INVALID
    kw.close()
    assert N.load().aur_reserve(None, 1) == N.AUR_ERR_INVALID


def test_reserve_rolls_back_when_memory_runs_out():
    """A capacity inside every array's address room whose rows do not fit the free memory: the row array (512 B a row)
    and the other base arrays map, the attribute columns cannot all map, and everything mapped is unmapped again --
    the memory comes back, stats and answers are unchanged, adds up to the old capacity and a later growth succeed."""
    torch = pytest.importorskip("torch")
    d = 256
    rng = np.random.default_rng(4)
    rows = O.round_to_bf16(rng.standard_normal((5000, d)).astype(np.float32))
    with Index(d, 1000) as ix:
        ids = np.arange(600, dtype=np.int64)
        ix.add(rows[:600], ids)
        for col in (2, 3, 4):
            ix.set_attrs(col, ids, (ids % 7).astype(np.int32))
        before, ans = ix.stats(), ix.search(rows[:8], 5)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0, _ = torch.cuda.mem_get_info()
        # base arrays 532 B a row (rows 512, inv 4, ids 8, user 4, org 4) fit in ~99 % of the free memory, the three
        # attribute columns' 12 B a row do not
        cap = free0 // 538
        assert ix._lib.aur_reserve(ix._h, int(cap)) == N.AUR_ERR_NOMEM
        free1, _ = torch.cuda.mem_get_info()
        assert free1 >= free0 - (64 << 20), (free0, free1)          # every new mapping was released
        after = ix.stats()
        assert (after["rows"], after["live"], after["capacity"]) == (before["rows"], before["live"], before["capacity"])
        _same(ix.search(rows[:8], 5), ans, "after the rollback")
        ix.add(rows[600:1000], np.arange(600, 1000, dtype=np.int64))
        ix.reserve(5000)
        ix.add(rows[1000:], np.arange(1000, 5000, dtype=np.int64))
        got = ix.search(rows[:64], 5)
        assert np.array_equal(got[0], O.cosine_topk(rows[:64], rows, 5)[0])


@pytest.mark.parametrize("multi", [False, True])
def test_knowledge_base_ingests_past_its_opening_capacity(tmp_path, multi):
    from aurora_b200 import retriever as R
    from tests.test_gpu_encoder_multi import WORDS, _live_rows, _shape, _text_encoder

    devs = [0, 1] if N.load().aur_device_count() >= 2 else [0, 0]
    te = _text_encoder(sorted(set(devs)) if multi else (0,))
    fac = (lambda d, c: MultiIndex(d, c, devices=devs)) if multi else None
    small = R.KnowledgeBase(te, capacity=512, index_factory=fac)
    large = R.KnowledgeBase(te, capacity=8192, index_factory=fac)
    assert te.can_append(small.index)
    rng = np.random.default_rng(9)
    for d in range(50):
        chunks = [{"chunk_index": c, "content": " ".join(rng.choice(WORDS, size=int(rng.integers(3, 30))))} for c in range(100)]
        for kb in (small, large):
            assert kb.insert(f"u{d % 4}", f"doc-{d}", "f.md", chunks, org_id=f"o{d % 3}") == 100
    shards = small.index.shards if multi else [small.index]
    assert sum(sh.stats()["rows"] for sh in shards) == 5000 and all(sh.capacity > 512 for sh in shards)
    assert _live_rows(small.index) == _live_rows(large.index)
    qs = ["disk pressure node", "kafka consumer lag alert", "payment service latency"]
    f = F("org_id").equal("o1") & F("document_id").like("doc-1*")
    for q in qs:
        for a in (None, 0.5):
            assert _shape(small.query(q, 10, alpha=a)) == _shape(large.query(q, 10, alpha=a))
            assert _shape(small.query(q, 10, user_id="u1", org_id="o0", alpha=a)) == _shape(large.query(q, 10, user_id="u1", org_id="o0", alpha=a))
            assert _shape(small.query(q, 10, filters=f, alpha=a)) == _shape(large.query(q, 10, filters=f, alpha=a))
    reqs = [(f"u{i % 4}", q, 6, a, f"o{i % 3}") for i, q in enumerate(qs) for a in (None, 0.3)]
    assert [_shape(r) for r in small.query_batch(reqs)] == [_shape(r) for r in large.query_batch(reqs)]
    snap = str(tmp_path / "kb")
    small.save(snap)
    loader = (lambda p, cap: MultiIndex.load(p, capacity=cap, devices=devs)) if multi else None
    again = R.KnowledgeBase.load(snap, te, capacity=512, index_loader=loader) if multi else R.KnowledgeBase.load(snap, te, capacity=512)
    assert _live_rows(again.index) == _live_rows(small.index)
    from aurora_b200.engine import GROW_STEP
    # each shard restored at its rows rounded up once to the growth step, not at twice its rows
    assert all(sh.capacity == GROW_STEP for sh in (again.index.shards if multi else [again.index]))
    for q in qs:
        assert _shape(again.query(q, 10, alpha=0.5)) == _shape(small.query(q, 10, alpha=0.5))

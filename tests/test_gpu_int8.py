"""int8 shards (AUR_I8) on the GPU.

The strongest check is the bf16 twin: a bf16 shard fed the int8 rows read back from the int8 shard (exact in bf16)
holds the same vectors up to a per-row scale, which cosine ignores, so every answer of every entry point must equal the
twin's bit for bit, ids and scores.  Besides that: the stored bytes equal oracle/quantize.py, searches equal the fp64
oracle over the int8 rows, and the knowledge base with dtype="int8" equals host fusion of the oracle legs."""

from __future__ import annotations

import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25
from aurora_b200.engine import DeviceBuffer, Index, KeywordIndex, hybrid_search, to_bf16_bits
from aurora_b200.filters import compile_program
from oracle import cosine_topk as O
from oracle import quantize as Qz
from tests.gpu_exact import check_exact, check_host_exact, dev_search
from tests.keyword_mirror import zipf_docs, zipf_queries

pytestmark = pytest.mark.gpu


def _bits(rng, n, d, scale=None):
    x = rng.standard_normal((n, d)).astype(np.float32)
    if scale is not None:
        x *= scale
    return to_bf16_bits(x)


def _f(bits):
    return Qz.bf16_bits_to_f64(bits).astype(np.float32)


def _pair(bits, ids, d, user=None, org=None, extra=64):
    """(int8 shard, its bf16 twin fed the int8 rows read back, the int8 rows)."""
    cap = bits.shape[0] + extra
    ix = Index(d, cap, dtype="int8")
    ix.add(bits, ids, user, org)
    q8, rid = ix.read_rows(0, bits.shape[0])
    assert np.array_equal(rid, ids)
    tw = Index(d, cap)
    tw.add(Qz.int8_to_bf16_bits(q8), ids, user, org)
    return ix, tw, q8


def _same(a, b, ctx=""):
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert np.array_equal(x.view(np.uint8) if x.dtype.kind == "f" else x, y.view(np.uint8) if y.dtype.kind == "f" else y), ctx
        else:
            assert x == y, ctx


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(11)
    n, d = 20_000, 768
    bits = _bits(rng, n, d, rng.uniform(0.01, 10.0, (n, 1)).astype(np.float32))
    ids = rng.permutation(n).astype(np.int64) * 3 + 5
    user = rng.integers(0, 20, n).astype(np.int32)
    org = np.where(rng.random(n) < 0.5, rng.integers(0, 4, n), -1).astype(np.int32)
    ix, tw, q8 = _pair(bits, ids, d, user, org)
    yield rng, bits, ids, user, org, ix, tw, q8
    ix.close(); tw.close()


# ------------------------------------------------------------------------------------------------ ingest
def test_ingest_bytes_match_the_oracle(corpus):
    _, bits, _, _, _, ix, _, q8 = corpus
    want, fin = Qz.quantize_rows(bits)
    assert fin.all()
    assert np.array_equal(q8, want)
    rows, _, _, _, live = ix.export()
    assert rows.dtype == np.int8 and np.array_equal(rows, want) and live.all()
    st = ix.stats()
    assert st["dtype"] == N.AUR_I8


@pytest.mark.parametrize("d", [208, 256])      # the generic path; the tensor-core path (dim % 128 == 0)
def test_ingest_dev_and_edge_rows(d):
    rng = np.random.default_rng(2)
    n = 60
    bits = _bits(rng, n, d)
    bits[3] = 0                                          # zero row
    bits[4, 7] = 0x7FC0                                  # NaN
    bits[5, 0] = 0x7F80                                  # +inf
    bits[6, 9] = 0xFF80                                  # -inf
    bits[7, :] = 0x0001                                  # subnormals
    bits[8, 1] = 0x7F7F                                  # the largest finite bf16
    ids = np.arange(n, dtype=np.int64)
    want, fin = Qz.quantize_rows(bits)
    assert fin.tolist()[3:9] == [True, False, False, False, True, True]
    with Index(d, 200, dtype="int8") as ix, Index(d, 200) as bf:
        buf = DeviceBuffer(bits.nbytes).upload(bits)
        ix.add_dev(buf.ptr, n, ids)
        ix.add(bits, ids + 1000)
        got, _ = ix.read_rows(0, 2 * n)
        assert np.array_equal(got[:n], want) and np.array_equal(got[n:], want)
        _, _, _, _, live = ix.export()
        assert live.all()
        # a non-finite row is never returned, as in a bf16 shard fed the same rows; k covers every row
        bf.add(bits, ids)
        q = np.concatenate([bits[[10, 11, 12]], np.zeros((1, d), np.uint16)])
        kernels = (N.KERNEL_AUTO, N.KERNEL_SIMT) + ((N.KERNEL_TC1, N.KERNEL_TC2) if d % 128 == 0 else ())
        for kern in kernels:
            ix.set_kernel(kern)
            i8_ids, i8_sc = ix.search(q, 128)
            b_ids, _ = bf.search(q, 128)
            for bad in (4, 5, 6, 1004, 1005, 1006):
                assert bad not in i8_ids
            for bad in (4, 5, 6):
                assert bad not in b_ids
            assert (i8_ids[:, :2 * n - 6] >= 0).all() and (i8_ids[:, 2 * n - 6:] == -1).all()
            assert (i8_sc[3, :2 * n - 6] == 0).all()          # the zero query scores 0 against every row
            sub = ix.search_subset(q, 128, np.array([4, 5, 10, 1006], np.int64))[0]
            assert set(sub[0][sub[0] >= 0].tolist()) == {10}


# ------------------------------------------------------------------------------------------------ the bf16 twin
@pytest.mark.parametrize("nq,k", [(1, 1), (63, 32), (65, 33), (257, 100), (64, 128), (1024, 32)])
def test_twin_search(corpus, nq, k):
    rng, _, _, _, _, ix, tw, _ = corpus
    q = _bits(rng, nq, 768)
    _same(ix.search(q, k), tw.search(q, k))
    _same(ix.search_snapshot(q, k), tw.search_snapshot(q, k))
    _same(dev_search(ix, q, k), dev_search(tw, q, k))


def test_twin_scoped_subset_lists_filtered(corpus):
    rng, _, ids, user, org, ix, tw, _ = corpus
    nq, k = 40, 32
    q = _bits(rng, nq, 768)
    qu = rng.integers(0, 20, nq).astype(np.int32)
    qo = rng.integers(-1, 4, nq).astype(np.int32)
    _same(ix.search(q, k, qu[:1].repeat(nq), qo[:1].repeat(nq)), tw.search(q, k, qu[:1].repeat(nq), qo[:1].repeat(nq)))
    _same(ix.search(q, k, qu, qo), tw.search(q, k, qu, qo))
    allow = rng.choice(ids, 3000, replace=False)
    _same(ix.search_subset(q, k, allow), tw.search_subset(q, k, allow))
    lists = [rng.choice(ids, m, replace=False) for m in (5, 200, 5000)]
    ql = rng.integers(0, 3, nq).astype(np.int32)
    _same(ix.search_lists(q, k, lists, ql), tw.search_lists(q, k, lists, ql))
    progs = [compile_program(None, {}, tenant=(int(u), int(o))) for u, o in ((1, 2), (3, -1), (7, 0))]
    qp = rng.integers(0, 3, nq).astype(np.int32)
    for mlr in (0, 1 << 30):
        _same(ix.search_filtered(q, k, progs, qp, max_list_rows=mlr), tw.search_filtered(q, k, progs, qp, max_list_rows=mlr))
    _same(ix.search_filtered(q, k, progs[:1], None, max_list_rows=0), tw.search_filtered(q, k, progs[:1], None, max_list_rows=0))
    assert np.array_equal(ix.filter_ids(progs[0]), tw.filter_ids(progs[0]))


def test_twin_hybrid(corpus):
    rng, _, ids, user, org, ix, tw, _ = corpus
    n = ids.shape[0]
    t, f, off = zipf_docs(np.random.default_rng(4), n, vocab=3000)
    kw = KeywordIndex(n * 2)
    try:
        kw.add(ids, t, f, off, user, org)
        nq = 24
        q = _bits(rng, nq, 768)
        qt, qo_ = zipf_queries(np.random.default_rng(5), nq, vocab=3000)
        for fusion in (N.FUSION_RANKED, N.FUSION_RELATIVE_SCORE):
            a = hybrid_search(ix, kw, q, 32, qt, qo_, 0.5, None, fusion, 40)
            b = hybrid_search(tw, kw, q, 32, qt, qo_, 0.5, None, fusion, 40)
            _same(a[:3], b[:3], fusion)
        progs = [compile_program(None, {}, tenant=(int(u), -1)) for u in (1, 2)]
        qp = (np.arange(nq) % 2).astype(np.int32)
        for mlr in (0, 1 << 30):
            a = hybrid_search(ix, kw, q, 32, qt, qo_, 0.5, programs=progs, q_program=qp, max_list_rows=mlr)
            b = hybrid_search(tw, kw, q, 32, qt, qo_, 0.5, programs=progs, q_program=qp, max_list_rows=mlr)
            _same(a[:3], b[:3], ("filtered", mlr))
    finally:
        kw.close()


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("d", [208, 384, 768, 1024])
@pytest.mark.parametrize("nq,k", [(1, 32), (65, 33), (257, 1), (64, 128)])
def test_oracle_grid(d, nq, k):
    rng = np.random.default_rng(d * 7 + nq + k)
    n = 6001
    bits = _bits(rng, n, d)
    ids = rng.permutation(n).astype(np.int64)
    with Index(d, n + 63, dtype="int8") as ix:
        ix.add(bits, ids)
        q8, _ = ix.read_rows(0, n)
        q = _bits(rng, nq, d)
        check_exact(dev_search(ix, q, k), _f(q), q8.astype(np.float32), k, ids=ids)
        check_host_exact(ix.search(q, k), _f(q), q8.astype(np.float32), k, ids=ids)


def test_mutations_compaction_and_capacity():
    rng = np.random.default_rng(9)
    d, cap = 384, 4100
    bits = _bits(rng, cap, d)
    with Index(d, cap, dtype="int8") as ix:
        ix.add(bits[:3000], np.arange(3000, dtype=np.int64))
        ix.remove(np.arange(0, 3000, 7))
        ix.add(bits[3000:3500], np.arange(100, 600, dtype=np.int64))      # upserts
        ix.add(bits[3500:cap], np.arange(5000, 5000 + cap - 3500, dtype=np.int64))   # exactly full
        with pytest.raises(RuntimeError):
            ix.add(bits[:1], np.array([99999], np.int64))
        q = _bits(rng, 70, d)

        def check():
            rows, rid, _, _, live = ix.export()
            check_host_exact(ix.search(q, 50), _f(q), rows.astype(np.float32), 50, ids=rid, live=live)

        check()
        before = ix.search(q, 50)
        assert ix.compact() > 0
        rows, _, _, _, live = ix.export()
        assert live.all()
        _same(ix.search(q, 50), before)
        check()


def test_adversarial_cut(corpus):
    rng = np.random.default_rng(21)
    d, k = 768, 32
    base = _bits(rng, 1, d)[0]
    bq, _ = Qz.quantize_rows(base[None])
    rows = [Qz.int8_to_bf16_bits(bq)[0]] * 20                 # an exact-duplicate group cut by k
    for j in range(60):                                       # rows one int8 step from it
        v = bq[0].astype(np.int16).copy()
        i = (j * 37) % d
        if abs(int(v[i])) < 127:
            v[i] += 1 if j % 2 else -1
        rows.append(Qz.int8_to_bf16_bits(v.astype(np.int8)[None])[0])
    noise = _bits(rng, 5000, d)
    allb = np.concatenate([np.stack(rows), noise])
    ids = rng.permutation(allb.shape[0]).astype(np.int64)
    ix, tw, q8 = _pair(allb, ids, d)
    try:
        dom = np.zeros((1, d), np.float32); dom[0, 3] = 1000.0; dom[0, 4:40] = 0.001
        q = np.concatenate([_f(base[None]), _f(base[None]) + 0.01 * rng.standard_normal((1, d)).astype(np.float32), dom,
                            np.zeros((1, d), np.float32)])
        qb = to_bf16_bits(q)
        for kern in (N.KERNEL_AUTO, N.KERNEL_SIMT):
            ix.set_kernel(kern)
            check_exact(dev_search(ix, qb, k), _f(qb), q8.astype(np.float32), k, ids=ids)
            _same(ix.search(qb, k), tw.search(qb, k))
    finally:
        ix.close(); tw.close()


def test_save_load_roundtrip(tmp_path):
    rng = np.random.default_rng(31)
    d = 256
    bits = _bits(rng, 3000, d)
    with Index(d, 4000, dtype="int8") as ix:
        ix.add(bits, np.arange(3000, dtype=np.int64))
        ix.remove(np.arange(0, 3000, 5))
        q = _bits(rng, 20, d)
        want = ix.search(q, 40)
        rows, rid, _, _, live = ix.export()
        ix.save(str(tmp_path / "s"))
    with Index.load(str(tmp_path / "s")) as ld:
        assert ld.dtype == N.AUR_I8
        r2, i2, _, _, l2 = ld.export()
        assert np.array_equal(r2, rows[live]) and np.array_equal(i2, rid[live]) and l2.all()
        _same(ld.search(q, 40), want)


def test_writer_under_readers():
    rng = np.random.default_rng(41)
    d, n, per = 256, 12_000, 500
    bits = _bits(rng, n, d)
    ids = np.arange(n, dtype=np.int64)
    q = _bits(rng, 8, d)
    q8_all, _ = Qz.quantize_rows(bits)
    with Index(d, n + 64, dtype="int8") as ix:
        stop = threading.Event()
        answers, errors = [], []

        def reader():
            try:
                while not stop.is_set():
                    answers.append(ix.search_snapshot(q, 16))
            except Exception as e:   # noqa: BLE001
                errors.append(e)

        th = [threading.Thread(target=reader) for _ in range(3)]
        for t in th:
            t.start()
        for s in range(0, n, per):
            ix.add(bits[s:s + per], ids[s:s + per])
        stop.set()
        for t in th:
            t.join()
        assert not errors
        for a_ids, a_sc, snap in answers[::max(1, len(answers) // 20)]:
            check_host_exact((a_ids, a_sc), _f(q), q8_all[:snap].astype(np.float32), 16, ids=ids[:snap])


# ------------------------------------------------------------------------------------------------ knowledge base
class _Int8Oracle:
    """CPU double of an int8 engine.Index: the rows are quantized as the shard does, then searched by the oracle."""

    def __new__(cls, dim, cap):
        from tests.doubles import OracleIndex

        class Q(OracleIndex):
            def add(self, rows, ids, user_codes=None, org_codes=None):
                q8, _ = Qz.quantize_rows(to_bf16_bits(np.asarray(rows, np.float32)))
                super().add(q8.astype(np.float32), ids, user_codes, org_codes)

        return Q(dim, cap)


def test_knowledge_base_int8(monkeypatch):
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder

    emb = HashEmbedder(64)
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    dev = R.KnowledgeBase(emb, capacity=4096, dtype="int8")
    host = R.KnowledgeBase(emb, capacity=4096, index_factory=_Int8Oracle)
    assert dev.index.dtype == N.AUR_I8 and dev._hybrid_device
    docs = ["disk full on node", "memory leak in worker", "network partition between zones", "cpu throttling alert",
            "database failover happened", "certificate expired on gateway"]
    for kb in (dev, host):
        for rep in range(25):
            for j, t in enumerate(docs):
                kb.insert(f"u{j % 3}", f"doc{j}", "f.md", [{"content": f"{t} #{rep % 5}", "chunk_index": rep}],
                          org_id="o1" if j % 2 else None)
    for qtext in ("disk node", "leak worker memory", "gateway certificate"):
        for alpha in (0.0, 0.5, 0.999):
            a = [(o.uuid, o.metadata.score) for o in dev.query(qtext, 10, alpha=alpha)]
            b = [(o.uuid, o.metadata.score) for o in host.query(qtext, 10, alpha=alpha)]
            assert a == b, (qtext, alpha)
            a = [(o.uuid, o.metadata.score) for o in dev.query(qtext, 8, user_id="u1", org_id="o1", alpha=alpha, scoped=True)]
            b = [(o.uuid, o.metadata.score) for o in host.query(qtext, 8, user_id="u1", org_id="o1", alpha=alpha, scoped=True)]
            assert a == b, (qtext, alpha, "scoped")


# ------------------------------------------------------------------------------------------------ the tensor-core path
@pytest.mark.parametrize("kern", [N.KERNEL_TC1, N.KERNEL_TC2, N.KERNEL_SIMT])
@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("d", [384, 1024])
def test_tc_kernels_and_tiles(kern, tile, d):
    """Every kernel and tile width over an int8 shard whose last tile is partial, against the oracle over the int8 rows
    and against the bf16 twin; the tensor-core launches must really be the int8 ones (aur_stats)."""
    rng = np.random.default_rng(d + tile + kern)
    n = 9_000 + 37
    bits = _bits(rng, n, d)
    ids = rng.permutation(n).astype(np.int64) * 2 + 1
    ix, tw, q8 = _pair(bits, ids, d, extra=27)
    try:
        for x in (ix, tw):
            N.check(x._lib.aur_set_option(x._h, b"tc_tile", tile))
            x.set_kernel(kern)
        for nq, k in ((1, 1), (65, 33), (257, 100)):
            q = _bits(rng, nq, d)
            try:
                got = dev_search(ix, q, k)
            except N.AuroraError as e:   # a k the forced tile's layout cannot hold: refused exactly as for bf16 rows
                assert e.code == -4, e
                with pytest.raises(N.AuroraError, match="k too large"):
                    tw.search(q, k)
                assert "k too large" in str(e)
                continue
            assert ix.stats()["last_kernel"] == kern
            if kern != N.KERNEL_SIMT:
                assert ix.stats()["last_tile_n"] == tile
            check_exact(got, _f(q), q8.astype(np.float32), k, ids=ids)
            _same(ix.search(q, k), tw.search(q, k), (kern, tile, nq, k))
    finally:
        ix.close(); tw.close()


def test_scope_paths(corpus):
    """One scope (row scale), 2..32 scopes (per-row bit masks on the tensor-core kernel) and more than 32 (generic)."""
    rng, _, _, user, org, ix, tw, q8 = corpus
    nq, k = 128, 32
    q = _bits(rng, nq, 768)
    for n_scopes, kern_want in ((1, None), (5, N.KERNEL_TC2), (32, N.KERNEL_TC2), (40, N.KERNEL_SIMT)):
        su = (np.arange(n_scopes) % 20).astype(np.int32)            # distinct (user, org) scopes
        so = (np.arange(n_scopes) // 20 - 1).astype(np.int32)
        pick = np.arange(nq) % n_scopes
        qu, qo = su[pick], so[pick]
        got = ix.search(q, k, qu, qo)
        if kern_want is not None:
            assert ix.stats()["last_kernel"] == kern_want, n_scopes
        _same(got, tw.search(q, k, qu, qo), n_scopes)
        for i in range(0, nq, 37):
            vis = (user == qu[i]) | ((qo[i] >= 0) & (org == qo[i]))
            check_host_exact((got[0][i:i + 1], got[1][i:i + 1]), _f(q[i:i + 1]), q8.astype(np.float32), k,
                             ids=corpus[2], live=vis)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_twin_hybrid_multi(n):
    from aurora_b200.engine import MultiIndex, MultiKeywordIndex

    gpus = N.load().aur_device_count()
    devices = [s % gpus for s in range(n)]
    rng = np.random.default_rng(50 + n)
    rows, d = 6000, 256
    bits = _bits(rng, rows, d)
    ids = rng.permutation(rows).astype(np.int64) * 7 + 3
    t, f, off = zipf_docs(rng, rows, vocab=2000)
    mi = MultiIndex(d, rows * 2, devices=devices, dtype="int8")
    mi.add(bits, ids)
    q8 = np.zeros((rows, d), np.int8)
    for sh in mi.shards:
        r8, rid, _, _, _ = sh.export()
        q8[np.searchsorted(np.sort(ids), rid)] = r8
    order = np.sort(ids)
    tw = MultiIndex(d, rows * 2, devices=devices)
    tw.add(Qz.int8_to_bf16_bits(q8), order)
    mk = MultiKeywordIndex(rows * 2, devices=devices)
    mk.add(ids, t, f, off)
    try:
        nq = 20
        q = _bits(rng, nq, d)
        qt, qo_ = zipf_queries(rng, nq, vocab=2000)
        for fusion in (N.FUSION_RANKED, N.FUSION_RELATIVE_SCORE):
            a = hybrid_search(mi, mk, q, 32, qt, qo_, 0.5, None, fusion, 40)
            b = hybrid_search(tw, mk, q, 32, qt, qo_, 0.5, None, fusion, 40)
            _same(a[:3], b[:3], (n, fusion))
        progs = [compile_program(None, {}, tenant=(0, -1))]
        a = hybrid_search(mi, mk, q, 32, qt, qo_, 0.5, programs=progs)
        b = hybrid_search(tw, mk, q, 32, qt, qo_, 0.5, programs=progs)
        _same(a[:3], b[:3], (n, "filtered"))
        want = O.cosine_topk(_f(q), q8.astype(np.float32), 32, ids=order)[0]
        assert np.array_equal(mi.search(q, 32)[0], want)
    finally:
        mi.close(); tw.close(); mk.close()


def test_encoder_append_into_int8():
    from aurora_b200.encoder import Encoder, EncoderConfig
    from oracle import bert_encoder as B

    cfg_o = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")
    cfg = EncoderConfig(hidden=cfg_o.hidden, layers=cfg_o.layers, heads=cfg_o.heads, inter=cfg_o.inter, vocab=cfg_o.vocab,
                        max_pos=cfg_o.max_pos, type_vocab=cfg_o.type_vocab, ln_eps=cfg_o.ln_eps, pool=cfg_o.pool,
                        normalize=cfg_o.normalize)
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 7, 12, mean_len=60, std_len=40, min_len=1, max_len=200)
    with Encoder(cfg, max_tokens=4096, max_seqs=16) as enc, Index(128, 64, dtype="int8") as ix:
        enc.load_weights(w)
        out = enc.encode_packed(tok, cu, bf16=True)
        enc.encode_append(ix, tok, cu, np.arange(len(cu) - 1, dtype=np.int64))
        got, _ = ix.read_rows(0, len(cu) - 1)
        want, fin = Qz.quantize_rows(out)
        assert fin.all() and np.array_equal(got, want)


def test_save_load_keeps_non_finite_rows_invisible(tmp_path):
    from aurora_b200.engine import MultiIndex

    rng = np.random.default_rng(61)
    d = 256
    bits = _bits(rng, 200, d)
    bits[5, 3] = 0x7FC0
    bits[9, 0] = 0x7F80
    ids = np.arange(200, dtype=np.int64)
    q = np.concatenate([bits[[1, 2]], np.zeros((1, d), np.uint16)])
    with Index(d, 256, dtype="int8") as ix:
        ix.add(bits, ids)
        want = ix.search(q, 128)
        assert 5 not in want[0] and 9 not in want[0]
        ix.save(str(tmp_path / "a"))
        with Index.load(str(tmp_path / "a")) as ld:
            assert np.array_equal(ld.export_raw()[4], ix.export_raw()[4])
            assert (ld.export_raw()[4][[5, 9]] == 2).all()
            _same(ld.search(q, 128), want)
    mi = MultiIndex(d, 512, devices=[0, 0], dtype="int8")
    mi.add(bits, ids)
    want = mi.search(q, 128)
    mi.save(str(tmp_path / "m"))
    m2 = MultiIndex.load(str(tmp_path / "m"), devices=[0, 0])
    try:
        _same(m2.search(q, 128), want)
        assert 5 not in want[0] and 9 not in want[0]
    finally:
        mi.close(); m2.close()


def test_knowledge_base_int8_batch_and_snapshot(monkeypatch, tmp_path):
    from aurora_b200 import retriever as R
    from tests.doubles import HashEmbedder

    emb = HashEmbedder(128)
    monkeypatch.setattr(bm25, "VECTORISE_FROM", 1 << 60)
    dev = R.KnowledgeBase(emb, capacity=4096, dtype="int8")
    host = R.KnowledgeBase(emb, capacity=4096, index_factory=_Int8Oracle)
    docs = ["disk full on node", "memory leak in worker", "network partition between zones", "cpu throttling alert"]
    for kb in (dev, host):
        for rep in range(20):
            for j, t in enumerate(docs):
                kb.insert(f"u{j % 2}", f"doc{j}", "f.md", [{"content": f"{t} #{rep % 5}", "chunk_index": rep}],
                          org_id="o1" if j % 2 else None)
    reqs = [("u1", "disk node", 6, 0.5, None), ("u0", "leak worker", 4, None, "o1"), ("u1", "cpu alert", 5, 0.0, None)]
    shape = lambda res: [[(o.uuid, o.metadata.score) for o in r] for r in res]   # noqa: E731
    assert shape(dev.query_batch(reqs)) == shape(host.query_batch(reqs))
    dev.save(str(tmp_path / "kb"))
    ld = R.KnowledgeBase.load(str(tmp_path / "kb"), emb, capacity=4096)
    assert ld.index.dtype == N.AUR_I8
    assert np.array_equal(ld.index.export()[0], dev.index.export()[0][dev.index.export()[4]])
    assert shape(ld.query_batch(reqs)) == shape(dev.query_batch(reqs))

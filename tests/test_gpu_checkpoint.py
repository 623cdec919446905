"""aur_live_bits / aur_export_rows and KnowledgeBase.checkpoint over CUDA shards: the bitmaps equal aur_export's live
flags, the row ranges equal its slices, the compaction count moves only on aur_compact, a held write phase blocks no
search or append, and a restore from a base plus deltas answers bit for bit like a restore from a full save."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import checkpoint as K
from aurora_b200 import retriever as R
from aurora_b200.engine import Index, MultiIndex
from aurora_b200.filters import Filter
from tests.doubles import HashEmbedder

pytestmark = pytest.mark.gpu

DTYPES = [("bf16", 768), ("int8", 768), ("f32", 96)]


def _rows(rng, n, dim):
    return rng.standard_normal((n, dim)).astype(np.float32)


def _assert_capture_matches_export(ix):
    rows, live, nonfinite, _ = ix.capture()
    e_rows, e_ids, e_user, e_org, e_live = ix.export_raw()
    assert rows == len(e_ids)
    assert len(live) == (rows + 31) // 32 and len(nonfinite) == len(live)
    assert np.array_equal(K.unpack_bits(live, rows), e_live > 0)
    assert np.array_equal(K.unpack_bits(nonfinite, rows), e_live == 2)
    if rows % 32:                                 # bits past the rows are clear
        assert live[-1] >> (rows % 32) == 0 and nonfinite[-1] >> (rows % 32) == 0
    for r0, n in ((0, rows), (rows // 3, rows // 2), (rows - 1 if rows else 0, min(rows, 1)), (rows, 0)):
        got = ix.export_rows(r0, n)
        for g, want in zip(got, (e_rows, e_ids, e_user, e_org)):
            assert np.array_equal(g, want[r0:r0 + n])


@pytest.mark.parametrize("dtype,dim", DTYPES)
def test_live_bits_and_export_rows_match_export(dtype, dim):
    rng = np.random.default_rng(1)
    with Index(dim, 1000, dtype=dtype) as ix:
        _assert_capture_matches_export(ix)                                # 0 rows
        x = _rows(rng, 77, dim)
        if dtype == "int8":                                               # rows stored from a NaN / inf: live = 2
            x[5, 3], x[40, 0], x[41, 7] = np.nan, np.inf, -np.inf
        ix.add(x, np.arange(77), rng.integers(5, size=77).astype(np.int32), rng.integers(-1, 3, size=77).astype(np.int32))
        _assert_capture_matches_export(ix)                                # not a multiple of 32
        ix.remove(np.array([0, 31, 32, 63, 76]))                          # tombstones on word edges
        ix.add(_rows(rng, 40, dim), np.arange(50, 90))                     # upserts
        _assert_capture_matches_export(ix)
        ix.reserve(150_000)                                               # grown in place
        ix.add(_rows(rng, 120_000, dim), np.arange(1000, 121_000))
        ix.remove(np.arange(1000, 121_000, 7))
        _assert_capture_matches_export(ix)
        if dtype == "int8":
            assert ix.export_raw()[4][[5, 40, 41]].tolist() == [2, 2, 2]


def test_too_few_words_and_ranges_outside_the_prefix_are_rejected():
    rng = np.random.default_rng(2)
    with Index(768, 1000) as ix:
        ix.add(_rows(rng, 65, 768), np.arange(65))
        lib = ix._lib
        live = np.full(8, 0xDEADBEEF, np.uint32)
        rows, comp = C.c_int64(-7), C.c_int64(-7)
        rc = lib.aur_live_bits(ix._h, live.ctypes.data_as(C.c_void_p), None, 2, C.byref(rows), C.byref(comp))
        assert rc == N.AUR_ERR_INVALID and rows.value == -7 and np.all(live == 0xDEADBEEF)   # nothing written
        rc = lib.aur_live_bits(ix._h, live.ctypes.data_as(C.c_void_p), None, 3, C.byref(rows), C.byref(comp))
        assert rc == N.AUR_OK and rows.value == 65 and comp.value == 0 and np.all(live[3:] == 0xDEADBEEF)
        for r0, n in ((-1, 2), (60, 6), (66, 0), (0, -1)):
            with pytest.raises(N.AuroraError):
                ix.export_rows(r0, n) if n >= 0 else N.check(lib.aur_export_rows(ix._h, r0, n, None, None, None, None))
    with Index(768, 64, dtype="int8") as i8:
        rows = C.c_int64(0)
        assert i8._lib.aur_live_bits(i8._h, live.ctypes.data_as(C.c_void_p), None, 8, C.byref(rows), None) == N.AUR_ERR_INVALID


def test_compaction_counter_moves_only_on_compact():
    rng = np.random.default_rng(3)
    with Index(768, 4096) as ix:
        ix.add(_rows(rng, 100, 768), np.arange(100))
        assert ix.capture()[3] == 0
        ix.remove(np.arange(10))
        ix.add(_rows(rng, 10, 768), np.arange(20, 30))
        ix.reserve(70_000)
        ix.search(_rows(rng, 3, 768), 5)
        ix.export_raw()
        assert ix.capture()[3] == 0
        assert ix.compact() == 20
        assert ix.capture()[3] == 1
        ix.compact()                                                      # nothing to reclaim: still a call
        assert ix.capture()[3] == 2
        _assert_capture_matches_export(ix)


def _kb_cuda(kind, devices=(0, 0)):
    emb = HashEmbedder(768)
    if kind == "index":
        fac = lambda dim, cap: Index(dim, cap)                               # noqa: E731
    else:
        fac = lambda dim, cap: MultiIndex(dim, cap, devices=list(devices))   # noqa: E731
    return R.KnowledgeBase(emb, capacity=2048, index_factory=fac), emb


def _loader(kind, devices=(0, 0)):
    if kind == "index":
        return lambda p, cap: Index.load(p, capacity=cap)
    return lambda p, cap: MultiIndex.load(p, capacity=cap, devices=list(devices))


def _chunks(tag, n):
    return [{"content": f"{tag} item{i} redis kafka alpha{i % 7} beta{i % 3}", "heading_context": f"h{i % 4}",
             "chunk_index": i} for i in range(n)]


QUERIES = ["redis alpha1", "kafka beta2 item3", "h2 item10 alpha5", "nothing matches zz"]


def _answers(kb):
    out = []
    for q in QUERIES:
        for alpha in (None, 0.5, 0.0):
            for scope in ({}, {"user_id": "u1", "scoped": True}, {"user_id": "u2", "org_id": "o2"}):
                out.append([(o.uuid, o.metadata.score, o.metadata.distance) for o in kb.query(q, 8, alpha=alpha, **scope)])
        f = Filter.by_property("document_id").equal("d2") | Filter.by_property("chunk_index").less_than(5)
        for alpha in (None, 0.5):
            out.append([(o.uuid, o.metadata.score, o.metadata.distance) for o in kb.query(q, 8, alpha=alpha, filters=f)])
    return out


def _live(index):
    out = {}
    for p in (getattr(index, "shards", None) or [index]):
        rows, ids, user, org, live = p.export_raw()
        for i in np.nonzero(live)[0]:
            out[int(ids[i])] = (rows[i].tobytes(), int(user[i]), int(org[i]), int(live[i]))
    return out


def _same(a, b):
    assert a._props == b._props and a._key2id == b._key2id and a._next_id == b._next_id and a.mutations == b.mutations
    assert _live(a.index) == _live(b.index)
    assert _answers(a) == _answers(b)


@pytest.mark.parametrize("kind", ["index", "multi"])
def test_restore_from_base_and_deltas_answers_like_a_full_save(tmp_path, kind):
    kb, emb = _kb_cuda(kind)
    d = str(tmp_path / "ckpt")
    kb.insert("u1", "d1", "a.md", _chunks("one", 300))
    kb.insert("u2", "d2", "b.md", _chunks("two", 200), org_id="o2")
    assert kb.checkpoint(d)["kind"] == "base"
    kb.insert("u1", "d1", "a.md", _chunks("one again", 30))                 # upserts of base rows
    kb.insert("u3", "d3", "c.md", _chunks("three", 40), org_id="o2")
    assert kb.checkpoint(d)["kind"] == "delta"
    kb.delete_where(Filter.by_property("document_id").equal("d3") & Filter.by_property("chunk_index").less_than(20))
    kb.delete_where(lambda p: p["document_id"] == "d2" and p["chunk_index"] % 9 == 0)
    assert kb.checkpoint(d)["kind"] == "delta"
    assert kb.checkpoint(d)["kind"] == "delta"                              # empty
    full = str(tmp_path / "full")
    kb.save(full)
    layouts = [(0,)] if kind == "index" else [(0,), (0, 0)]
    for devs in layouts:
        a = R.KnowledgeBase.load(d, emb, capacity=2048, index_loader=_loader(kind, devs))
        b = R.KnowledgeBase.load(full, emb, capacity=2048, index_loader=_loader(kind, devs))
        _same(a, b)
    kb.index.compact()
    kb.insert("u4", "d4", "e.md", _chunks("four", 10))
    assert kb.checkpoint(d)["kind"] == "base"
    kb.save(full)
    _same(R.KnowledgeBase.load(d, emb, capacity=2048, index_loader=_loader(kind)),
          R.KnowledgeBase.load(full, emb, capacity=2048, index_loader=_loader(kind)))


def test_a_held_write_phase_blocks_no_search_or_append(tmp_path):
    rng = np.random.default_rng(5)
    kb, _ = _kb_cuda("index")
    kb.insert("u1", "d1", "a.md", _chunks("one", 500))
    d = str(tmp_path / "ckpt")
    for stage in ("captured", "segment"):
        reached, release = threading.Event(), threading.Event()

        def hook(s, stage=stage):
            if s == stage:
                reached.set()
                assert release.wait(60)
        t = threading.Thread(target=kb.checkpoint, args=(d,), kwargs={"on_stage": hook})
        t.start()
        assert reached.wait(60)
        done = threading.Event()

        def other():
            ix = kb.index
            ix.search(_rows(rng, 4, 768), 10)                                  # aur_search on the same shard
            n = ix.stats()["rows"]
            ix.add(_rows(rng, 8, 768), np.arange(10_000 + n, 10_008 + n))    # aur_add
            assert kb.query("one item3", 2)
            done.set()
        o = threading.Thread(target=other)
        o.start()
        ok = done.wait(60)
        release.set()
        t.join(60)
        o.join(60)
        assert ok, f"a search or an append waited for the checkpoint's write phase ({stage})"


def test_export_rows_runs_beside_appends_and_searches():
    """aur_export_rows of a large range while other threads append and search the shard: every call answers, and the
    exported rows equal aur_export's."""
    rng = np.random.default_rng(6)
    with Index(768, 300_000) as ix:
        ix.add(_rows(rng, 200_000, 768), np.arange(200_000))
        stop = threading.Event()
        errs = []

        def writer():
            i = 0
            while not stop.is_set() and i < 50:
                ix.add(_rows(rng, 256, 768), np.arange(1_000_000 + 256 * i, 1_000_000 + 256 * (i + 1)))
                ix.search(_rows(rng, 2, 768), 8)
                i += 1
        w = threading.Thread(target=writer)
        w.start()
        try:
            got = ix.export_rows(0, 200_000)
        except Exception as e:      # pragma: no cover
            errs.append(e)
        stop.set()
        w.join(60)
        assert not errs
        e_rows, e_ids, e_user, e_org, _ = ix.export_raw()
        for g, want in zip(got, (e_rows, e_ids, e_user, e_org)):
            assert np.array_equal(g, want[:200_000])

"""KnowledgeBase.checkpoint on the CPU: a restore from a base plus deltas equals a restore from a full save, the write
phase runs outside the lock, and every crash point keeps what was acknowledged (CPU doubles)."""

import json
import os
import shutil
import threading

import numpy as np
import pytest

from aurora_b200 import checkpoint as K
from aurora_b200 import retriever as R
from aurora_b200.engine import MultiIndex
from aurora_b200.filters import Filter
from tests.doubles import HashEmbedder, OracleIndex


class CaptureIndex(OracleIndex):
    """OracleIndex with the shard's checkpoint surface: capture() as aur_live_bits gives it, export_rows() as
    aur_export_rows, and a compaction counter bumped by compact()."""

    def __init__(self, dim, capacity):
        super().__init__(dim, capacity)
        self.compactions = 0

    def capture(self):
        return len(self.ids), K.pack_bits(self.live), K.pack_bits(np.zeros(len(self.ids), bool)), self.compactions

    def export_rows(self, row0, n):
        sl = slice(row0, row0 + n)
        if row0 < 0 or n < 0 or row0 + n > len(self.ids):
            raise ValueError("outside the published prefix")
        return self.rows[sl], self.ids[sl], self.user[sl], self.org[sl]

    def compact(self):
        self.compactions += 1
        return super().compact()


DIM = 64
EMB = HashEmbedder(DIM)
KINDS = ["export", "capture", "multi2"]


def _factory(kind):
    if kind == "export":
        return lambda dim, cap: OracleIndex(dim, cap)
    if kind == "capture":
        return lambda dim, cap: CaptureIndex(dim, cap)
    return lambda dim, cap: MultiIndex(dim, cap, devices=[0, 1], shard_factory=lambda d, c, dev: CaptureIndex(d, c))


def _loader(kind, n_devices=2):
    if kind == "export":
        return lambda p, cap: OracleIndex.load(p, cap)
    if kind == "capture":
        return lambda p, cap: CaptureIndex.load(p, cap)
    return lambda p, cap: MultiIndex.load(p, cap, devices=list(range(n_devices)),
                                          shard_factory=lambda d, c, dev: CaptureIndex(d, c))


def _kb(kind):
    return R.KnowledgeBase(EMB, capacity=4096, index_factory=_factory(kind))


def _chunks(tag, n):
    return [{"content": f"{tag} item{i} runbook entry alpha{i % 5}", "heading_context": f"h{i % 3}", "chunk_index": i}
            for i in range(n)]


def _live_rows(index):
    parts = getattr(index, "shards", None) or [index]
    out = {}
    for p in parts:
        rows, ids, user, org, live = p.export()
        for i in np.nonzero(np.asarray(live))[0]:
            assert int(ids[i]) not in out
            out[int(ids[i])] = (np.asarray(rows[i]).tobytes(), int(user[i]), int(org[i]))
    return out


QUERIES = ["alpha1 runbook", "item3 entry", "redis failover alpha2", "h1 item0"]


def _answers(kb):
    out = []
    for q in QUERIES:
        for alpha in (None, 0.5):
            out.append([(o.uuid, o.metadata.score) for o in kb.query(q, 6, alpha=alpha)])
            out.append([(o.uuid, o.metadata.score) for o in kb.query(q, 4, alpha=alpha, user_id="u1", scoped=True)])
        f = Filter.by_property("document_id").equal("d2")
        out.append([(o.uuid, o.metadata.score) for o in kb.query(q, 5, filters=f)])
    return out


def _state(kb):
    return (kb._props, kb._key2id, kb._user_code, kb._org_code, kb._next_id, kb.mutations, _live_rows(kb.index),
            _answers(kb))


def _assert_same(a, b):
    sa, sb = _state(a), _state(b)
    for x, y, name in zip(sa, sb, ("props", "keys", "user codes", "org codes", "next_id", "generation", "live rows",
                                   "answers")):
        assert x == y, name


def _restore(directory, kind, n_devices=2):
    return R.KnowledgeBase.load(directory, EMB, capacity=4096, index_loader=_loader(kind, n_devices))


def _check(kb, ckpt_dir, tmp_path, kind, step):
    ref_dir = str(tmp_path / f"full{step}")
    kb.save(ref_dir)
    want = _restore(ref_dir, kind)
    _assert_same(_restore(ckpt_dir, kind), want)
    if kind == "multi2":                # restored onto another number of devices: rows placed by id mod n
        for n in (1, 3):
            _assert_same(_restore(ckpt_dir, kind, n), want)
    names = os.listdir(ckpt_dir)
    meta = json.load(open(os.path.join(ckpt_dir, "meta.json")))
    assert [n for n in names if n.startswith("shard.")] == [meta["shard"]]
    assert sorted(n for n in names if n.startswith(K.PREFIXES)) == sorted(K.referenced(meta))


@pytest.mark.parametrize("kind", KINDS)
def test_base_plus_deltas_restores_like_a_full_save(tmp_path, kind):
    kb = _kb(kind)
    d = str(tmp_path / "ckpt")
    kb.insert("u1", "d1", "a.md", _chunks("first", 40))
    kb.insert("u2", "d2", "b.md", _chunks("second", 30), org_id="o2")
    r = kb.checkpoint(d)
    assert r["kind"] == "base" and r["bytes"] > 0 and r["locked_ms"] >= 0
    _check(kb, d, tmp_path, kind, 0)

    kb.insert("u1", "d1", "a.md", _chunks("first revised", 5))          # upserts of rows in the base
    kb.insert("u3", "d3", "c.md", _chunks("third", 6), org_id="o3")
    assert kb.checkpoint(d)["kind"] == "delta"
    _check(kb, d, tmp_path, kind, 1)

    kb.delete_where(Filter.by_property("document_id").equal("d3"))      # rows of the previous delta
    kb.delete_where(lambda p: p["document_id"] == "d2" and p["chunk_index"] < 4)   # rows of the base
    kb.insert("u1", "d1", "a.md", _chunks("first revised twice", 2))    # an upsert of an upserted row
    assert kb.checkpoint(d)["kind"] == "delta"
    _check(kb, d, tmp_path, kind, 2)

    r = kb.checkpoint(d)                                                 # nothing changed: an empty delta
    assert r["kind"] == "delta"
    _check(kb, d, tmp_path, kind, 3)

    assert kb.index.compact() > 0
    kb.insert("u4", "d4", "e.md", _chunks("fourth", 3))
    assert kb.checkpoint(d)["kind"] == "base"                            # renumbered rows: a new base
    _check(kb, d, tmp_path, kind, 4)
    kb.delete_where(lambda p: p["document_id"] == "d4")
    assert kb.checkpoint(d)["kind"] == "delta"
    _check(kb, d, tmp_path, kind, 5)


def test_compaction_alone_forces_a_base(tmp_path):
    kb = _kb("capture")
    d = str(tmp_path / "ckpt")
    kb.insert("u1", "d1", "a.md", _chunks("x", 10))
    kb.checkpoint(d)
    kb.delete_where(lambda p: p["chunk_index"] < 3)
    kb.index.compact()                   # no mutation, but every row after the first tombstone moved
    assert kb.checkpoint(d)["kind"] == "base"
    _check(kb, d, tmp_path, "capture", 0)


def test_base_rule_delta_share_and_segment_count(tmp_path):
    kb = _kb("capture")
    d = str(tmp_path / "ckpt")
    kb.insert("u1", "d1", "a.md", _chunks("x", 64))
    assert kb.checkpoint(d)["kind"] == "base"
    kinds = []
    for i in range(K.MAX_DELTAS + 1):
        kb.insert("u1", f"e{i}", "a.md", _chunks(f"y{i}", 1))
        kinds.append(kb.checkpoint(d)["kind"])
    assert kinds == ["delta"] * K.MAX_DELTAS + ["base"]                 # the 17th delta would make 17 on disk
    kb.insert("u1", "big", "a.md", _chunks("z", 20))                     # 20 rows: at most a quarter of the base's 81
    assert kb.checkpoint(d)["kind"] == "delta"
    kb.insert("u1", "big2", "a.md", _chunks("w", 1))                     # 21: more than a quarter
    assert kb.checkpoint(d)["kind"] == "base"
    _check(kb, d, tmp_path, "capture", 0)


def test_old_format_meta_still_loads_and_is_superseded(tmp_path):
    kb = _kb("export")
    d = str(tmp_path / "snap")
    kb.insert("u1", "d1", "a.md", _chunks("old", 12))
    kb.save(d)                                      # today's format: inline props
    assert "props" in json.load(open(os.path.join(d, "meta.json")))
    _assert_same(_restore(d, "export"), kb)
    kb2 = _restore(d, "export")
    kb2.insert("u2", "d2", "b.md", _chunks("new", 3))
    assert kb2.checkpoint(d)["kind"] == "base"      # a restored store starts with a base
    kb2.delete_where(lambda p: p["chunk_index"] == 1)
    assert kb2.checkpoint(d)["kind"] == "delta"
    _check(kb2, d, tmp_path, "export", 0)


def _held(stage_name):
    """on_stage hook that stops the write phase at stage_name until released."""
    reached, release = threading.Event(), threading.Event()

    def hook(stage):
        if stage == stage_name:
            reached.set()
            assert release.wait(30)
    return hook, reached, release


@pytest.mark.parametrize("kind", ["export", "capture"])
def test_mutations_during_the_write_phase_go_to_the_log_and_the_next_checkpoint(tmp_path, kind):
    d = str(tmp_path / "ckpt")
    kb = _kb(kind)
    log = os.path.join(d, "mutations.log")
    os.makedirs(d)
    kb.attach_wal(log)
    kb.insert("u1", "d1", "a.md", _chunks("base", 40))
    kb.checkpoint(d)
    kb.insert("u1", "d2", "b.md", _chunks("captured", 4))
    hook, reached, release = _held("captured")
    res = {}
    t = threading.Thread(target=lambda: res.update(kb.checkpoint(d, on_stage=hook)))
    t.start()
    assert reached.wait(30)
    gen = kb.mutations
    kb.insert("u2", "d3", "c.md", _chunks("during", 3))               # acknowledged during the write phase
    kb.delete_where(lambda p: p["document_id"] == "d1" and p["chunk_index"] == 0)
    release.set()
    t.join(30)
    assert res["kind"] == "delta" and res["generation"] == gen
    snap = _restore(d, kind)                                          # the segment: the state at capture
    assert snap.mutations == gen and snap.count_where(lambda p: p["document_id"] == "d3") == 0
    assert snap.count_where(lambda p: p["document_id"] == "d1") == 40
    recs = [json.loads(line) for line in open(log)]
    assert [r["gen"] for r in recs] == [gen, gen + 3]                 # the trimmed log: exactly the later records
    snap.attach_wal(log)
    _assert_same(snap, kb)
    assert kb.checkpoint(d)["kind"] == "delta"                         # ... and the next checkpoint has them
    _assert_same(_restore(d, kind), kb)


def test_queries_and_inserts_go_on_while_the_write_phase_is_held(tmp_path):
    kb = _kb("capture")
    d = str(tmp_path / "ckpt")
    kb.insert("u1", "d1", "a.md", _chunks("x", 20))
    for stage in ("captured", "segment"):
        hook, reached, release = _held(stage)
        t = threading.Thread(target=kb.checkpoint, args=(d,), kwargs={"on_stage": hook})
        t.start()
        assert reached.wait(30)
        done = threading.Event()

        def other():
            assert kb.query("x item1", 3)
            kb.insert("u9", f"during-{stage}", "z.md", _chunks(f"during{stage}", 2))
            assert kb.query(f"during{stage} item1", 1, user_id="u9", scoped=True)[0].properties["document_id"] == f"during-{stage}"
            done.set()
        o = threading.Thread(target=other)
        o.start()
        assert done.wait(30), "a query or an insert waited for the checkpoint's write phase"
        release.set()
        t.join(30)
        o.join(30)
    assert _restore(d, "capture").count_where(lambda p: p["document_id"] == "during-segment") == 0   # after its capture
    kb.checkpoint(d)
    _check(kb, d, tmp_path, "capture", 0)


class Crash(Exception):
    pass


@pytest.mark.parametrize("stage", ["segment", "manifest", "trim"])
@pytest.mark.parametrize("second", [False, True])
def test_a_crash_at_any_stage_loses_nothing_acknowledged(tmp_path, stage, second):
    """second: the crash hits a delta (after a base) instead of the first base."""
    d = str(tmp_path / "ckpt")
    os.makedirs(d)
    log = os.path.join(d, "mutations.log")
    kb = _kb("capture")
    kb.attach_wal(log)
    kb.insert("u1", "d1", "a.md", _chunks("a", 8))
    if second:
        kb.checkpoint(d)
    kb.insert("u1", "d1", "a.md", _chunks("a revised", 2))
    kb.insert("u2", "d2", "b.md", _chunks("b", 5), org_id="o")
    kb.delete_where(lambda p: p["document_id"] == "d1" and p["chunk_index"] == 5)

    def boom(s):
        if s == stage:
            raise Crash(s)
    with pytest.raises(Crash):
        kb.checkpoint(d, on_stage=boom)
    kb.insert("u3", "d3", "c.md", _chunks("c", 2))           # acknowledged after the failed checkpoint
    # the process dies here: a copy of the directory is what a restart finds
    crashed = str(tmp_path / "crashed")
    shutil.copytree(d, crashed)
    if os.path.exists(os.path.join(crashed, "meta.json")):
        back = _restore(crashed, "capture")
    else:
        back = _kb("capture")
    back.attach_wal(os.path.join(crashed, "mutations.log"))
    _assert_same(back, kb)
    assert kb.checkpoint(d)["kind"] == "base"                 # the store starts over from a base
    _assert_same(_restore(d, "capture"), kb)

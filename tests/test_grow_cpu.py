"""KnowledgeBase growth on the host: before an insert appends anything, every shard that lacks room for the rows the
insert places on it (``id mod n``) is asked to grow to that need rounded up to 65,536 rows; an index without
``reserve`` still raises "shard full"."""

from __future__ import annotations

import numpy as np
import pytest

from aurora_b200 import retriever as R
from aurora_b200.engine import GROW_STEP, MultiIndex, grow_for
from tests.doubles import HashEmbedder, OracleIndex


class GrowingIndex(OracleIndex):
    """The CPU double with ``reserve``: records every request and grows its capacity."""

    def __init__(self, dim, capacity):
        super().__init__(dim, capacity)
        self.reserved = []

    def reserve(self, capacity):
        self.reserved.append(int(capacity))
        self.capacity = max(self.capacity, int(capacity))

    @classmethod
    def load(cls, path, capacity=None):
        """As engine.Index.load: room for the snapshot's rows first, then one add."""
        z = np.load(path if path.endswith(".npz") else path + ".npz")
        ix = cls(int(z["dim"]), int(capacity or z["capacity"]))
        grow_for(ix, z["ids"])
        ix.add(z["rows"], z["ids"], z["user"], z["org"])
        return ix


class KwStore:
    """A keyword store double with ``reserve``: counts appended documents, records reserves, raises when full."""

    def __init__(self, capacity):
        self.capacity, self.docs, self.reserved = int(capacity), 0, []

    def add(self, ids, terms, tfs, offsets, user_codes=None, org_codes=None):
        if self.docs + len(ids) > self.capacity:
            raise RuntimeError("keyword store full")
        self.docs += len(ids)

    def stats(self):
        return {"docs": self.docs}

    def reserve(self, capacity):
        self.reserved.append(int(capacity))
        self.capacity = max(self.capacity, int(capacity))


def _chunks(n, tag="x"):
    return [{"content": f"{tag} chunk {i} about disks", "chunk_index": i} for i in range(n)]


def test_single_shard_grows_to_the_need_rounded_up():
    kb = R.KnowledgeBase(HashEmbedder(32), capacity=100, index_factory=lambda d, c: GrowingIndex(d, c))
    assert kb.insert("u", "a", "f.md", _chunks(80)) == 80
    assert kb.index.reserved == []                                   # fits: nothing asked
    assert kb.insert("u", "b", "f.md", _chunks(50, "b")) == 50
    assert kb.index.reserved == [GROW_STEP]                          # 130 rows needed -> one step
    assert kb.insert("u", "b", "f.md", _chunks(50, "b")) == 50       # upserts append rows too: 180 <= 65,536
    assert kb.index.reserved == [GROW_STEP]
    assert kb.index.stats()["rows"] == 180 and kb.query("disks", 3)


def test_multi_index_shards_receive_the_needs_of_the_id_placement():
    shards = []

    def factory(d, c, dev):
        shards.append(GrowingIndex(d, c))
        return shards[-1]

    kb = R.KnowledgeBase(HashEmbedder(32), capacity=96,
                         index_factory=lambda d, c: MultiIndex(d, c, devices=[0, 0, 0], shard_factory=factory))
    per = shards[0].capacity                                         # shard_capacity(96, 3) = 32 + 64
    assert per == 96
    kb.insert("u", "a", "f.md", _chunks(200))                       # ids 0 .. 199: 67, 67, 66 per shard: room
    kb.insert("u", "b", "f.md", _chunks(100, "b"))                  # ids 200 .. 299: 100, 100, 100 in all
    need = np.bincount(np.arange(300) % 3, minlength=3)
    assert [s.reserved for s in shards] == [[GROW_STEP] if m > per else [] for m in need]
    assert [s.stats()["rows"] for s in shards] == list(need)
    assert kb.index.capacity >= 3 * GROW_STEP


def test_grow_for_skips_shards_without_share_or_reserve():
    a, b = GrowingIndex(8, 4), OracleIndex(8, 4)
    mi = MultiIndex(8, 8, devices=[0, 0], _shards=[a, b])
    grow_for(mi, np.array([0, 2, 4, 6, 8, 1], np.int64))            # shard 0: 5 rows > 4; shard 1: 1 row, no reserve
    assert a.reserved == [GROW_STEP] and a.capacity == GROW_STEP and b.capacity == 4
    grow_for(mi, np.array([], np.int64))
    assert a.reserved == [GROW_STEP]


def test_loading_a_grown_base_reserves_its_rows_once(tmp_path, monkeypatch):
    """A restore grows the shard to the snapshot's rows rounded up once: the keyword side's room check after the load
    must not count the loaded rows a second time (a reserve of twice the corpus)."""
    from aurora_b200 import engine
    from aurora_b200.bm25 import DeviceBM25

    stores = []
    monkeypatch.setattr(engine, "GROW_STEP", 64)
    # a keyword store the knowledge base treats as a device one (the load path that appends every text in one call)
    monkeypatch.setattr(R.KnowledgeBase, "_keyword_store", lambda self, cap: DeviceBM25(store=stores.append(KwStore(cap)) or stores[-1]))
    kb = R.KnowledgeBase(HashEmbedder(32), capacity=16, index_factory=lambda d, c: GrowingIndex(d, c))
    assert kb._kw_device
    kb.insert("u", "a", "f.md", _chunks(100))
    assert kb.index.reserved == [128] and stores[0].reserved == [128]
    kb.save(str(tmp_path / "kb"))
    again = R.KnowledgeBase.load(str(tmp_path / "kb"), HashEmbedder(32), capacity=16,
                                 index_loader=lambda p, cap: GrowingIndex.load(p, capacity=cap))
    assert again.index.reserved == [128] and again.index.capacity == 128
    assert stores[1].reserved == [128] and stores[1].docs == 100
    assert again.index.stats()["rows"] == 100


def test_index_without_reserve_still_raises_shard_full():
    kb = R.KnowledgeBase(HashEmbedder(32), capacity=10, index_factory=lambda d, c: OracleIndex(d, c))
    kb.insert("u", "a", "f.md", _chunks(10))
    with pytest.raises(RuntimeError, match="shard full"):
        kb.insert("u", "b", "f.md", _chunks(1, "b"))

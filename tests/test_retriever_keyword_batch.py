"""query_batch with a batched keyword store: an object deleted after the batch's keyword search and before its results
are fused (another request thread's delete) drops out of the answer instead of failing the batch.  CPU only: the
keyword store is a host stand-in with DeviceBM25's batch surface (the GPU run is in test_gpu_keyword.py)."""

from aurora_b200 import retriever as R
from aurora_b200.bm25 import BM25Index
from tests.doubles import HashEmbedder, OracleIndex


class DeletingKeywordStore:
    """search_batch answers like BM25Index, then deletes the first id it returned through the knowledge base."""

    def __init__(self, kb):
        self.kb, self.host, self.deleted = kb, BM25Index(), []

    def add_many(self, ids, texts, user_codes=None, org_codes=None):
        for d, t in zip(ids, texts):
            self.host.add(int(d), t)

    def remove_many(self, ids):
        return sum(self.host.remove(int(d)) for d in ids)

    def search_batch(self, queries, limit, q_user=None, q_org=None):
        out = [self.host.search(q, limit) for q in queries]
        victim = next(d for lst in out for d, _ in lst)
        key = self.kb._id2key[victim]
        self.kb._delete_keys([key])
        self.deleted.append(key)
        return out


def test_object_deleted_between_keyword_search_and_fusion_drops_out():
    kb = R.KnowledgeBase(HashEmbedder(64), capacity=512, index_factory=lambda d, c: OracleIndex(d, c))
    store = DeletingKeywordStore(kb)
    kb.sparse, kb._kw_device = store, True
    kb.insert("u1", "doc", "f.md", [{"content": t, "chunk_index": i} for i, t in
                                    enumerate(["disk full on node", "disk pressure", "cpu spike", "oom kill disk"])])
    res = kb.query_batch([("u1", "disk", 5, 0.5, None), ("u1", "disk node", 5, 0.0, None), ("u1", "cpu", 5, None, None)])
    assert len(store.deleted) == 1
    gone = store.deleted[0]
    assert res[0] and res[1]                                   # the other matches are still there
    assert all(o.uuid != gone for objs in res for o in objs)

"""Drop-in for ``server/routes/knowledge_base/weaviate_client.py`` backed by the H100 engine.

Same public names, keyword arguments, return shapes and error conventions as the
reference module (file:line cited on every function), so its callers keep working
unchanged:

* ``routes/knowledge_base/routes.py:455-485``            (REST ``/search``)
* ``chat/backend/agent/tools/knowledge_base_search_tool.py:61-70`` (LangGraph tool)
* ``routes/knowledge_base/tasks.py:75-83``               (Celery ingest worker)
* ``chat/backend/agent/tools/discovery_finding_tool.py:68-89``
* ``chat/background/rca_prompt_builder.py:266-328``      (via ``_get_weaviate_client()``)

What changes underneath: the Weaviate server (vector index) and the t2v-transformers
container (text -> vector) are replaced by an in-HBM corpus shard searched with the
fused similarity + top-k CUDA kernels (``aurora_b200.engine.Index``) and an encoder
object.  Documented deviations (see DESIGN.md): ``score`` is the cosine of the dense leg
(the reference's hybrid call returns a ranked-fusion score; BM25 is a "next" row), and the
embedded text is ``heading_context + "\\n" + content`` (the reference vectorises all TEXT
properties, weaviate_client.py:113-126).

There is no CPU fallback: without the CUDA library / a GPU the first call raises inside
and the reference's own conventions apply (search -> ``[]``, insert re-raises, ...).
"""

from __future__ import annotations

import logging
import os
import threading
import uuid
from datetime import datetime, timezone
from types import SimpleNamespace
from typing import Any, Callable, Dict, List, Optional, Tuple

import numpy as np

from ._native import AUR_BF16, AUR_I8, FUSION_RANKED, FUSION_RELATIVE_SCORE
from .bm25 import BM25Index
from .filters import AttrColumn, Filter, HybridFusion, compile_program  # noqa: F401  (Filter, HybridFusion: re-exported)

logger = logging.getLogger(__name__)

COLLECTION_NAME = "KnowledgeBaseChunk"  # weaviate_client.py:23
_MAX_FETCH = 128                        # engine's largest k
# A filtered query reads only its allowed rows (Index.search_lists) while they are at most this fraction of the live
# objects; above it the masked full scan (search_subset) answers sooner.  Measured at one query over 1M x 768 bf16
# (DESIGN.md section 9, tools/list_bench.py): the list path wins at 3 000 rows (0.3 %), the full scan at 10 000 (1 %).
_LIST_MAX_FRACTION = 0.005
_ATTR_COLS = range(2, 18)               # the shard's attribute columns (include/aurora_b200.h, aur_set_attrs)
# hybrid fusions the knowledge base implements, as aur_hybrid_search's AUR_FUSION_* values
_FUSION = {HybridFusion.RANKED: FUSION_RANKED, HybridFusion.RELATIVE_SCORE: FUSION_RELATIVE_SCORE}


def _sanitize(value: Any) -> str:
    """utils.log_sanitizer.sanitize stand-in: strip control characters from logged values."""
    return "".join(ch if ch.isprintable() else "?" for ch in str(value))


def generate_uuid5(identifier: str) -> str:
    """weaviate.util.generate_uuid5 with the default (empty) namespace argument:
    uuid5(NAMESPACE_DNS, str(identifier)).  Used for idempotent upserts (weaviate_client.py:172)."""
    return str(uuid.uuid5(uuid.NAMESPACE_DNS, str(identifier)))


class KnowledgeBase:
    """Chunk store: vectors in the GPU index, properties in a host-side table.

    ``encoder`` must provide ``dim`` and ``encode(list[str]) -> np.ndarray [n, dim]``
    (float32 or bf16 bits).  ``index_factory(dim, capacity)`` builds the vector shard;
    the default is the CUDA engine.
    """

    def __init__(self, encoder, capacity: int = 1 << 20, device: int = 0,
                 index_factory: Optional[Callable[[int, int], Any]] = None, dtype: str = "bf16"):
        if encoder is None:
            raise RuntimeError("aurora_b200.retriever needs an encoder (text -> vector); none configured")
        self.encoder = encoder
        self.dim = int(encoder.dim)
        if index_factory is None:
            from .engine import Index  # raises loudly if the CUDA library is missing

            def index_factory(dim, cap):
                return Index(dim, cap, dtype=dtype, device=device)   # "int8": half the HBM, exact over the int8 rows
        self.index = index_factory(self.dim, int(capacity))
        # keyword leg of the hybrid query: on the GPU beside a CUDA vector index, else the host index
        self.sparse = self._keyword_store(int(capacity))
        self._kw_device = not isinstance(self.sparse, BM25Index)
        self._hybrid_device = self._fuses_on_device()
        self._lock = threading.RLock()  # the reference's module globals are unlocked (weaviate_client.py:31-32)
        self._props: Dict[int, Dict[str, Any]] = {}   # id -> properties
        self._key2id: Dict[str, int] = {}             # uuid5 -> id
        self._id2key: Dict[int, str] = {}
        self._by_user: Dict[str, set] = {}            # host-side inverted lists: narrow a filter's metadata scan
        self._by_org: Dict[str, set] = {}
        self._next_id = 0
        self._user_code: Dict[str, int] = {}
        self._org_code: Dict[str, int] = {}
        self.saved_mutations = 0
        self.mutations = 0              # inserts + deletes over the store's life (the daemon's snapshot policy reads it)
        self._wal = None                # mutation log between snapshots (attach_wal)
        self._wal_path: Optional[str] = None
        self._wal_sync = True
        self._replaying = False
        self._scope_cache: Dict[Tuple[Optional[str], Optional[str]], tuple] = {}   # tenant -> (mutations, id set, sorted ids)
        # filters evaluated on the device: a property gets an attribute column of the shard the first time a filter names
        # it, and keeps it current from then on (insert_objects)
        self._attr_cols: Dict[str, AttrColumn] = {}
        self._attr_free = list(_ATTR_COLS)
        self._attr_host: set = set()    # properties with a value that has no code (unhashable): their filters stay on the host

    def _keyword_store(self, capacity: int):
        """``DeviceBM25`` on the vector index's GPU when that index is an ``engine.Index``; over a ``MultiIndex`` of them,
        one keyword store on each shard's GPU (``engine.MultiKeywordIndex``, searched as one corpus); else
        ``BM25Index``.  All score the same (DESIGN.md section 10)."""
        from .bm25 import DeviceBM25
        from .engine import Index, MultiIndex, MultiKeywordIndex

        ix = self.index
        if isinstance(ix, Index):
            return DeviceBM25(capacity, device=ix.device)
        if isinstance(ix, MultiIndex) and ix.shards and all(isinstance(sh, Index) for sh in ix.shards):
            return DeviceBM25(store=MultiKeywordIndex(capacity, devices=[sh.device for sh in ix.shards]))
        return BM25Index()

    def _fuses_on_device(self) -> bool:
        """Whether a hybrid query runs as one device call, both legs and their fusion (``engine.hybrid_search``): a bf16
        or int8 ``engine.Index`` and a ``DeviceBM25`` over a ``KeywordIndex`` on its GPU, or a ``MultiIndex`` of such
        ``engine.Index`` shards and a ``DeviceBM25`` over a ``MultiKeywordIndex`` on the same devices in the same order.
        Filtered queries too, when their filter compiles to a device program (attribute columns are then kept on the
        keyword store as well).  f32 shards, the CPU doubles and filters that stay on the host fuse on the host
        (``bm25.ranked_fusion`` / ``relative_score_fusion``)."""
        from .bm25 import DeviceBM25
        from .engine import Index, KeywordIndex, MultiIndex, MultiKeywordIndex

        ix, sp = self.index, self.sparse
        if not isinstance(sp, DeviceBM25):
            return False
        if isinstance(ix, MultiIndex):
            return (bool(ix.shards) and all(isinstance(sh, Index) and sh.dtype in (AUR_BF16, AUR_I8) for sh in ix.shards)
                    and isinstance(sp.store, MultiKeywordIndex) and sp.store.devices == ix.devices
                    and len(sp.store.stores) == len(ix.shards))
        return (isinstance(ix, Index) and ix.dtype in (AUR_BF16, AUR_I8) and isinstance(sp.store, KeywordIndex)
                and sp.store.device == ix.device)

    def _scope_codes(self, user_id: Optional[str], org_id: Optional[str]) -> Tuple[int, int]:
        """Tenant scope as the kernels take it: (user code, org code); -2 matches no row, org -1 = no org."""
        cu = self._code(self._user_code, user_id, False) if user_id else -2
        co = self._code(self._org_code, org_id, False) if org_id else -1
        return cu, (-1 if co == -2 else co)

    # ------------------------------------------------------------------ tenant codes
    def _code(self, table: Dict[str, int], key: Optional[str], create: bool) -> int:
        if not key:
            return -1
        if key not in table:
            if not create:
                return -2  # matches no row
            table[key] = len(table)
        return table[key]

    # ------------------------------------------------------------------ mutation log (durability between snapshots)
    def attach_wal(self, path: str, sync: bool = True) -> int:
        """Log every acknowledged mutation to ``path`` (JSON lines, fsync'd before the call returns) so that a crash
        loses nothing a caller was told had been stored -- Weaviate keeps its own WAL on the data volume
        (docker-compose.yaml:477-478).  Records already in the file that are newer than this store's state (a restart
        after a crash: ``load`` restored the last snapshot) are replayed first: inserts re-encode their text -- the encoder
        is deterministic -- deletes name the object keys.  ``save`` truncates the log.  Returns the replayed count."""
        import json

        with self._lock:
            replayed = 0
            if os.path.exists(path):
                self._replaying = True
                try:
                    good = 0
                    with open(path, "rb") as f:
                        for raw in f:
                            try:
                                if not raw.endswith(b"\n"):
                                    raise ValueError("no terminator")
                                rec = json.loads(raw.decode("utf-8"))
                            except ValueError:
                                break                    # torn final record of a crash mid-write: never acknowledged
                            good += len(raw)
                            if int(rec.get("gen", -1)) < self.mutations:
                                continue                 # already inside the snapshot this store was loaded from
                            if rec["op"] == "put":
                                self.insert_objects([tuple(o) for o in rec["objs"]], rec.get("user"), rec.get("org"))
                            elif rec["op"] == "del":
                                self._delete_keys(rec["keys"])
                            replayed += 1
                finally:
                    self._replaying = False
                if good < os.path.getsize(path):
                    with open(path, "r+b") as f:       # drop the torn tail so that new records start on a fresh line
                        f.truncate(good)
            self._wal_path, self._wal_sync = path, sync
            self._wal = open(path, "a", encoding="utf-8")
            return replayed

    def _log(self, rec: Dict[str, Any]) -> None:
        if self._wal is None or self._replaying:
            return
        import json

        self._wal.write(json.dumps(rec, separators=(",", ":")) + "\n")
        self._wal.flush()
        if self._wal_sync:
            os.fsync(self._wal.fileno())

    def _delete_keys(self, keys: List[str]) -> int:
        ids = [self._key2id[k] for k in keys if k in self._key2id]
        return self._delete_ids(ids)

    # ------------------------------------------------------------------ ingest
    def insert(self, user_id: str, document_id: str, source_filename: str, chunks: List[Dict[str, Any]],
               org_id: Optional[str] = None) -> int:
        now = datetime.now(timezone.utc).isoformat()          # weaviate_client.py:165
        objs = []
        for chunk in chunks:
            try:
                chunk_index = chunk.get("chunk_index", 0)
                props = {
                    "user_id": user_id, "document_id": document_id, "chunk_index": chunk_index,
                    "content": chunk.get("content", ""), "heading_context": chunk.get("heading_context", ""),
                    "source_filename": source_filename, "created_at": now,
                }
                if org_id:
                    props["org_id"] = org_id               # weaviate_client.py:183-184
                key = generate_uuid5(f"{user_id}:{document_id}:{chunk_index}")
                heading = props["heading_context"]
                objs.append((key, props, (heading + "\n" if heading else "") + props["content"]))
            except Exception as e:  # per-object failure: counted out, not fatal (weaviate_client.py:189-190)
                logger.error(f"[KB B200] Error adding chunk: {e}")
        return self.insert_objects(objs, user_id, org_id)

    def insert_objects(self, objs: List[Tuple[str, Dict[str, Any], str]], user_id: Optional[str],
                       org_id: Optional[str] = None) -> int:
        """Upsert ``(uuid key, properties, text to embed)`` objects of one tenant: the text is encoded on the
        GPU and the vector appended to the shard; an existing key replaces its old vector and properties."""
        if not objs:
            return 0
        texts = [t for _, _, t in objs]
        fused = hasattr(self.encoder, "encode_append") and hasattr(self.index, "_h")   # CUDA encoder + CUDA shard
        vecs = None if fused else self.encoder.encode(texts)
        with self._lock:
            gen = self.mutations
            ids = np.empty(len(objs), dtype=np.int64)
            for i, (key, _, _) in enumerate(objs):
                if key not in self._key2id:
                    self._key2id[key] = self._next_id
                    self._id2key[self._next_id] = key
                    self._next_id += 1
                ids[i] = self._key2id[key]
            ucode = np.full(len(objs), self._code(self._user_code, user_id, True), dtype=np.int32)
            ocode = np.full(len(objs), self._code(self._org_code, org_id, True), dtype=np.int32)
            if fused:
                self.encoder.encode_append(self.index, texts, ids, ucode, ocode)
            else:
                self.index.add(vecs, ids, ucode, ocode)
            for i, (_, props, text) in enumerate(objs):
                rid = int(ids[i])
                old = self._props.get(rid)
                if old is not None:
                    self._unindex(rid, old)
                self._props[rid] = props
                self._by_user.setdefault(props.get("user_id"), set()).add(rid)
                if props.get("org_id"):
                    self._by_org.setdefault(props["org_id"], set()).add(rid)
                if not self._kw_device:
                    self.sparse.add(rid, text)
            if self._kw_device:
                self.sparse.add_many(ids, texts, ucode, ocode)
            if self._attr_cols:             # before the lock is released: no query sees the new rows without their codes
                self._set_attr_codes(np.unique(ids))
            self.mutations += len(objs)
            self._log({"op": "put", "gen": gen, "user": user_id, "org": org_id, "objs": [list(o) for o in objs]})
        return len(objs)

    def _tenant_scope(self, user_id: Optional[str], org_id: Optional[str]):
        """(set, ascending int64 array) of the ids a tenant sees (its user's rows OR its org's), kept until the next
        mutation: building them is O(tenant size), a query is not.  Caller holds the lock."""
        key = (user_id or None, org_id or None)
        hit = self._scope_cache.get(key)
        if hit is not None and hit[0] == self.mutations:
            return hit[1], hit[2]
        by_u = self._by_user.get(user_id, set()) if user_id else set()
        by_o = self._by_org.get(org_id, set()) if org_id else set()
        ids = (by_u | by_o) if (by_u and by_o) else (by_u or by_o)
        arr = np.fromiter(ids, dtype=np.int64, count=len(ids))
        arr.sort()
        if len(self._scope_cache) >= 256:
            self._scope_cache.clear()
        self._scope_cache[key] = (self.mutations, ids, arr)
        return ids, arr

    # ------------------------------------------------------------------ device filters
    def _set_attr_codes(self, rids: np.ndarray) -> None:
        """Every attribute column's codes of the rows ``rids`` from their current properties.  Caller holds the lock."""
        for name, col in list(self._attr_cols.items()):
            try:
                codes = np.array([col.code(self._props[int(r)]) for r in rids], dtype=np.int32)
            except TypeError:               # a value without a code: this property's filters go back to the host path
                del self._attr_cols[name]
                self._attr_host.add(name)
                self._attr_free.append(col.col)   # the slot serves the next property (its codes are rewritten then)
                continue
            self._write_attr(col.col, rids, codes)

    def _write_attr(self, col: int, rids: np.ndarray, codes: np.ndarray) -> None:
        """Attribute column ``col`` of the rows ``rids`` on the vector index and, when hybrid queries fuse on the device
        (their filter programs then run on the keyword store too), on the keyword store.  Caller holds the lock."""
        self.index.set_attrs(col, rids, codes)
        if self._hybrid_device:
            self.sparse.store.set_attrs(col, rids, codes)

    def _attr_column(self, name: str) -> AttrColumn:
        """The attribute column of property ``name``, built from the whole table on first use.  Caller holds the lock."""
        col = self._attr_cols.get(name)
        if col is not None:
            return col
        if name in self._attr_host or not self._attr_free:
            raise KeyError(name)
        col = AttrColumn(name, self._attr_free[0])
        rids = np.fromiter(self._props.keys(), dtype=np.int64, count=len(self._props))
        try:
            codes = np.array([col.code(self._props[int(r)]) for r in rids], dtype=np.int32)
        except TypeError:
            self._attr_host.add(name)
            raise
        self._write_attr(col.col, rids, codes)     # a slot handed back by another property is rewritten on every row
        self._attr_free.pop(0)
        self._attr_cols[name] = col
        return col

    def _device_program(self, filters, tenant: bool, user_id: Optional[str], org_id: Optional[str]):
        """``filters`` AND the tenant scope as a device program over attribute columns, or None when the query is
        resolved on the host: an index without device filters (CPU doubles, f32 shards), a property without a column, or
        a leaf whose evaluation raises (the host path then raises as it always has).  The tenant scope is written over
        the ``user_id`` / ``org_id`` properties, exactly as the host predicate reads it.  Caller holds the lock."""
        if not hasattr(self.index, "search_filtered") or getattr(self.index, "dtype", None) not in (AUR_BF16, AUR_I8):
            return None
        expr = filters
        if tenant:
            terms = ([Filter.by_property("user_id").equal(user_id)] if user_id else []) + \
                    ([Filter.by_property("org_id").equal(org_id)] if org_id else [])
            if not terms:
                return None                 # matches nothing: the host path answers without a search
            expr = filters & (terms[0] if len(terms) == 1 else terms[0] | terms[1])
        names: List[str] = []

        def walk(t):
            if t[0] in ("and", "or"):
                walk(t[1])
                walk(t[2])
            elif t[1] not in names:
                names.append(t[1])
        try:
            walk(expr.tree)
            return compile_program(expr, {n: self._attr_column(n) for n in names})
        except Exception:                   # noqa: BLE001 - any failure keeps the host path and its behaviour
            return None

    def _unindex(self, rid: int, props: Dict[str, Any]) -> None:
        self._by_user.get(props.get("user_id"), set()).discard(rid)
        if props.get("org_id"):
            self._by_org.get(props["org_id"], set()).discard(rid)

    # ------------------------------------------------------------------ search
    def query(self, query: str, limit: int, filters=None, user_id: Optional[str] = None,
              org_id: Optional[str] = None, alpha: Optional[float] = None, scoped: bool = False,
              fusion: str = HybridFusion.RANKED,
              _dense: Optional[List[Tuple[int, float]]] = None,
              _sparse: Optional[List[Tuple[int, float]]] = None,
              _fused: Optional[list] = None) -> List[SimpleNamespace]:
        """Top-``limit`` objects.  ``alpha`` None or >= 1: pure vector search, ``score`` = cosine
        (near_text, incident_feedback/weaviate_client.py:286-297).  ``alpha`` < 1: hybrid
        (weaviate_client.py:252-259), ``score`` = the fused score of the dense and BM25 lists with weights
        alpha and 1 - alpha: ``fusion`` = ``HybridFusion.RANKED`` (weight / (rank + 60) per list) or
        ``HybridFusion.RELATIVE_SCORE`` (weight times the score min-max normalised over its list).

        Filters are PRE-filters, as in Weaviate: the tenant scope (user OR org) runs inside the kernel;
        a ``filters`` expression on a CUDA shard is compiled to a program over the shard's attribute
        columns and evaluated there (``Index.search_filtered``); elsewhere it is resolved against the
        metadata table to the set of allowed ids.  Either way the kernel searches only the matching rows,
        so a small tenant's chunks are found even when the global top-k belongs to other tenants.

        A hybrid query on a CUDA shard is one device call (``DeviceBM25.search_batch`` with ``dense``): both legs and
        their fusion run on the GPU and only the fused top-``limit`` comes back.  A filtered one goes the same way when
        its filter compiles to a device program, which both legs then evaluate on the GPU.  Objects deleted after
        that call drop out of the answer; the others keep the scores the device computed (the answer as of the
        search).  Elsewhere the two lists come back and are fused on the host.

        ``scoped``: the caller is a tenant-facing entry point (search_knowledge_base): a missing user AND
        org matches nothing instead of everything (the reference always applies ``user_id == u``,
        weaviate_client.py:244-249)."""
        if limit <= 0:
            return []
        if scoped and not user_id and not org_id:
            return []
        if fusion is None:
            fusion = HybridFusion.RANKED
        if fusion not in _FUSION:
            raise NotImplementedError(f"hybrid fusion {fusion!r}: only HybridFusion.RANKED and RELATIVE_SCORE are implemented")
        hybrid = alpha is not None and alpha < 1.0
        dense_w = 1.0 if not hybrid else max(0.0, float(alpha))
        on_device = (_fused is None and _dense is None and _sparse is None and hybrid and filters is None
                     and self._hybrid_device)
        if on_device:                       # a query whose dense leg is ignored still passes a vector: zeros
            qv = self.encoder.encode([query]) if dense_w > 0.0 else np.zeros((1, self.dim), np.float32)
        else:
            qv = self.encoder.encode([query]) if (dense_w > 0.0 and _dense is None and _fused is None) else None
        with self._lock:
            tenant = scoped or user_id is not None or org_id is not None
            if on_device:
                q_user = q_org = None
                if tenant:
                    cu, co = self._scope_codes(user_id, org_id)
                    q_user, q_org = np.array([cu], np.int32), np.array([co], np.int32)
                _fused = self.sparse.search_batch([query], _MAX_FETCH, q_user, q_org,
                                                  dense=(self.index, qv, np.array([dense_w]), _FUSION[fusion],
                                                         min(limit, 2 * _MAX_FETCH)))[0]
            if _fused is not None:          # fused on the device (here or by query_batch)
                return self._shape([(rid, fs, cos) for rid, (fs, cos) in _fused if rid in self._props][:limit])

            def tenant_ok(props) -> bool:
                if not tenant:
                    return True
                return (bool(user_id) and props.get("user_id") == user_id) or \
                       (bool(org_id) and props.get("org_id") == org_id)

            allowed: Optional[List[int]] = None
            prog = self._device_program(filters, tenant, user_id, org_id) if filters is not None else None
            if prog is not None and hybrid and self._hybrid_device and _dense is None and _sparse is None:
                # the whole filtered hybrid query in one device call: both legs evaluate the program on the GPU
                if qv is None:              # the dense leg is ignored (alpha <= 0) but still takes a vector
                    qv = np.zeros((1, self.dim), np.float32)
                fused = self.sparse.search_batch(
                    [query], _MAX_FETCH, dense=(self.index, qv, np.array([dense_w]), _FUSION[fusion], min(limit, 2 * _MAX_FETCH)),
                    programs=[prog], max_list_rows=int(_LIST_MAX_FRACTION * len(self._props)))[0]
                return self._shape([(rid, fs, cos) for rid, (fs, cos) in fused if rid in self._props][:limit])
            if filters is not None and prog is None:
                # narrow the scan with the filter's own equality terms and the tenant scope, then run the predicate
                eq = filters.required_equalities()
                pools = []
                if "org_id" in eq:
                    pools.append(self._by_org.get(eq["org_id"], set()))
                if "user_id" in eq:
                    pools.append(self._by_user.get(eq["user_id"], set()))
                if tenant:
                    pools.append(self._by_user.get(user_id, set()) | (self._by_org.get(org_id, set()) if org_id else set()))
                cand = set.intersection(*pools) if pools else self._props.keys()
                allowed = [rid for rid in cand if filters.matches(self._props[rid]) and tenant_ok(self._props[rid])]

            dense: List[Tuple[int, float]] = []
            if _dense is not None:          # dense leg already computed by query_batch (same scope, same fetch)
                dense = [(rid, sc) for rid, sc in _dense if rid in self._props]
            elif qv is not None and (prog is not None or allowed is None or allowed):
                fetch = max(1, min(_MAX_FETCH, limit if not hybrid else _MAX_FETCH))
                if prog is not None:        # no id crosses PCIe; the list-vs-scan rule is the host path's
                    ids, scores, _, _ = self.index.search_filtered(
                        qv, fetch, [prog], max_list_rows=int(_LIST_MAX_FRACTION * len(self._props)))
                elif (allowed is not None and hasattr(self.index, "search_lists")
                        and len(allowed) <= _LIST_MAX_FRACTION * len(self._props)):   # reads only the allowed rows
                    ids, scores = self.index.search_lists(qv, fetch, [np.asarray(allowed, dtype=np.int64)],
                                                          np.zeros(1, np.int32))
                elif allowed is not None:
                    ids, scores = self.index.search_subset(qv, fetch, np.asarray(allowed, dtype=np.int64))
                else:
                    q_user = q_org = None
                    if tenant:
                        q_user = np.array([self._code(self._user_code, user_id, False) if user_id else -2], dtype=np.int32)
                        q_org = np.array([self._code(self._org_code, org_id, False) if org_id else -1], dtype=np.int32)
                        if q_org[0] == -2:
                            q_org[0] = -1
                    ids, scores = self.index.search(qv, fetch, q_user, q_org)
                for rid, sc in zip(ids[0], scores[0]):
                    if rid < 0:
                        break
                    if int(rid) in self._props:
                        dense.append((int(rid), float(sc)))
            if not hybrid:
                picked = [(rid, sc, sc) for rid, sc in dense[:limit]]
            else:
                # keyword leg under the same pre-filter: the resolved filter's ids, else the tenant's own inverted lists.
                # A device program reaches here only with the keyword leg on the host (BM25Index beside an index that
                # evaluates programs, e.g. a MultiIndex of CPU shard doubles): the device knowledge base fused above.
                if prog is not None and _sparse is None:
                    allowed = self.index.filter_ids(prog).tolist()
                if _sparse is not None:     # keyword leg already computed by query_batch (same scope, same fetch);
                    # objects deleted since then drop out, as for the dense leg
                    sparse = [(rid, sc) for rid, sc in _sparse if rid in self._props]
                elif self._kw_device:       # the device applies the tenant scope itself, as the dense leg does
                    if allowed is not None:
                        sparse = self.sparse.search(query, _MAX_FETCH, allowed=allowed)
                    elif tenant:
                        cu, co = self._scope_codes(user_id, org_id)
                        sparse = self.sparse.search_batch([query], _MAX_FETCH, np.array([cu], np.int32),
                                                          np.array([co], np.int32))[0]
                    else:
                        sparse = self.sparse.search(query, _MAX_FETCH)
                else:
                    allowed_arr = None
                    if allowed is not None:
                        allowed_set = set(allowed)
                    elif tenant:
                        allowed_set, allowed_arr = self._tenant_scope(user_id, org_id)
                    else:
                        allowed_set = None
                    sparse = self.sparse.search(query, _MAX_FETCH, allowed=allowed_set, allowed_sorted=allowed_arr)
                from . import bm25

                cos = dict(dense)
                if fusion == HybridFusion.RELATIVE_SCORE:
                    fused = bm25.relative_score_fusion([(dense_w, dense), (1.0 - dense_w, sparse)], limit)
                else:
                    fused = bm25.ranked_fusion([(dense_w, [d for d, _ in dense]), (1.0 - dense_w, [d for d, _ in sparse])],
                                               limit)
                picked = [(rid, fs, cos.get(rid)) for rid, fs in fused]
            return self._shape(picked)

    def _shape(self, picked) -> List[SimpleNamespace]:
        """(id, score, dense cosine or None) -> result objects.  Caller holds the lock."""
        out = []
        for rid, score, cosine in picked:
            meta = SimpleNamespace(score=float(score), distance=None if cosine is None else 1.0 - float(cosine))
            out.append(SimpleNamespace(properties=dict(self._props[rid]), uuid=self._id2key.get(rid), metadata=meta))
        return out

    def query_batch(self, reqs: List[Tuple[Optional[str], str, int, Optional[float], Optional[str]]]) -> List[List[SimpleNamespace]]:
        """Several tenant-scoped searches at once: ``(user_id, query, limit, alpha, org_id)`` each.  All query texts go
        through ONE encoder batch; the dense leg is ONE kernel launch per result size (the tenant scopes of the batch ride
        along as per-row bit masks on the tensor-core kernel); on a GPU keyword store the keyword leg of every hybrid request
        (alpha < 1) is ONE device search with per-request tenant codes; fusion / shaping per request as in ``query``.
        On a CUDA shard whose hybrid requests carry at most 32 distinct tenant scopes, those requests are instead ONE device
        call for both legs and their ranked fusion (``DeviceBM25.search_batch`` with ``dense``, per-request weights), and
        only shaping is left per request."""
        need = [i for i, (u, q, lim, a, o) in enumerate(reqs) if lim > 0 and (u or o) and (a is None or a > 0.0)]
        hyb = [i for i, (u, q, lim, a, o) in enumerate(reqs) if lim > 0 and (u or o) and a is not None and a < 1.0]
        vecs = self.encoder.encode([reqs[i][1] for i in need]) if need else None
        dense: Dict[int, List[Tuple[int, float]]] = {}
        sparse: Dict[int, List[Tuple[int, float]]] = {}
        fused: Dict[int, list] = {}
        with self._lock:
            if hyb and self._hybrid_device:
                codes = [self._scope_codes(reqs[i][0], reqs[i][4]) for i in hyb]
                if len(set(codes)) <= 32:   # the tensor-core kernel's per-row scope masks hold them
                    row = {i: pos for pos, i in enumerate(need)}
                    hv = np.zeros((len(hyb), self.dim), vecs.dtype if vecs is not None else np.float32)
                    for j, i in enumerate(hyb):
                        if i in row:        # alpha <= 0: the dense leg is ignored, its vector stays zero
                            hv[j] = vecs[row[i]]
                    lists = self.sparse.search_batch(
                        [reqs[i][1] for i in hyb], _MAX_FETCH, np.array([c[0] for c in codes], np.int32),
                        np.array([c[1] for c in codes], np.int32),
                        dense=(self.index, hv, np.array([max(0.0, float(reqs[i][3])) for i in hyb]), FUSION_RANKED,
                               min(max(reqs[i][2] for i in hyb), 2 * _MAX_FETCH)))
                    fused = dict(zip(hyb, lists))
            kw_need = [i for i in hyb if i not in fused] if self._kw_device else []
            if kw_need:
                codes = [self._scope_codes(reqs[i][0], reqs[i][4]) for i in kw_need]
                lists = self.sparse.search_batch([reqs[i][1] for i in kw_need], _MAX_FETCH,
                                                 np.array([c[0] for c in codes], np.int32),
                                                 np.array([c[1] for c in codes], np.int32))
                sparse = dict(zip(kw_need, lists))
            groups: Dict[int, List[Tuple[int, int, int]]] = {}      # fetch size -> [(position, user code, org code)]
            for pos, i in enumerate(need):
                if i in fused:
                    continue
                u, _, lim, a, o = reqs[i]
                hybrid = a is not None and a < 1.0
                fetch = max(1, min(_MAX_FETCH, lim if not hybrid else _MAX_FETCH))
                cu = self._code(self._user_code, u, False) if u else -2
                co = self._code(self._org_code, o, False) if o else -1
                groups.setdefault(fetch, []).append((pos, cu, -1 if co == -2 else co))
            for fetch, members in groups.items():
                pos = [m[0] for m in members]
                scopes: Dict[Tuple[int, int], int] = {}
                for m in members:
                    scopes.setdefault((m[1], m[2]), len(scopes))
                if len(scopes) > 32 and hasattr(self.index, "search_lists"):
                    # more scopes than the tensor-core kernel's row bit masks hold: one id list per scope (the rows
                    # _tenant_scope gives the keyword leg) and one list search that reads only those rows
                    lists: List[np.ndarray] = [np.empty(0, np.int64)] * len(scopes)
                    for m in members:
                        slot = scopes[(m[1], m[2])]
                        if not len(lists[slot]):
                            u, o = reqs[need[m[0]]][0], reqs[need[m[0]]][4]
                            lists[slot] = self._tenant_scope(u, o)[1]
                    ids, scores = self.index.search_lists(vecs[pos], fetch, lists,
                                                          np.array([scopes[(m[1], m[2])] for m in members], np.int32))
                else:
                    # one launch for the whole group: up to 32 distinct tenant scopes per batch ride on the tensor-core
                    # kernel as per-row bit masks (csrc/capi.cu search_host); the library falls back by itself beyond
                    ids, scores = self.index.search(vecs[pos], fetch, np.array([m[1] for m in members], np.int32),
                                                    np.array([m[2] for m in members], np.int32))
                for row, p_ in enumerate(pos):
                    dense[need[p_]] = [(int(r), float(s_)) for r, s_ in zip(ids[row], scores[row]) if r >= 0]
        out = []
        for i, (u, q, lim, a, o) in enumerate(reqs):
            out.append(self.query(q, lim, user_id=u, org_id=o, alpha=a, scoped=True, _dense=dense.get(i),
                                  _sparse=sparse.get(i), _fused=fused.get(i)))
        return out

    # ------------------------------------------------------------------ persistence
    def save(self, directory: str) -> None:
        """Durable snapshot (replaces the Weaviate data volume, docker-compose.yaml:477-478): the live
        vectors as ``shard.npz`` (tombstones compacted away) and the chunk metadata as ``meta.json``."""
        import json

        os.makedirs(directory, exist_ok=True)
        with self._lock:
            # both files are written beside their final names and renamed, shard first: a crash leaves either the
            # old pair or the new pair (meta.json names the shard generation it belongs to)
            gen = int(self.mutations)
            tmp_shard = os.path.join(directory, "shard.tmp")
            self.index.save(tmp_shard)
            os.replace(tmp_shard + ".npz", os.path.join(directory, f"shard.{gen}.npz"))
            meta = {"shard": f"shard.{gen}.npz", "version": 1, "generation": gen, "dim": self.dim, "next_id": self._next_id,
                    "user_code": self._user_code,
                    "org_code": self._org_code, "key2id": self._key2id,
                    "props": {str(k): v for k, v in self._props.items()}}
            tmp = os.path.join(directory, "meta.json.tmp")
            with open(tmp, "w", encoding="utf-8") as f:
                json.dump(meta, f)
            os.replace(tmp, os.path.join(directory, "meta.json"))
            for name in os.listdir(directory):     # older generations are garbage once meta.json points at the new one
                if name.startswith("shard.") and name.endswith(".npz") and name != meta["shard"]:
                    try:
                        os.remove(os.path.join(directory, name))
                    except OSError:
                        pass
            self.saved_mutations = gen
            if self._wal is not None:               # everything logged so far is inside the snapshot: start a fresh log.
                self._wal.close()                   # (a crash before this point leaves old records; replay skips them by gen)
                tmp_wal = self._wal_path + ".tmp"
                open(tmp_wal, "w").close()
                os.replace(tmp_wal, self._wal_path)
                self._wal = open(self._wal_path, "a", encoding="utf-8")

    @classmethod
    def load(cls, directory: str, encoder, capacity: int = 1 << 20, device: int = 0, index_loader=None,
             text_of: Optional[Callable[[Dict[str, Any]], str]] = None) -> "KnowledgeBase":
        """Rebuild from ``save``: vectors go back into HBM as they were stored (no re-encoding), the
        keyword index is rebuilt from the chunk texts."""
        import json

        if text_of is None:
            def text_of(p):
                heading = p.get("heading_context", "")
                return (heading + "\n" if heading else "") + p.get("content", "")
        with open(os.path.join(directory, "meta.json"), encoding="utf-8") as f:
            meta = json.load(f)
        if int(meta["dim"]) != int(encoder.dim):
            raise ValueError(f"snapshot is {meta['dim']}-d, encoder is {encoder.dim}-d")
        if index_loader is None:
            from .engine import Index

            def index_loader(path, cap):
                return Index.load(path, capacity=cap, device=device)
        loaded = index_loader(os.path.join(directory, meta.get("shard", "shard.npz")), int(capacity))
        kb = cls(encoder, capacity=capacity, device=device, index_factory=lambda dim, cap: loaded)
        kb._next_id = int(meta["next_id"])
        kb.mutations = kb.saved_mutations = int(meta.get("generation", 0))     # the log's records are ordered by it
        kb._user_code = {k: int(v) for k, v in meta["user_code"].items()}
        kb._org_code = {k: int(v) for k, v in meta["org_code"].items()}
        kb._key2id = {k: int(v) for k, v in meta["key2id"].items()}
        kb._id2key = {v: k for k, v in kb._key2id.items()}
        kb._props = {int(k): v for k, v in meta["props"].items()}
        for rid, p in kb._props.items():
            kb._by_user.setdefault(p.get("user_id"), set()).add(rid)
            if p.get("org_id"):
                kb._by_org.setdefault(p["org_id"], set()).add(rid)
            if not kb._kw_device:
                kb.sparse.add(rid, text_of(p))
        if kb._kw_device and kb._props:     # one device append for the whole store
            rids = list(kb._props)
            kb.sparse.add_many(rids, [text_of(kb._props[r]) for r in rids],
                               np.array([kb._code(kb._user_code, kb._props[r].get("user_id"), False) for r in rids], np.int32),
                               np.array([kb._code(kb._org_code, kb._props[r].get("org_id"), False) for r in rids], np.int32))
        return kb

    # ------------------------------------------------------------------ deletes / counts
    def _matching_ids(self, pred) -> List[int]:
        return [rid for rid, p in self._props.items() if pred(p)]

    def delete_where(self, pred) -> int:
        with self._lock:
            return self._delete_ids(self._matching_ids(pred))

    def _delete_ids(self, ids: List[int]) -> int:
        with self._lock:
            if ids:
                gen = self.mutations
                keys = [self._id2key.get(rid) for rid in ids]
                self.index.remove(np.array(ids, dtype=np.int64))
                if self._kw_device:
                    self.sparse.remove_many(ids)
                for rid in ids:
                    p = self._props.pop(rid)
                    self._unindex(rid, p)
                    if not self._kw_device:
                        self.sparse.remove(rid)
                    self._key2id.pop(self._id2key.pop(rid, None), None)
                self.mutations += len(ids)
                self._log({"op": "del", "gen": gen, "keys": [k for k in keys if k]})
            return len(ids)

    def count_where(self, pred) -> int:
        with self._lock:
            return len(self._matching_ids(pred))


# ---------------------------------------------------------------------- façade for _get_weaviate_client()
class _QueryFacade:
    def __init__(self, kb: KnowledgeBase):
        self._kb = kb

    def hybrid(self, query: str, limit: int = 10, alpha: float = 0.5, fusion_type=None, filters=None,
               return_metadata=None, **_):
        """``fusion_type`` None means RANKED, what the reference requests (Weaviate's own default since 1.24 is
        RELATIVE_SCORE); RELATIVE_SCORE is implemented too, anything else raises NotImplementedError."""
        if fusion_type not in (None, HybridFusion.RANKED, HybridFusion.RELATIVE_SCORE):
            raise NotImplementedError("only HybridFusion.RANKED (what the reference requests) and RELATIVE_SCORE are implemented")
        return SimpleNamespace(objects=self._kb.query(query, limit, filters=filters, alpha=alpha,
                                                      fusion=fusion_type or HybridFusion.RANKED))

    def near_text(self, query: str, limit: int = 10, filters=None, return_metadata=None, **_):
        return SimpleNamespace(objects=self._kb.query(query, limit, filters=filters))


class _CollectionFacade:
    """The slice of a weaviate Collection that rca_prompt_builder.py:291-317 touches."""

    def __init__(self, kb: KnowledgeBase):
        self.name = COLLECTION_NAME
        self.query = _QueryFacade(kb)


class _ClientFacade:
    def is_ready(self) -> bool:
        return True

    def close(self) -> None:
        pass


# ---------------------------------------------------------------------- module state + configuration
_kb: Optional[KnowledgeBase] = None
_kb_factory: Optional[Callable[[], KnowledgeBase]] = None
_state_lock = threading.Lock()


def configure(encoder=None, capacity: Optional[int] = None, device: Optional[int] = None, index_factory=None,
              factory: Optional[Callable[[], KnowledgeBase]] = None, dtype: Optional[str] = None) -> None:
    """Install the backend.  Environment: AURORA_B200_CAPACITY, AURORA_B200_DEVICE, AURORA_B200_DTYPE (the shard's row
    format: bf16, the default, or int8)."""
    global _kb, _kb_factory
    with _state_lock:
        _kb = None
        if factory is not None:
            _kb_factory = factory
            return
        cap = capacity if capacity is not None else int(os.getenv("AURORA_B200_CAPACITY", str(1 << 20)))
        dev = device if device is not None else int(os.getenv("AURORA_B200_DEVICE", "0"))
        dt = dtype if dtype is not None else os.getenv("AURORA_B200_DTYPE", "bf16")
        _kb_factory = lambda: KnowledgeBase(encoder, capacity=cap, device=dev, index_factory=index_factory, dtype=dt)  # noqa: E731


def _get_kb() -> KnowledgeBase:
    global _kb
    with _state_lock:
        if _kb is None:
            if _kb_factory is None:
                raise RuntimeError("aurora_b200.retriever is not configured: call configure(encoder=...) first")
            _kb = _kb_factory()
        return _kb


def _get_weaviate_client():
    """weaviate_client.py:35-101.  Returns (client, collection) façades; raises when the
    backend cannot be created (the reference raises on connection failure, :99-101)."""
    kb = _get_kb()
    return _ClientFacade(), _CollectionFacade(kb)


# ---------------------------------------------------------------------- public API (reference signatures)
def insert_chunks(user_id: str, document_id: str, source_filename: str, chunks: List[Dict[str, Any]],
                  org_id: str = None) -> int:
    """weaviate_client.py:136-212.  [] -> 0; returns inserted count; backend failure re-raises
    so the Celery task retries (tasks.py:100-111)."""
    if not chunks:
        return 0
    try:
        n = _get_kb().insert(user_id, document_id, source_filename, chunks, org_id)
        logger.info(f"[KB B200] Successfully inserted {n} chunks for doc {document_id}")
        return n
    except Exception as e:
        logger.error(f"[KB B200] Error inserting chunks: {e}")
        raise


def search_knowledge_base(user_id: str, query: str, limit: int = 5, alpha: float = 0.5, min_score: float = 0.0,
                          org_id: str = None) -> List[Dict[str, Any]]:
    """weaviate_client.py:215-285.  Blank query -> []; any exception -> log + [];
    scope = user_id == u OR org_id == o (:244-249); min_score applies only if > 0 (:266)."""
    if not query.strip():
        return []
    try:
        objs = _get_kb().query(query, limit, user_id=user_id, org_id=org_id, alpha=alpha, scoped=True)
        results = []
        for obj in objs:
            score = obj.metadata.score if obj.metadata else 0.0
            if min_score > 0.0 and score < min_score:
                continue
            p = obj.properties
            results.append({
                "content": p.get("content", ""),
                "heading_context": p.get("heading_context", ""),
                "source_filename": p.get("source_filename", ""),
                "document_id": p.get("document_id", ""),
                "chunk_index": p.get("chunk_index", 0),
                "score": score,
            })
        logger.info(f"[KB B200] Search for '{_sanitize(query)[:50]}...' returned {len(results)} results")
        return results
    except Exception as e:
        logger.error(f"[KB B200] Error searching: {e}")
        return []


def _shape_results(objs, min_score: float) -> List[Dict[str, Any]]:
    results = []
    for obj in objs:
        score = obj.metadata.score if obj.metadata else 0.0
        if min_score > 0.0 and score < min_score:
            continue
        p = obj.properties
        results.append({"content": p.get("content", ""), "heading_context": p.get("heading_context", ""),
                        "source_filename": p.get("source_filename", ""), "document_id": p.get("document_id", ""),
                        "chunk_index": p.get("chunk_index", 0), "score": score})
    return results


def search_knowledge_base_batch(requests: List[Tuple]) -> List[List[Dict[str, Any]]]:
    """Several ``search_knowledge_base`` calls answered together -- ``(user_id, query, limit, alpha, min_score, org_id)``
    each, same result per element as the single call (weaviate_client.py:215-285).  The engine daemon coalesces the
    concurrent calls of the reference's gunicorn threads into this (one encoder batch, one launch per tenant scope)."""
    out: List[List[Dict[str, Any]]] = [[] for _ in requests]
    live = [i for i, r in enumerate(requests) if isinstance(r[1], str) and r[1].strip()]
    if not live:
        return out
    try:
        reqs = [(requests[i][0], requests[i][1], requests[i][2], requests[i][3], requests[i][5]) for i in live]
        for i, objs in zip(live, _get_kb().query_batch(reqs)):
            out[i] = _shape_results(objs, requests[i][4])
    except Exception as e:
        logger.error(f"[KB B200] Error in batched search: {e}")
        return [[] for _ in requests]
    return out


def delete_document_chunks(user_id: str, document_id: str) -> int:
    """weaviate_client.py:288-319.  Deleted count; -1 on error."""
    try:
        return _get_kb().delete_where(lambda p: p.get("user_id") == user_id and p.get("document_id") == document_id)
    except Exception as e:
        logger.error(f"[KB B200] Error deleting chunks for doc {_sanitize(document_id)}: {_sanitize(e)}")
        return -1


def delete_user_chunks(user_id: str) -> int:
    """weaviate_client.py:322-344.  Deleted count; -1 on error."""
    try:
        return _get_kb().delete_where(lambda p: p.get("user_id") == user_id)
    except Exception as e:
        logger.error(f"[KB B200] Error deleting chunks for user {_sanitize(user_id)}: {_sanitize(e)}")
        return -1


def get_document_chunk_count(user_id: str, document_id: str) -> int:
    """weaviate_client.py:347-371.  0 on error."""
    try:
        return _get_kb().count_where(lambda p: p.get("user_id") == user_id and p.get("document_id") == document_id)
    except Exception as e:
        logger.error(f"[KB B200] Error getting chunk count: {e}")
        return 0


def delete_discovery_chunks(org_id: str, before: str = None) -> int:
    """weaviate_client.py:374-394: org_id == o AND document_id LIKE 'discovery:*'
    [AND created_at < before].  0 on error."""
    try:
        f = Filter.by_property("org_id").equal(org_id) & Filter.by_property("document_id").like("discovery:*")
        if before:
            f = f & Filter.by_property("created_at").less_than(before)
        return _get_kb().delete_where(f.matches)
    except Exception as e:
        logger.error(f"[KB B200] Error deleting discovery chunks: {e}")
        return 0

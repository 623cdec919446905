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
from typing import Any, Callable, Dict, List, NamedTuple, Optional, Tuple

import numpy as np

from . import bm25
from ._native import AUR_BF16, AUR_I8, FUSION_RANKED, FUSION_RELATIVE_SCORE
from .bm25 import BM25Index
from .filters import AttrColumn, Filter, HybridFusion, _Expr, compile_program  # noqa: F401  (Filter, HybridFusion: re-exported)

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


class _Request(NamedTuple):
    """One search as ``KnowledgeBase.query`` takes it (``fusion`` None already read as RANKED)."""
    text: str
    limit: int
    alpha: Optional[float]
    fusion: str
    filters: Any
    user: Optional[str]
    org: Optional[str]
    scoped: bool

    @property
    def searchable(self) -> bool:
        """False when the answer is [] without a search: no result asked for, or a tenant-facing search without a tenant."""
        return self.limit > 0 and bool(self.user or self.org or not self.scoped)

    @property
    def hybrid(self) -> bool:
        return self.alpha is not None and self.alpha < 1.0

    @property
    def dense_w(self) -> float:
        """The dense leg's weight: 1 for a vector search, else alpha (at least 0; 0 leaves the dense leg unsearched)."""
        return max(0.0, float(self.alpha)) if self.hybrid else 1.0


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
        # incremental checkpoints: what the last one left on disk (None: the next one writes a base) and, once a
        # checkpoint has captured, the objects upserted / deleted since its capture (id -> key)
        self._ckpt: Optional[Dict[str, Any]] = None
        self._ckpt_lock = threading.Lock()   # one checkpoint at a time
        self._tracking = False
        self._dirty_put: Dict[int, str] = {}
        self._dirty_del: Dict[int, Optional[str]] = {}

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
        is deterministic -- deletes name the object keys.  ``save`` truncates the log; ``checkpoint`` keeps only the records
        written after its capture.  Returns the replayed count."""
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
        # fused when the encoder appends to this index on the device: a CUDA Index, or a MultiIndex with an encoder on
        # every shard's GPU (TextEncoder.replicate); else encode, then index.add (CPU doubles, f32 shards)
        can_append = getattr(self.encoder, "can_append", None)
        fused = bool(can_append and can_append(self.index))
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
            self._make_room(ids)
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
                if self._tracking:
                    self._dirty_put[rid] = self._id2key.get(rid)
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

    def _make_room(self, ids: np.ndarray) -> None:
        """Grow every vector shard and keyword store that lacks room for these ids' rows before anything is appended,
        so the store keeps accepting chunks past the capacity it opened with (``engine.grow_for``)."""
        from .engine import grow_for

        grow_for(self.index, ids)
        store = getattr(self.sparse, "store", None) if self._kw_device else None
        if store is not None:
            grow_for(store, ids)

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
              fusion: str = HybridFusion.RANKED) -> List[SimpleNamespace]:
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
        req = _Request(query, limit, alpha, HybridFusion.RANKED if fusion is None else fusion, filters, user_id, org_id,
                       scoped)
        if req.searchable and req.fusion not in _FUSION:
            raise NotImplementedError(f"hybrid fusion {fusion!r}: only HybridFusion.RANKED and RELATIVE_SCORE are implemented")
        return self._search([req])[0]

    def query_batch(self, reqs: List[Tuple[Optional[str], str, int, Optional[float], Optional[str]]]) -> List[List[SimpleNamespace]]:
        """Several tenant-scoped searches at once: ``(user_id, query, limit, alpha, org_id)`` each, answered as ``query``
        answers them with ``scoped=True``.  All query texts go through ONE encoder batch; the dense leg is ONE kernel
        launch per result size (the tenant scopes of the batch ride along as per-row bit masks on the tensor-core kernel);
        on a GPU keyword store the keyword leg of every hybrid request (alpha < 1) is ONE device search with per-request
        tenant codes.  On a CUDA shard whose hybrid requests carry at most 32 distinct tenant scopes, those requests are
        instead ONE device call for both legs and their ranked fusion (``DeviceBM25.search_batch`` with ``dense``,
        per-request weights), and only shaping is left per request."""
        return self._search([_Request(q, lim, a, HybridFusion.RANKED, None, u, o, True) for u, q, lim, a, o in reqs])

    def _search(self, reqs: List[_Request]) -> List[List[SimpleNamespace]]:
        """The answers to ``reqs``.  Encode every dense leg in one call; under the lock resolve each request's scope;
        answer on the device the hybrid requests that fuse there, one call per kind of scope and fusion; search the other
        requests' legs, batched per kind of scope (and result size for the dense leg); fuse and shape on the host."""
        live = [i for i, r in enumerate(reqs) if r.searchable]
        enc = [i for i in live if reqs[i].dense_w > 0.0]
        vecs = self.encoder.encode([reqs[i].text for i in enc]) if enc else None
        row = {i: j for j, i in enumerate(enc)}
        out: List[List[SimpleNamespace]] = [[] for _ in reqs]
        with self._lock:
            scope = {i: self._resolve_scope(reqs[i]) for i in live}
            fused: Dict[int, list] = {}
            calls: Dict[tuple, List[int]] = {}
            for i in live:
                if reqs[i].hybrid and self._hybrid_device and scope[i][0] != "ids":
                    calls.setdefault((scope[i][0], reqs[i].fusion), []).append(i)
            for (kind, fusion), g in calls.items():
                vals = [scope[i][1] for i in g]
                if kind == "codes" and len(set(vals)) > 32:   # more than the tensor-core kernel's per-row scope masks hold
                    continue
                hv = np.zeros((len(g), self.dim), vecs.dtype if vecs is not None else np.float32)
                for j, i in enumerate(g):
                    if i in row:            # alpha <= 0: the dense leg is ignored, its vector stays zero
                        hv[j] = vecs[row[i]]
                w = np.array([reqs[i].dense_w for i in g])
                lists = self.sparse.search_batch([reqs[i].text for i in g], _MAX_FETCH, **self._scope_args(kind, vals),
                                                 dense=(self.index, hv, w, _FUSION[fusion],
                                                        min(max(reqs[i].limit for i in g), 2 * _MAX_FETCH)))
                fused.update(zip(g, lists))

            groups: Dict[tuple, List[int]] = {}     # (fetch size, kind of scope, request of an allow-list) -> requests
            for i in live:
                kind, val = scope[i]
                if i in row and i not in fused and (kind != "ids" or val):
                    fetch = max(1, min(_MAX_FETCH, _MAX_FETCH if reqs[i].hybrid else reqs[i].limit))
                    groups.setdefault((fetch, kind, i if kind == "ids" else None), []).append(i)
            dense: Dict[int, List[Tuple[int, float]]] = {}
            for (fetch, kind, _), g in groups.items():
                q, vals = vecs[[row[i] for i in g]], [scope[i][1] for i in g]
                if kind == "ids":
                    allowed = np.asarray(vals[0], dtype=np.int64)
                    if hasattr(self.index, "search_lists") and len(allowed) <= _LIST_MAX_FRACTION * len(self._props):
                        ids, scores = self.index.search_lists(q, fetch, [allowed], np.zeros(1, np.int32))  # reads only those rows
                    else:
                        ids, scores = self.index.search_subset(q, fetch, allowed)
                elif kind == "program":     # no id crosses PCIe; the list-vs-scan rule is the host path's
                    ids, scores, _, _ = self.index.search_filtered(q, fetch, **self._scope_args(kind, vals))
                elif kind == "codes" and len(set(vals)) > 32 and hasattr(self.index, "search_lists"):
                    # more scopes than the tensor-core kernel's row bit masks hold: one id list per scope (the rows
                    # _tenant_scope gives the keyword leg) and one list search that reads only those rows
                    slots: Dict[Tuple[int, int], int] = {}
                    lists = []
                    for i, v in zip(g, vals):
                        if v not in slots:
                            slots[v] = len(slots)
                            lists.append(self._tenant_scope(reqs[i].user, reqs[i].org)[1])
                    ids, scores = self.index.search_lists(q, fetch, lists, np.array([slots[v] for v in vals], np.int32))
                else:
                    # one launch for the whole group: up to 32 distinct tenant scopes per batch ride on the tensor-core
                    # kernel as per-row bit masks (csrc/capi.cu stage_tenant_scope); the library falls back by itself beyond
                    ids, scores = self.index.search(q, fetch, **self._scope_args(kind, vals))
                for i, r_ids, r_scores in zip(g, ids, scores):
                    dense[i] = [(int(d), float(s)) for d, s in zip(r_ids, r_scores) if d >= 0]

            # keyword leg under the same pre-filter: a program's or the filter's ids, else the tenant scope (on the device
            # by codes, as the dense leg applies it; on the host by the tenant's own inverted lists)
            sparse: Dict[int, List[Tuple[int, float]]] = {}
            kw_calls: Dict[str, List[int]] = {}
            for i in live:
                if not reqs[i].hybrid or i in fused:
                    continue
                kind, val = scope[i]
                if kind == "program":       # only beside a keyword leg that cannot evaluate it (the others fused above)
                    kind, val = "ids", self.index.filter_ids(val).tolist()
                if kind == "ids":
                    sparse[i] = self.sparse.search(reqs[i].text, _MAX_FETCH,
                                                   allowed=val if self._kw_device else set(val))
                elif self._kw_device:
                    kw_calls.setdefault(kind, []).append(i)
                else:
                    allowed_set, allowed_arr = self._tenant_scope(reqs[i].user, reqs[i].org) if kind == "codes" else (None, None)
                    sparse[i] = self.sparse.search(reqs[i].text, _MAX_FETCH, allowed=allowed_set, allowed_sorted=allowed_arr)
            for kind, g in kw_calls.items():
                sparse.update(zip(g, self.sparse.search_batch([reqs[i].text for i in g], _MAX_FETCH,
                                                              **self._scope_args(kind, [scope[i][1] for i in g]))))

            # objects deleted since a leg's search (the keyword store's own call may delete) drop out of the answer
            for i in live:
                r = reqs[i]
                if i in fused:              # the device's scores: the answer as of the search
                    out[i] = self._shape([(d, fs, cos) for d, (fs, cos) in fused[i] if d in self._props][:r.limit])
                    continue
                d_leg = [(d, s) for d, s in dense.get(i, []) if d in self._props]
                if not r.hybrid:
                    out[i] = self._shape([(d, s, s) for d, s in d_leg[:r.limit]])
                    continue
                s_leg = [(d, s) for d, s in sparse[i] if d in self._props]
                if r.fusion == HybridFusion.RELATIVE_SCORE:
                    picked = bm25.relative_score_fusion([(r.dense_w, d_leg), (1.0 - r.dense_w, s_leg)], r.limit)
                else:
                    picked = bm25.ranked_fusion([(r.dense_w, [d for d, _ in d_leg]),
                                                 (1.0 - r.dense_w, [d for d, _ in s_leg])], r.limit)
                cos = dict(d_leg)
                out[i] = self._shape([(d, fs, cos.get(d)) for d, fs in picked])
        return out

    def _resolve_scope(self, r: _Request):
        """The rows ``r`` may see, as ``(kind, value)``: ``("all", None)``, ``("codes", (user code, org code))``,
        ``("program", device program)`` or ``("ids", allowed id list)`` (a filter resolved on the host).  Caller holds
        the lock."""
        tenant = r.scoped or r.user is not None or r.org is not None
        if r.filters is None:
            return ("codes", self._scope_codes(r.user, r.org)) if tenant else ("all", None)
        prog = self._device_program(r.filters, tenant, r.user, r.org)
        if prog is not None:
            return "program", prog
        # narrow the scan with the filter's own equality terms and the tenant scope, then run the predicate
        eq = r.filters.required_equalities()
        pools = []
        if "org_id" in eq:
            pools.append(self._by_org.get(eq["org_id"], set()))
        if "user_id" in eq:
            pools.append(self._by_user.get(eq["user_id"], set()))
        if tenant:
            pools.append(self._by_user.get(r.user, set()) | (self._by_org.get(r.org, set()) if r.org else set()))
        cand = set.intersection(*pools) if pools else self._props.keys()

        def tenant_ok(props) -> bool:
            return not tenant or (bool(r.user) and props.get("user_id") == r.user) or \
                (bool(r.org) and props.get("org_id") == r.org)
        return "ids", [rid for rid in cand if r.filters.matches(self._props[rid]) and tenant_ok(self._props[rid])]

    def _scope_args(self, kind: str, vals: list) -> Dict[str, Any]:
        """The scopes of one batch of a kind as the index's and the keyword store's searches take them.  Caller holds
        the lock."""
        if kind == "codes":
            return {"q_user": np.array([v[0] for v in vals], np.int32), "q_org": np.array([v[1] for v in vals], np.int32)}
        if kind == "program":               # q_program None: every query on program 0
            return {"programs": vals, "q_program": np.arange(len(vals), dtype=np.int32) if len(vals) > 1 else None,
                    "max_list_rows": int(_LIST_MAX_FRACTION * len(self._props))}
        return {}

    def _shape(self, picked) -> List[SimpleNamespace]:
        """(id, score, dense cosine or None) -> result objects.  Caller holds the lock."""
        out = []
        for rid, score, cosine in picked:
            meta = SimpleNamespace(score=float(score), distance=None if cosine is None else 1.0 - float(cosine))
            out.append(SimpleNamespace(properties=dict(self._props[rid]), uuid=self._id2key.get(rid), metadata=meta))
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
            if self._ckpt is not None and self._ckpt["dir"] == os.path.abspath(directory):
                self._ckpt_reset()                  # the directory no longer holds the checkpoint's base
            if self._wal is not None:               # everything logged so far is inside the snapshot: start a fresh log.
                self._wal.close()                   # (a crash before this point leaves old records; replay skips them by gen)
                tmp_wal = self._wal_path + ".tmp"
                open(tmp_wal, "w").close()
                os.replace(tmp_wal, self._wal_path)
                self._wal = open(self._wal_path, "a", encoding="utf-8")

    def _ckpt_reset(self) -> None:
        """The next checkpoint writes a base; nothing is tracked until it captures.  Caller holds the lock or owns the
        store alone."""
        self._ckpt, self._tracking = None, False
        self._dirty_put, self._dirty_del = {}, {}

    def checkpoint(self, directory: str, on_stage: Optional[Callable[[str], None]] = None) -> Dict[str, Any]:
        """Durable snapshot like ``save``, but incremental and without pausing the store (DESIGN.md section 8,
        "Snapshots").  Under the lock only the change is captured: every shard's row count, live bitmap and compaction
        count (``Index.capture``), the objects upserted and deleted since the last checkpoint, and the mutation log's
        length.  Outside it the rows appended since the last checkpoint are read (``Index.export_rows``) and written with
        the bitmaps as one delta file per shard plus the metadata delta, then the manifest ``meta.json`` is renamed into
        place; searches, inserts and deletes go on meanwhile.  Last, under the lock again, the log keeps only the records
        written after the capture.

        A base (every live row and the whole property table) is written instead when there is none yet in this
        directory from this store, a shard was compacted since the last capture, the rows appended since the base exceed
        a quarter of its rows, or more than 16 deltas would be on disk.  ``on_stage(name)`` is called after the capture
        ("captured"), once the segment files are durable ("segment"), once the manifest is ("manifest") and before the log
        is trimmed ("trim").  Returns {"kind": "base" | "delta", "generation", "bytes", "locked_ms", "seconds"}."""
        os.makedirs(directory, exist_ok=True)
        directory = os.path.abspath(directory)
        with self._ckpt_lock:
            for _ in range(4):     # a compaction that lands between capture and copy discards the segment: retry as a base
                res = self._checkpoint_once(directory, on_stage or (lambda stage: None))
                if res is not None:
                    return res
            raise RuntimeError("checkpoint: every attempt raced a compaction")

    def _checkpoint_once(self, directory: str, on_stage) -> Optional[Dict[str, Any]]:
        import json
        import time

        from . import checkpoint as K

        t0 = time.perf_counter()
        with self._lock:
            t_lock = time.perf_counter()
            st = self._ckpt
            if st is None or st["dir"] != directory or st["shards"].index is not self.index:
                st = None
            shards = st["shards"] if st else K.Shards(self.index)
            caps = shards.capture()
            gen = int(self.mutations)
            base = (st is None or any(c[3] != k for c, k in zip(caps, st["compactions"]))
                    or sum(c[0] - m for c, m in zip(caps, st["base_marks"])) > K.MAX_DELTA_FRACTION * st["base_entries"]
                    or len(st["meta"]["deltas"]) + 1 > K.MAX_DELTAS)
            if base:
                objs = (dict(self._props), dict(self._id2key))          # shallow: property dicts are replaced, never edited
            else:
                objs = ([(rid, key, self._props[rid]) for rid, key in self._dirty_put.items()], list(self._dirty_del.items()))
            self._tracking = True
            self._dirty_put, self._dirty_del = {}, {}
            codes = (dict(self._user_code), dict(self._org_code), int(self._next_id))
            wal_off = None
            if self._wal is not None:
                self._wal.flush()
                wal_off = os.fstat(self._wal.fileno()).st_size
            locked_ms = (time.perf_counter() - t_lock) * 1e3
        try:
            on_stage("captured")
            ranges = [(0, c[0]) if base else (m, c[0] - m) for c, m in zip(caps, [0] * len(caps) if base else st["marks"])]
            data = shards.export_rows(ranges)
            if any(a[3] != c[3] for a, c in zip(shards.capture(), caps)):
                self._ckpt = None           # renumbered while the rows were read: what was read is discarded
                return None
            tag = K.new_tag(gen)
            written = 0
            # only the rows live at capture: a row dead then never comes back, so nothing later needs it
            keep = [K.bits_at(c[1], np.arange(r0, r0 + n)) for c, (r0, n) in zip(caps, ranges)]
            if base:
                props, id2key = objs
                part = np.concatenate([np.full(int(k.sum()), s, np.int32) for s, k in enumerate(keep)])
                row = np.concatenate([np.arange(r0, r0 + n, dtype=np.int64)[k] for (r0, n), k in zip(ranges, keep)])
                ids = np.concatenate([d[1][k] for d, k in zip(data, keep)])
                nonfinite = np.concatenate([K.bits_at(c[2], np.arange(r0, r0 + n))[k]
                                            for c, (r0, n), k in zip(caps, ranges, keep)])
                shard_name = f"shard.{gen}.npz"
                written += K.write_npz(os.path.join(directory, shard_name),
                                       rows=np.concatenate([d[0][k] for d, k in zip(data, keep)]), ids=ids,
                                       user=np.concatenate([d[2][k] for d, k in zip(data, keep)]),
                                       org=np.concatenate([d[3][k] for d, k in zip(data, keep)]), nonfinite=nonfinite,
                                       dim=self.dim, dtype=getattr(self.index, "dtype", AUR_BF16),
                                       capacity=int(getattr(self.index, "capacity", len(ids))))
                seg = {"tag": tag, "rows": f"base.{tag}.npz", "meta": f"base.{tag}.jsonl", "entries": int(len(ids))}
                written += K.write_npz(os.path.join(directory, seg["rows"]), ids=ids, part=part, row=row)
                written += K.write_jsonl(os.path.join(directory, seg["meta"]),
                                         ([rid, id2key.get(rid), p] for rid, p in props.items()))
                meta_base, deltas = seg, []
            else:
                puts, dels = objs
                seg = {"tag": tag, "generation": gen, "shards": [f"delta.{tag}.{s}.npz" for s in range(len(caps))],
                       "meta": f"delta.{tag}.jsonl"}
                for s, (c, (r0, n), d, k) in enumerate(zip(caps, ranges, data, keep)):
                    written += K.write_npz(os.path.join(directory, seg["shards"][s]), rows=d[0][k], ids=d[1][k],
                                           user=d[2][k], org=d[3][k],
                                           nonfinite=K.bits_at(c[2], np.arange(r0, r0 + n))[k],
                                           row=np.arange(r0, r0 + n, dtype=np.int64)[k], live=c[1], nonfinite_bits=c[2],
                                           rows_total=c[0])
                written += K.write_jsonl(os.path.join(directory, seg["meta"]),
                                         [["put", rid, key, p] for rid, key, p in puts] + [["del", rid, key] for rid, key in dels])
                shard_name, meta_base, deltas = st["meta"]["shard"], st["meta"]["base"], st["meta"]["deltas"] + [seg]
            K.fsync_dir(directory)
            on_stage("segment")
            user_code, org_code, next_id = codes
            meta = {"shard": shard_name, "version": 2, "generation": gen, "dim": self.dim, "next_id": next_id,
                    "user_code": user_code, "org_code": org_code, "parts": len(caps), "base": meta_base, "deltas": deltas}
            path = os.path.join(directory, "meta.json")
            written += K.write_file(path, lambda f: f.write(json.dumps(meta).encode("utf-8")))
            K.fsync_dir(directory)
            self.saved_mutations = max(self.saved_mutations, gen)
            on_stage("manifest")
            K.remove_unreferenced(directory, meta)
            self._ckpt = {"dir": directory, "shards": shards, "meta": meta, "marks": [c[0] for c in caps],
                          "compactions": [c[3] for c in caps],
                          "base_marks": [c[0] for c in caps] if base else st["base_marks"],
                          "base_entries": meta_base["entries"]}
            on_stage("trim")
            with self._lock:
                t_trim = time.perf_counter()
                self._trim_wal(wal_off)
                locked_ms += (time.perf_counter() - t_trim) * 1e3
        except BaseException:
            with self._lock:
                self._ckpt_reset()          # the next checkpoint starts over from a base
            raise
        return {"kind": "base" if base else "delta", "generation": gen, "bytes": int(written),
                "locked_ms": round(locked_ms, 3), "seconds": round(time.perf_counter() - t0, 3)}

    def _trim_wal(self, offset: Optional[int]) -> None:
        """Keep only the log's bytes from ``offset`` on (the records written after a checkpoint's capture), under the
        same file name.  Caller holds the lock."""
        from .checkpoint import fsync_dir

        if self._wal is None or offset is None:
            return
        self._wal.flush()
        with open(self._wal_path, "rb") as f:
            f.seek(offset)
            tail = f.read()
        tmp = self._wal_path + ".tmp"
        with open(tmp, "wb") as f:
            f.write(tail)
            f.flush()
            os.fsync(f.fileno())
        self._wal.close()
        os.replace(tmp, self._wal_path)
        fsync_dir(os.path.dirname(os.path.abspath(self._wal_path)))
        self._wal = open(self._wal_path, "a", encoding="utf-8")

    @classmethod
    def load(cls, directory: str, encoder, capacity: int = 1 << 20, device: int = 0, index_loader=None,
             text_of: Optional[Callable[[Dict[str, Any]], str]] = None) -> "KnowledgeBase":
        """Rebuild from ``save`` or ``checkpoint``: vectors go back into HBM as they were stored (no re-encoding), the
        keyword index is rebuilt from the chunk texts.  A checkpoint's base goes through ``index_loader``, its deltas
        through the loaded index's own ``remove`` and ``add``; the store's next checkpoint writes a new base."""
        import json

        from . import checkpoint as K

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
        if "base" in meta:
            K.apply_deltas(loaded, directory, meta)
            props, key2id = K.read_objects(directory, meta)
        else:
            props, key2id = {int(k): v for k, v in meta["props"].items()}, meta["key2id"]
        kb = cls(encoder, capacity=capacity, device=device, index_factory=lambda dim, cap: loaded)
        kb._next_id = int(meta["next_id"])
        kb.mutations = kb.saved_mutations = int(meta.get("generation", 0))     # the log's records are ordered by it
        kb._user_code = {k: int(v) for k, v in meta["user_code"].items()}
        kb._org_code = {k: int(v) for k, v in meta["org_code"].items()}
        kb._key2id = {k: int(v) for k, v in key2id.items()}
        kb._id2key = {v: k for k, v in kb._key2id.items()}
        kb._props = props
        for rid, p in kb._props.items():
            kb._by_user.setdefault(p.get("user_id"), set()).add(rid)
            if p.get("org_id"):
                kb._by_org.setdefault(p["org_id"], set()).add(rid)
            if not kb._kw_device:
                kb.sparse.add(rid, text_of(p))
        if kb._kw_device and kb._props:     # one device append for the whole store
            rids = list(kb._props)
            from .engine import grow_for

            grow_for(kb.sparse.store, rids)   # (the index loader made room for the vectors it added)
            kb.sparse.add_many(rids, [text_of(kb._props[r]) for r in rids],
                               np.array([kb._code(kb._user_code, kb._props[r].get("user_id"), False) for r in rids], np.int32),
                               np.array([kb._code(kb._org_code, kb._props[r].get("org_id"), False) for r in rids], np.int32))
        return kb

    # ------------------------------------------------------------------ deletes / counts
    def _delete_program(self, pred):
        """``pred`` as a device program for ``remove_filtered`` / ``count_filtered``, or None when it is resolved by the
        host scan: a plain predicate (not a ``Filter`` expression), an index without those calls (CPU doubles, a
        ``MultiIndex`` of them), or whatever keeps ``_device_program`` on the host.  Caller holds the lock."""
        shards = getattr(self.index, "shards", [self.index])
        if not isinstance(pred, _Expr) or not all(hasattr(sh, "remove_filtered") for sh in [self.index, *shards]):
            return None
        return self._device_program(pred, False, None, None)

    def _matching_ids(self, pred) -> List[int]:
        match = pred.matches if isinstance(pred, _Expr) else pred
        return [rid for rid, p in self._props.items() if match(p)]

    def delete_where(self, pred) -> int:
        """Delete the objects ``pred`` matches (a ``Filter`` expression or a predicate over the properties); returns how
        many.  An expression that compiles to a device program is resolved on the GPU, so host work follows the matching
        objects, not the store's size."""
        with self._lock:
            prog = self._delete_program(pred)
            if prog is None:
                return self._delete_ids(self._matching_ids(pred))
            ids = [int(r) for r in self.index.remove_filtered(prog)]
            if ids:
                self._forget_ids(ids)
            return len(ids)

    def _delete_ids(self, ids: List[int]) -> int:
        with self._lock:
            if ids:
                self.index.remove(np.array(ids, dtype=np.int64))
                self._forget_ids(ids)
            return len(ids)

    def _forget_ids(self, ids: List[int]) -> None:
        """Everything but the vector shard's rows of deleted objects: the keyword store's, their properties and keys, the
        mutation count and the log record.  Caller holds the lock."""
        gen = self.mutations
        keys = [self._id2key.get(rid) for rid in ids]
        if self._kw_device:
            self.sparse.remove_many(ids)
        for rid, key in zip(ids, keys):
            p = self._props.pop(rid)
            if self._tracking:
                self._dirty_put.pop(rid, None)
                self._dirty_del[rid] = key
            self._unindex(rid, p)
            if not self._kw_device:
                self.sparse.remove(rid)
            self._key2id.pop(self._id2key.pop(rid, None), None)
        self.mutations += len(ids)
        self._log({"op": "del", "gen": gen, "keys": [k for k in keys if k]})

    def count_where(self, pred) -> int:
        """How many objects ``pred`` matches; counted on the GPU under the same rule as ``delete_where``."""
        with self._lock:
            prog = self._delete_program(pred)
            return len(self._matching_ids(pred)) if prog is None else self.index.count_filtered(prog)


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
    """Install the backend.  Environment: AURORA_B200_CAPACITY (the initial capacity: the shards grow as chunks arrive),
    AURORA_B200_DEVICE, AURORA_B200_DTYPE (the shard's row format: bf16, the default, or int8)."""
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
        results = _shape_results(_get_kb().query(query, limit, user_id=user_id, org_id=org_id, alpha=alpha, scoped=True),
                                 min_score)
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
        return _get_kb().delete_where(Filter.by_property("user_id").equal(user_id)
                                      & Filter.by_property("document_id").equal(document_id))
    except Exception as e:
        logger.error(f"[KB B200] Error deleting chunks for doc {_sanitize(document_id)}: {_sanitize(e)}")
        return -1


def delete_user_chunks(user_id: str) -> int:
    """weaviate_client.py:322-344.  Deleted count; -1 on error."""
    try:
        return _get_kb().delete_where(Filter.by_property("user_id").equal(user_id))
    except Exception as e:
        logger.error(f"[KB B200] Error deleting chunks for user {_sanitize(user_id)}: {_sanitize(e)}")
        return -1


def get_document_chunk_count(user_id: str, document_id: str) -> int:
    """weaviate_client.py:347-371.  0 on error."""
    try:
        return _get_kb().count_where(Filter.by_property("user_id").equal(user_id)
                                     & Filter.by_property("document_id").equal(document_id))
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
        return _get_kb().delete_where(f)
    except Exception as e:
        logger.error(f"[KB B200] Error deleting discovery chunks: {e}")
        return 0

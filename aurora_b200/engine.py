"""Python handle over one corpus shard in HBM (the C ABI of include/aurora_b200.h).

numpy in / numpy out for the host entry points; ``*_dev`` methods take raw device
pointers (``tensor.data_ptr()``) so torch is only plumbing for memory and streams.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import _native as N


def to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bit patterns (uint16), round-to-nearest-even.  Host-side format
    conversion of inputs only; no scoring happens on the CPU."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))
    return (r >> np.uint32(16)).astype(np.uint16)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Index:
    """One row-shard of the corpus, resident on one GPU."""

    def __init__(self, dim: int, capacity: int, dtype: str = "bf16", device: int = 0):
        self._lib = N.load()
        self.dim, self.capacity, self.device = int(dim), int(capacity), int(device)
        self.dtype = {"bf16": N.AUR_BF16, "f32": N.AUR_F32}[dtype]
        self._h = C.c_void_p()
        cfg = N.AurConfig(device=self.device, dim=self.dim, dtype=self.dtype, reserved=0, capacity=self.capacity)
        N.check(self._lib.aur_open(C.byref(cfg), C.byref(self._h)))

    # -------------------------------------------------------------- lifecycle
    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.aur_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -------------------------------------------------------------- helpers
    def _rows_buffer(self, x: np.ndarray) -> np.ndarray:
        x = np.asarray(x)
        if x.ndim != 2 or x.shape[1] != self.dim:
            raise ValueError(f"expected [n, {self.dim}] rows, got {x.shape}")
        if self.dtype == N.AUR_BF16:
            if x.dtype == np.uint16:
                return np.ascontiguousarray(x)
            return to_bf16_bits(x)
        return np.ascontiguousarray(x, dtype=np.float32)

    # -------------------------------------------------------------- ingest
    def add(self, rows: np.ndarray, ids: np.ndarray, user_codes: Optional[np.ndarray] = None,
            org_codes: Optional[np.ndarray] = None) -> None:
        buf = self._rows_buffer(rows)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.shape != (buf.shape[0],):
            raise ValueError("ids must be [n]")
        u = None if user_codes is None else np.ascontiguousarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.ascontiguousarray(org_codes, dtype=np.int32)
        N.check(self._lib.aur_add(self._h, _ptr(buf), _ptr(ids), _ptr(u), _ptr(o), buf.shape[0]))

    def add_dev(self, rows_ptr: int, n: int, ids: np.ndarray, user_codes=None, org_codes=None, stream: int = 0) -> None:
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        u = None if user_codes is None else np.ascontiguousarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.ascontiguousarray(org_codes, dtype=np.int32)
        N.check(self._lib.aur_add_dev(self._h, C.c_void_p(rows_ptr), _ptr(ids), _ptr(u), _ptr(o), int(n),
                                      C.c_void_p(stream)))

    def remove(self, ids) -> int:
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        removed = C.c_int64(0)
        N.check(self._lib.aur_remove(self._h, _ptr(ids), ids.shape[0], C.byref(removed)))
        return int(removed.value)

    # -------------------------------------------------------------- snapshot
    def export(self):
        """All appended rows in append order: (rows [n, dim] uint16 bf16 bits or float32, ids, user codes,
        org codes, live mask).  Tombstoned rows are included with live = False."""
        n = self.stats()["rows"]
        rows = np.empty((n, self.dim), dtype=np.uint16 if self.dtype == N.AUR_BF16 else np.float32)
        ids = np.empty(n, dtype=np.int64)
        user, org = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        live = np.empty(n, dtype=np.uint8)
        N.check(self._lib.aur_export(self._h, _ptr(rows), _ptr(ids), _ptr(user), _ptr(org), _ptr(live), n))
        return rows, ids, user, org, live.astype(bool)

    def save(self, path: str) -> None:
        """Snapshot of the live rows (tombstones are compacted away) as one .npz file."""
        rows, ids, user, org, live = self.export()
        np.savez(path, rows=rows[live], ids=ids[live], user=user[live], org=org[live], dim=self.dim,
                 dtype=self.dtype, capacity=self.capacity)

    @classmethod
    def load(cls, path: str, capacity: Optional[int] = None, device: int = 0) -> "Index":
        z = np.load(path if path.endswith(".npz") else path + ".npz")
        dtype = "bf16" if int(z["dtype"]) == N.AUR_BF16 else "f32"
        ix = cls(int(z["dim"]), int(capacity or z["capacity"]), dtype=dtype, device=device)
        if len(z["ids"]):
            ix.add(z["rows"], z["ids"], z["user"], z["org"])
        return ix

    # -------------------------------------------------------------- search
    def search(self, queries: np.ndarray, k: int, q_user: Optional[np.ndarray] = None,
               q_org: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
        """Host buffers in, host buffers out: (ids [nq,k] int64, scores [nq,k] float32)."""
        q = self._rows_buffer(queries)
        nq = q.shape[0]
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        u = None if q_user is None else np.ascontiguousarray(q_user, dtype=np.int32)
        o = None if q_org is None else np.ascontiguousarray(q_org, dtype=np.int32)
        N.check(self._lib.aur_search(self._h, _ptr(q), nq, int(k), _ptr(u), _ptr(o), _ptr(scores), _ptr(ids)))
        return ids, scores

    def search_snapshot(self, queries: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray, int]:
        """(ids, scores, snapshot_rows): the search together with the number of appended rows it saw -- with a
        concurrent writer the answer is the top-k of exactly that prefix."""
        q = self._rows_buffer(queries)
        nq = q.shape[0]
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        snap = C.c_int64(-1)
        N.check(self._lib.aur_search_ex(self._h, _ptr(q), nq, int(k), None, None, _ptr(scores), _ptr(ids), C.byref(snap)))
        return ids, scores, int(snap.value)

    def read_rows(self, row0: int, n: int):
        """(rows [n, dim] uint16 bf16 bits or float32, ids [n]) of appended rows row0 .. row0 + n."""
        rows = np.empty((n, self.dim), dtype=np.uint16 if self.dtype == N.AUR_BF16 else np.float32)
        ids = np.empty(n, dtype=np.int64)
        N.check(self._lib.aur_read_rows(self._h, int(row0), int(n), _ptr(rows), _ptr(ids)))
        return rows, ids

    def compact(self) -> int:
        """Reclaim tombstoned rows (exclusive; waits for searches in flight).  Returns the rows freed."""
        freed = C.c_int64(0)
        N.check(self._lib.aur_compact(self._h, C.byref(freed)))
        return int(freed.value)

    def search_subset(self, queries: np.ndarray, k: int, allow_ids: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """Search restricted to the rows whose ids are listed (a resolved metadata pre-filter): the other rows'
        inverse norms are masked on the device and the same kernels run."""
        q = self._rows_buffer(queries)
        nq = q.shape[0]
        allow = np.ascontiguousarray(allow_ids, dtype=np.int64)
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        N.check(self._lib.aur_search_subset(self._h, _ptr(q), nq, int(k), _ptr(allow), allow.shape[0], _ptr(scores), _ptr(ids)))
        return ids, scores

    def search_lists(self, queries: np.ndarray, k: int, lists, q_list) -> Tuple[np.ndarray, np.ndarray]:
        """Search with a pre-filter per query: query q sees only the rows whose ids are in ``lists[q_list[q]]`` (a
        sequence of id arrays; several queries may name the same list).  Only the listed rows are read, so the cost
        follows the lists' sizes, not the shard's.  bf16 indexes.  Returns (ids [nq,k] int64, scores [nq,k] float32)."""
        ids, scores, _ = self.search_lists_snapshot(queries, k, lists, q_list)
        return ids, scores

    def search_lists_snapshot(self, queries: np.ndarray, k: int, lists, q_list):
        """``search_lists`` together with the number of appended rows it saw (see ``search_snapshot``)."""
        q = self._rows_buffer(queries)
        nq = q.shape[0]
        flat, offsets = lists_csr(lists)
        ql = np.ascontiguousarray(q_list, dtype=np.int32)
        if ql.shape != (nq,):
            raise ValueError("q_list must be [nq]")
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        snap = C.c_int64(-1)
        N.check(self._lib.aur_search_lists(self._h, _ptr(q), nq, int(k), _ptr(flat), _ptr(offsets), len(offsets) - 1,
                                           _ptr(ql), _ptr(scores), _ptr(ids), C.byref(snap)))
        return ids, scores, int(snap.value)

    # -------------------------------------------------------------- device-evaluated filters
    def set_attrs(self, col: int, ids, codes) -> None:
        """Attribute column ``col`` (2 .. 17) of the rows ``ids`` := ``codes`` (int32, -1 = absent); unknown ids are
        ignored.  The column starts all absent on first use."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        codes = np.ascontiguousarray(codes, dtype=np.int32)
        if codes.shape != ids.shape:
            raise ValueError("ids and codes must have the same length")
        N.check(self._lib.aur_set_attrs(self._h, int(col), _ptr(ids), _ptr(codes), ids.shape[0]))

    def search_filtered(self, queries: np.ndarray, k: int, programs, q_program=None, max_list_rows: int = 0):
        """Search with pre-filters evaluated on the device: query q sees the live rows ``programs[q_program[q]]`` matches
        (``filters.compile_program`` outputs, at most 32; ``q_program`` None = every query on program 0).  One program
        matching more than ``max_list_rows`` rows runs the masked full scan, anything else the list kernels.  Returns
        (ids [nq,k] int64, scores [nq,k] float32, matching rows per program int64, snapshot rows)."""
        from .filters import pack_programs

        q = self._rows_buffer(queries)
        nq = q.shape[0]
        tok, off, bm = pack_programs(programs)
        ql = np.zeros(nq, np.int32) if q_program is None else np.ascontiguousarray(q_program, dtype=np.int32)
        if ql.shape != (nq,):
            raise ValueError("q_program must be [nq]")
        scores = np.empty((nq, k), dtype=np.float32)
        ids = np.empty((nq, k), dtype=np.int64)
        matched = np.zeros(len(programs), dtype=np.int64)
        snap = C.c_int64(-1)
        N.check(self._lib.aur_search_filtered(self._h, _ptr(q), nq, int(k), _ptr(tok), _ptr(off), len(programs), _ptr(bm),
                                              bm.shape[0], _ptr(ql), int(max_list_rows), _ptr(scores), _ptr(ids),
                                              _ptr(matched), C.byref(snap)))
        return ids, scores, matched, int(snap.value)

    def filter_ids(self, program) -> np.ndarray:
        """Ids of the live rows one ``filters.compile_program`` program matches, in row order."""
        from .filters import pack_programs

        tok, _, bm = pack_programs([program])
        cap = 1 << 16
        while True:                 # the call reports the count: one retry with room for every match (more if rows arrive)
            out = np.empty(cap, dtype=np.int64)
            n = C.c_int64(0)
            N.check(self._lib.aur_filter_ids(self._h, _ptr(tok), tok.shape[0], _ptr(bm), bm.shape[0], _ptr(out), cap,
                                             C.byref(n)))
            if n.value <= cap:
                return out[:n.value]
            cap = int(n.value)

    def search_dev(self, q_ptr: int, nq: int, k: int, scores_ptr: int, ids_ptr: int, scores64_ptr: int = 0,
                   q_user_ptr: int = 0, q_org_ptr: int = 0, stream: int = 0) -> None:
        """Everything in HBM; asynchronous on ``stream`` (0 = the index's own stream)."""
        N.check(self._lib.aur_search_dev(self._h, C.c_void_p(q_ptr), int(nq), int(k), C.c_void_p(q_user_ptr),
                                         C.c_void_p(q_org_ptr), C.c_void_p(scores_ptr), C.c_void_p(ids_ptr),
                                         C.c_void_p(scores64_ptr), C.c_void_p(stream)))

    def debug_tc_scores(self, q_ptr: int, nq: int, cta_group: int, out_ptr: int, stream: int = 0) -> int:
        n = C.c_int32(0)
        N.check(self._lib.aur_debug_tc_scores(self._h, C.c_void_p(q_ptr), int(nq), int(cta_group),
                                              C.c_void_p(out_ptr), C.byref(n), C.c_void_p(stream)))
        return int(n.value)

    # -------------------------------------------------------------- misc
    def set_kernel(self, kernel: int) -> None:
        N.check(self._lib.aur_set_option(self._h, b"kernel", int(kernel)))

    def sync(self) -> None:
        N.check(self._lib.aur_sync(self._h))

    def stats(self) -> dict:
        st = N.AurStats()
        N.check(self._lib.aur_get_stats(self._h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in N.AurStats._fields_}


def lists_csr(lists):
    """A sequence of id arrays as (ids int64, offsets int64 [len + 1]): list l = ids[offsets[l]:offsets[l + 1]]."""
    parts = [np.asarray(a, dtype=np.int64).reshape(-1) for a in lists]
    offsets = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([len(a) for a in parts], out=offsets[1:])
    flat = np.ascontiguousarray(np.concatenate(parts)) if parts and offsets[-1] else np.zeros(1, dtype=np.int64)
    return flat, offsets


def shard_capacity(capacity: int, n: int) -> int:
    """Rows reserved on each of n shards of a store placed by ``id mod n`` (MultiIndex, MultiKeywordIndex): an even
    share plus headroom, since id mod n is balanced only statistically."""
    per = (int(capacity) + n - 1) // n
    return per + max(64, per // 8)


class MultiIndex:
    """One process, one shard per GPU of the host (the daemon's deployment on an 8-GPU box): the corpus is row-sharded
    by ``id mod n`` -- an upsert or a delete always lands on the shard that holds the old row -- every search runs on
    all shards at once (one host thread per device; the C calls release the GIL) and the per-shard top-k lists are
    merged on the host by (score desc, id asc), the order the device merge uses (csrc/kernels_simt.cu merge_topk_kernel).
    Same surface as ``Index`` for what ``retriever.KnowledgeBase`` and the daemon call.  The rank-per-GPU deployment with
    the fused peer-store exchange (sharded.ShardedIndex) stays the throughput path; this one trades ~0.1 ms of host
    merge for a single owner process.  ``shard_factory(dim, capacity, device)`` builds one shard (tests: a CPU double)."""

    def __init__(self, dim: int, capacity: int, devices=None, dtype: str = "bf16", shard_factory=None, _shards=None):
        from concurrent.futures import ThreadPoolExecutor

        if devices is None:
            devices = list(range(N.load().aur_device_count()))
        if not devices:
            raise RuntimeError("MultiIndex needs at least one device")
        self.dim, self.capacity, self.devices = int(dim), int(capacity), [int(d) for d in devices]
        n = len(self.devices)
        per = shard_capacity(self.capacity, n)
        self._native_merge = shard_factory is None and _shards is None
        if shard_factory is None:
            shard_factory = lambda dim_, cap_, dev_: Index(dim_, cap_, dtype=dtype, device=dev_)   # noqa: E731
        self.shards = _shards if _shards is not None else [shard_factory(self.dim, per, d) for d in self.devices]
        self.dtype = getattr(self.shards[0], "dtype", N.AUR_BF16)
        self._pool = ThreadPoolExecutor(max_workers=n, thread_name_prefix="aurora-b200-shard")

    # -------------------------------------------------------------- plumbing
    def _each(self, fn):
        """fn(shard index, shard) on every shard concurrently; results in shard order."""
        if len(self.shards) == 1:
            return [fn(0, self.shards[0])]
        return list(self._pool.map(lambda t: fn(*t), enumerate(self.shards)))

    def _split(self, ids: np.ndarray):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        owner = np.mod(ids, len(self.shards))
        return ids, [np.nonzero(owner == s)[0] for s in range(len(self.shards))]

    def _merge(self, parts, k: int):
        if len(parts) == 1:
            return parts[0]
        if self._native_merge:      # k-way merge of the sorted lists in C (csrc/host_merge.cpp): microseconds
            ids = np.ascontiguousarray(np.stack([p[0] for p in parts]), dtype=np.int64)
            sc = np.ascontiguousarray(np.stack([p[1] for p in parts]), dtype=np.float32)
            nq, k_in = ids.shape[1], ids.shape[2]
            out_s, out_i = np.empty((nq, k), dtype=np.float32), np.empty((nq, k), dtype=np.int64)
            N.check(N.load().aur_merge_topk_host(_ptr(sc), _ptr(ids), len(parts), nq, k_in, k, _ptr(out_s), _ptr(out_i)))
            return out_i, out_s
        ids = np.concatenate([p[0] for p in parts], axis=1)         # CPU doubles in the tests: the same order in numpy
        sc = np.concatenate([p[1] for p in parts], axis=1)
        key_id = np.where(ids < 0, np.iinfo(np.int64).max, ids)      # empty slots last
        order = np.lexsort((key_id, -sc.astype(np.float64)), axis=1)[:, :k]
        return np.take_along_axis(ids, order, axis=1), np.take_along_axis(sc, order, axis=1)

    # -------------------------------------------------------------- ingest / deletes
    def add(self, rows: np.ndarray, ids: np.ndarray, user_codes=None, org_codes=None) -> None:
        rows = np.asarray(rows)
        ids, sel = self._split(ids)
        u = None if user_codes is None else np.asarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.asarray(org_codes, dtype=np.int32)

        def put(s, shard):
            ix = sel[s]
            if len(ix):
                shard.add(rows[ix], ids[ix], None if u is None else u[ix], None if o is None else o[ix])
        self._each(put)

    def remove(self, ids) -> int:
        ids, sel = self._split(ids)
        return int(sum(self._each(lambda s, shard: shard.remove(ids[sel[s]]) if len(sel[s]) else 0)))

    # -------------------------------------------------------------- search
    def search(self, queries: np.ndarray, k: int, q_user=None, q_org=None):
        return self._merge(self._each(lambda s, shard: shard.search(queries, k, q_user, q_org)), k)

    def search_subset(self, queries: np.ndarray, k: int, allow_ids: np.ndarray):
        allow, sel = self._split(allow_ids)
        return self._merge(self._each(lambda s, shard: shard.search_subset(queries, k, allow[sel[s]])), k)

    def search_lists(self, queries: np.ndarray, k: int, lists, q_list):
        """Index.search_lists over every shard: each list is split by ``id mod n``, each shard searches its part."""
        split = [self._split(a) for a in lists]
        return self._merge(self._each(lambda s, shard: shard.search_lists(
            queries, k, [ids[sel[s]] for ids, sel in split], q_list)), k)

    def set_attrs(self, col: int, ids, codes) -> None:
        ids, sel = self._split(ids)
        codes = np.asarray(codes, dtype=np.int32)
        self._each(lambda s, shard: shard.set_attrs(col, ids[sel[s]], codes[sel[s]]))   # every shard gets the column

    def search_filtered(self, queries: np.ndarray, k: int, programs, q_program=None, max_list_rows: int = 0):
        """Index.search_filtered on every shard, each with an even share of ``max_list_rows``; merged as search_lists.
        Returns (ids, scores, matching rows per program summed over the shards, snapshot rows per shard)."""
        share = int(max_list_rows) // len(self.shards)
        parts = self._each(lambda s, shard: shard.search_filtered(queries, k, programs, q_program, share))
        ids, sc = self._merge([(p[0], p[1]) for p in parts], k)
        return ids, sc, np.sum([p[2] for p in parts], axis=0), [p[3] for p in parts]

    def filter_ids(self, program) -> np.ndarray:
        return np.concatenate(self._each(lambda s, shard: shard.filter_ids(program)))

    # -------------------------------------------------------------- maintenance
    def stats(self) -> dict:
        per = self._each(lambda s, shard: shard.stats())
        out = {key: int(sum(p.get(key, 0) for p in per)) for key in ("rows", "live", "searches")}
        out["last_kernel"] = per[0].get("last_kernel", 0)
        out["shards"] = len(per)
        out["rows_per_shard"] = [int(p.get("rows", 0)) for p in per]
        return out

    def compact(self) -> int:
        return int(sum(self._each(lambda s, shard: shard.compact())))

    def sync(self) -> None:
        self._each(lambda s, shard: shard.sync())

    def save(self, path: str) -> None:
        """One .npz like Index.save (live rows of all shards): a snapshot restores onto any number of devices."""
        parts = self._each(lambda s, shard: shard.export())
        cat = lambda i: np.concatenate([np.asarray(p[i])[p[4]] for p in parts])   # noqa: E731
        np.savez(path, rows=cat(0), ids=cat(1), user=cat(2), org=cat(3), dim=self.dim, dtype=self.dtype, capacity=self.capacity)

    @classmethod
    def load(cls, path: str, capacity: Optional[int] = None, devices=None, shard_factory=None) -> "MultiIndex":
        z = np.load(path if path.endswith(".npz") else path + ".npz")
        dtype = "bf16" if int(z["dtype"]) == N.AUR_BF16 else "f32"
        mi = cls(int(z["dim"]), int(capacity or z["capacity"]), devices=devices, dtype=dtype, shard_factory=shard_factory)
        if len(z["ids"]):
            mi.add(z["rows"], z["ids"], z["user"], z["org"])
        return mi

    def close(self) -> None:
        for sh in self.shards:
            sh.close()
        self.shards = []
        self._pool.shutdown(wait=False)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class KeywordIndex:
    """BM25 keyword store resident on one GPU (aur_kw_*): documents as (term id, tf) postings, keyed by the same ids and
    tenant codes as ``Index``.  The vocabulary (text -> term ids) lives in ``bm25.DeviceBM25``."""

    def __init__(self, capacity: int, postings_capacity: int = 0, device: int = 0):
        self._lib = N.load()
        self.capacity, self.device = int(capacity), int(device)
        self._h = C.c_void_p()
        N.check(self._lib.aur_kw_open(self.device, self.capacity, int(postings_capacity), C.byref(self._h)))

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.aur_kw_close(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, ids, term_ids, tfs, offsets, user_codes=None, org_codes=None) -> None:
        """Upsert len(ids) documents: document i has postings [offsets[i], offsets[i+1]) of term_ids / tfs (term ids
        strictly increasing within a document)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if offsets.shape != (ids.shape[0] + 1,):
            raise ValueError("offsets must be [n + 1]")
        t = np.ascontiguousarray(term_ids, dtype=np.int32)
        f = np.ascontiguousarray(tfs, dtype=np.int32)
        u = None if user_codes is None else np.ascontiguousarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.ascontiguousarray(org_codes, dtype=np.int32)
        N.check(self._lib.aur_kw_add(self._h, _ptr(ids), _ptr(u), _ptr(o), _ptr(t), _ptr(f), _ptr(offsets), ids.shape[0]))

    def remove(self, ids) -> int:
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        removed = C.c_int64(0)
        N.check(self._lib.aur_kw_remove(self._h, _ptr(ids), ids.shape[0], C.byref(removed)))
        return int(removed.value)

    def compact(self) -> int:
        freed = C.c_int64(0)
        N.check(self._lib.aur_kw_compact(self._h, C.byref(freed)))
        return int(freed.value)

    def stats(self) -> dict:
        st = N.AurKwStats()
        N.check(self._lib.aur_kw_get_stats(self._h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in N.AurKwStats._fields_}

    def search(self, q_terms, q_offsets, k: int, q_user=None, q_org=None, allow_ids=None):
        """(ids [nq,k] int64, scores [nq,k] float64, snapshot rows).  Query q's term ids are
        q_terms[q_offsets[q]:q_offsets[q+1]] in summation order.  ``allow_ids``: None = every document."""
        a = _kw_query_args(q_terms, q_offsets, k, q_user, q_org, allow_ids)
        snap = C.c_int64(-1)
        N.check(self._lib.aur_kw_search(self._h, *a["args"], C.byref(snap)))
        return a["ids"], a["scores"], int(snap.value)


def hybrid_search(index, kw_index, queries: np.ndarray, fetch: int, q_terms, q_offsets,
                  w_dense, w_sparse=None, fusion: int = N.FUSION_RANKED, k_out: Optional[int] = None, q_user=None,
                  q_org=None):
    """Both legs of the hybrid query and their fusion in one device call (aur_hybrid_search): the dense leg's top-``fetch``
    of ``queries`` over ``index`` and the keyword leg's top-``fetch`` of ``q_terms`` / ``q_offsets`` over ``kw_index``
    (same tenant scope), fused per query with weights ``w_dense`` / ``w_sparse`` (default ``1 - w_dense``).  Returns
    (ids [nq, k_out] int64, fused scores [nq, k_out] float64, dense cosines [nq, k_out] float32 (NaN: not in the dense
    list), (dense snapshot rows, keyword snapshot rows)); padding (-1, -inf, NaN).

    ``index`` / ``kw_index`` are an ``Index`` and a ``KeywordIndex``, or a ``MultiIndex`` of bf16 ``Index`` shards and a
    ``MultiKeywordIndex`` on the same devices in the same order (aur_hybrid_search_multi): each leg is then the global
    top-``fetch`` of ``MultiIndex.search`` / ``MultiKeywordIndex.search``, merged and fused on shard 0's GPU, and the
    snapshots are (one per shard, one per store)."""
    multi = isinstance(index, MultiIndex)
    if multi:
        if not isinstance(kw_index, MultiKeywordIndex):
            raise TypeError("a MultiIndex is searched together with a MultiKeywordIndex")
        if not index.shards or not all(isinstance(sh, Index) and sh.dtype == N.AUR_BF16 for sh in index.shards):
            raise TypeError("hybrid_search over a MultiIndex needs bf16 engine.Index shards")
        if kw_index.devices != index.devices or len(kw_index.stores) != len(index.shards):
            raise ValueError(f"keyword stores on devices {kw_index.devices}, vector shards on {index.devices}")
        q = index.shards[0]._rows_buffer(queries)
    else:
        q = index._rows_buffer(queries)
    nq = q.shape[0]
    k_out = 2 * int(fetch) if k_out is None else int(k_out)
    wd = np.ascontiguousarray(np.broadcast_to(np.asarray(w_dense, dtype=np.float64), (nq,)))
    ws = 1.0 - wd if w_sparse is None else np.ascontiguousarray(np.broadcast_to(np.asarray(w_sparse, dtype=np.float64), (nq,)))
    a = _kw_query_args(q_terms, q_offsets, 1, q_user, q_org, None)
    qt, q_off, u, o, _ = a["keep"]
    if q_off.shape[0] - 1 != nq:
        raise ValueError(f"{nq} query vectors but {q_off.shape[0] - 1} keyword queries")
    scores = np.empty((nq, k_out), dtype=np.float64)
    ids = np.empty((nq, k_out), dtype=np.int64)
    cosine = np.empty((nq, k_out), dtype=np.float32)
    if multi:
        n = len(index.shards)
        shards = (C.c_void_p * n)(*[sh._h.value for sh in index.shards])
        stores = (C.c_void_p * n)(*[st._h.value for st in kw_index.stores])
        snaps = np.full(2 * n, -1, dtype=np.int64)
        N.check(N.load().aur_hybrid_search_multi(shards, stores, n, _ptr(q), nq, int(fetch), _ptr(qt), _ptr(q_off), _ptr(u),
                                                 _ptr(o), _ptr(wd), _ptr(ws), int(fusion), k_out, _ptr(scores), _ptr(ids),
                                                 _ptr(cosine), _ptr(snaps)))
        return ids, scores, cosine, (snaps[:n].tolist(), snaps[n:].tolist())
    snaps = (C.c_int64 * 2)(-1, -1)
    N.check(index._lib.aur_hybrid_search(index._h, kw_index._h, _ptr(q), nq, int(fetch), _ptr(qt), _ptr(q_off), _ptr(u),
                                         _ptr(o), _ptr(wd), _ptr(ws), int(fusion), k_out, _ptr(scores), _ptr(ids),
                                         _ptr(cosine), snaps))
    return ids, scores, cosine, (int(snaps[0]), int(snaps[1]))


def _kw_query_args(q_terms, q_offsets, k, q_user, q_org, allow_ids):
    """The query-side arguments of aur_kw_search / aur_kw_search_multi and the output arrays they fill (kept alive in
    the returned dict for the duration of the call)."""
    q_off = np.ascontiguousarray(q_offsets, dtype=np.int64)
    nq = q_off.shape[0] - 1
    qt = np.ascontiguousarray(q_terms, dtype=np.int32)
    if qt.size == 0:
        qt = np.zeros(1, dtype=np.int32)
    scores = np.empty((nq, k), dtype=np.float64)
    ids = np.empty((nq, k), dtype=np.int64)
    u = None if q_user is None else np.ascontiguousarray(q_user, dtype=np.int32)
    o = None if q_org is None else np.ascontiguousarray(q_org, dtype=np.int32)
    allow, n_allow = None, 0
    if allow_ids is not None:
        allow = np.ascontiguousarray(allow_ids, dtype=np.int64)
        n_allow = allow.shape[0]
        if n_allow == 0:
            allow = np.zeros(1, dtype=np.int64)     # a real pointer: "nothing is allowed"
    args = (_ptr(qt), _ptr(q_off), int(nq), int(k), _ptr(u), _ptr(o), _ptr(allow), int(n_allow), _ptr(scores), _ptr(ids))
    return {"args": args, "ids": ids, "scores": scores, "keep": (qt, q_off, u, o, allow)}


class MultiKeywordIndex:
    """One BM25 keyword store per GPU of the host, searched as one corpus (aur_kw_search_multi): documents are placed by
    ``id mod n`` like ``MultiIndex``'s rows -- an upsert or a delete always reaches the store that holds the old row --
    and every search scores each store's prefix on its own GPU with the idf and avgdl of the union of the stores'
    snapshots, so the answer is bit for bit that of a single ``KeywordIndex`` holding every document.  Same surface as
    ``KeywordIndex``; ``search`` reports the snapshot rows of every store.  ``store_factory(capacity,
    postings_capacity, device)`` builds one store (tests: a recording double)."""

    _SUMMED = ("docs", "live", "capacity", "postings_used", "postings_allocated", "total_len")

    def __init__(self, capacity: int, devices=None, postings_capacity: int = 0, store_factory=None):
        from concurrent.futures import ThreadPoolExecutor

        if devices is None:
            devices = list(range(N.load().aur_device_count()))
        if not devices:
            raise RuntimeError("MultiKeywordIndex needs at least one device")
        self.capacity, self.devices = int(capacity), [int(d) for d in devices]
        n = len(self.devices)
        if n > 64:
            raise ValueError("MultiKeywordIndex takes at most 64 stores")
        per = shard_capacity(self.capacity, n)
        per_post = shard_capacity(postings_capacity, n) if postings_capacity else 0
        if store_factory is None:
            store_factory = lambda cap, post, dev: KeywordIndex(cap, postings_capacity=post, device=dev)   # noqa: E731
        self.stores = [store_factory(per, per_post, d) for d in self.devices]
        self._pool = ThreadPoolExecutor(max_workers=n, thread_name_prefix="aurora-b200-kw")

    def _each(self, fn):
        """fn(store index, store) on every store concurrently (each waits on its own GPU); results in store order."""
        if len(self.stores) == 1:
            return [fn(0, self.stores[0])]
        return list(self._pool.map(lambda t: fn(*t), enumerate(self.stores)))

    def _split(self, ids: np.ndarray):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        owner = np.mod(ids, len(self.stores))
        return ids, [np.nonzero(owner == s)[0] for s in range(len(self.stores))]

    def add(self, ids, term_ids, tfs, offsets, user_codes=None, org_codes=None) -> None:
        """KeywordIndex.add, each document to store ``id mod n``: its CSR rows are cut out and their offsets rebased."""
        ids, sel = self._split(ids)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        if offsets.shape != (ids.shape[0] + 1,):
            raise ValueError("offsets must be [n + 1]")
        t = np.ascontiguousarray(term_ids, dtype=np.int32)
        f = np.ascontiguousarray(tfs, dtype=np.int32)
        u = None if user_codes is None else np.asarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.asarray(org_codes, dtype=np.int32)

        def put(s, store):
            rows = sel[s]
            if not len(rows):
                return
            lens = offsets[rows + 1] - offsets[rows]
            sub_off = np.zeros(len(rows) + 1, dtype=np.int64)
            np.cumsum(lens, out=sub_off[1:])
            take = np.repeat(offsets[rows] - sub_off[:-1], lens) + np.arange(sub_off[-1], dtype=np.int64)
            store.add(ids[rows], t[take], f[take], sub_off, None if u is None else u[rows], None if o is None else o[rows])
        self._each(put)

    def remove(self, ids) -> int:
        ids, sel = self._split(ids)
        return int(sum(self._each(lambda s, store: store.remove(ids[sel[s]]) if len(sel[s]) else 0)))

    def compact(self) -> int:
        return int(sum(self._each(lambda s, store: store.compact())))

    def stats(self) -> dict:
        """KeywordIndex.stats summed over the stores (the last search: launches and spills summed, terms and device time
        the largest of any store); ``stores`` lists every store's own."""
        per = self._each(lambda s, store: store.stats())
        out = {key: int(sum(p[key] for p in per)) for key in self._SUMMED}
        out["last_launches"] = int(sum(p["last_launches"] for p in per))
        out["last_spilled"] = int(sum(p["last_spilled"] for p in per))
        out["last_terms"] = max(p["last_terms"] for p in per)
        out["last_ms"] = max(p["last_ms"] for p in per)
        out["stores"] = per
        return out

    def search(self, q_terms, q_offsets, k: int, q_user=None, q_org=None, allow_ids=None):
        """(ids [nq,k] int64, scores [nq,k] float64, snapshot rows [n stores]): KeywordIndex.search over the union of the
        stores."""
        a = _kw_query_args(q_terms, q_offsets, k, q_user, q_org, allow_ids)
        handles = (C.c_void_p * len(self.stores))(*[st._h.value for st in self.stores])
        snaps = np.full(len(self.stores), -1, dtype=np.int64)
        N.check(N.load().aur_kw_search_multi(handles, len(self.stores), *a["args"], _ptr(snaps)))
        return a["ids"], a["scores"], [int(x) for x in snaps]

    def close(self) -> None:
        for st in self.stores:
            st.close()
        self.stores = []
        self._pool.shutdown(wait=False)


def merge_topk_packed_dev(device: int, packed_ptr: int, n_shards: int, nq: int, k: int, out_scores_ptr: int,
                          out_ids_ptr: int, out_scores64_ptr: int = 0, stream: int = 0) -> None:
    """packed: [n_shards][2][nq][k] 8-byte words (plane 0 fp64 scores, plane 1 int64 ids)."""
    lib = N.load()
    N.check(lib.aur_merge_topk_packed_dev(int(device), C.c_void_p(packed_ptr), int(n_shards), int(nq), int(k),
                                          C.c_void_p(out_scores_ptr), C.c_void_p(out_ids_ptr),
                                          C.c_void_p(out_scores64_ptr), C.c_void_p(stream)))


def merge_topk_dev(device: int, in_scores64_ptr: int, in_ids_ptr: int, n_shards: int, nq: int, k: int,
                   out_scores_ptr: int, out_ids_ptr: int, out_scores64_ptr: int = 0, stream: int = 0) -> None:
    lib = N.load()
    N.check(lib.aur_merge_topk_dev(int(device), C.c_void_p(in_scores64_ptr), C.c_void_p(in_ids_ptr), int(n_shards),
                                   int(nq), int(k), C.c_void_p(out_scores_ptr), C.c_void_p(out_ids_ptr),
                                   C.c_void_p(out_scores64_ptr), C.c_void_p(stream)))


def cosine_pairs(a: np.ndarray, b: np.ndarray, clamp: bool = False, device: int = 0) -> np.ndarray:
    """Row-wise cosine on the GPU (fp64 accumulate).  Mirrors
    SimilarityStrategy._cosine_similarity (similarity.py:84-98) for batches."""
    lib = N.load()
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    if a.shape != b.shape or a.ndim != 2:
        raise ValueError("a and b must both be [n, dim]")
    out = np.empty(a.shape[0], dtype=np.float64)
    N.check(lib.aur_cosine_pairs(int(device), _ptr(a), _ptr(b), a.shape[0], a.shape[1], int(bool(clamp)), _ptr(out)))
    return out


class DeviceBuffer:
    """Raw HBM buffer owned through the C ABI (for callers without torch)."""

    def __init__(self, nbytes: int, device: int = 0):
        self._lib = N.load()
        self.device, self.nbytes = int(device), int(nbytes)
        p = C.c_void_p()
        N.check(self._lib.aur_dev_malloc(self.device, self.nbytes, C.byref(p)))
        self.ptr = int(p.value)

    def upload(self, a: np.ndarray) -> "DeviceBuffer":
        a = np.ascontiguousarray(a)
        if a.nbytes > self.nbytes:
            raise ValueError("buffer too small")
        N.check(self._lib.aur_memcpy_h2d(self.device, C.c_void_p(self.ptr), _ptr(a), a.nbytes))
        return self

    def download(self, a: np.ndarray) -> np.ndarray:
        if not a.flags["C_CONTIGUOUS"] or a.nbytes > self.nbytes:
            raise ValueError("need a contiguous array no larger than the buffer")
        N.check(self._lib.aur_memcpy_d2h(self.device, _ptr(a), C.c_void_p(self.ptr), a.nbytes))
        return a

    def free(self) -> None:
        if self.ptr:
            self._lib.aur_dev_free(self.device, C.c_void_p(self.ptr))
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

"""Files and helpers of ``KnowledgeBase.checkpoint``: incremental snapshots of a serving knowledge base.

A snapshot directory holds one manifest, ``meta.json``, and the files it names:

* the base: ``shard.{gen}.npz`` (``Index.save`` format: the live rows of every shard at the base's capture, so
  ``Index.load`` / ``MultiIndex.load`` / any ``index_loader`` restores it), ``base.{tag}.npz`` (the shard and row
  number every one of those rows had, by id) and ``base.{tag}.jsonl`` (every object's id, key and properties);
* the deltas since the base, in order: ``delta.{tag}.{s}.npz`` per shard s (the rows appended since the previous
  checkpoint that were live at capture, their row numbers, and the shard's full live and nonfinite bitmaps) and
  ``delta.{tag}.jsonl`` (the objects upserted and deleted since the previous checkpoint).

A shard's rows never move between two captures with the same compaction count, so a row's liveness at the last
capture is one bit of the last delta's bitmap.  DESIGN.md section 8 ("Snapshots") has the rules.
"""

from __future__ import annotations

import json
import os
import uuid
from typing import Any, Callable, Dict, List, Optional

import numpy as np

MAX_DELTAS = 16            # a delta beyond this many since the base writes a new base instead
MAX_DELTA_FRACTION = 0.25  # ... as do more rows appended since the base than this share of the base's rows
PREFIXES = ("shard.", "base.", "delta.")   # the files a checkpoint owns in its directory (besides meta.json)


def pack_bits(mask: np.ndarray) -> np.ndarray:
    """bool [n] -> uint32 words [ceil(n / 32)], bit r % 32 of word r // 32 = mask[r] (aur_live_bits' layout)."""
    b = np.packbits(np.asarray(mask, dtype=bool), bitorder="little")
    pad = (-len(b)) % 4
    return np.concatenate([b, np.zeros(pad, np.uint8)]).view("<u4").astype(np.uint32)


def bits_at(words: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """The bits of ``rows`` (int array) in ``words``: bool [len(rows)]."""
    rows = np.asarray(rows, dtype=np.int64)
    if not len(rows):
        return np.zeros(0, dtype=bool)
    return ((np.asarray(words, dtype=np.uint32)[rows >> 5] >> (rows & 31).astype(np.uint32)) & 1).astype(bool)


def unpack_bits(words: np.ndarray, n: int) -> np.ndarray:
    return bits_at(words, np.arange(int(n), dtype=np.int64))


class ExportCapture:
    """``capture`` / ``export_rows`` of an index without them (the CPU doubles), through its ``export``: one export per
    capture, whose rows the following ``export_rows`` calls slice.  Rows were renumbered (a compaction) when the ids of
    the previous capture are no longer a prefix of this one's; that counts as one compaction."""

    def __init__(self, index):
        self.index = index
        self._ids: Optional[np.ndarray] = None
        self._snap = None
        self._compactions = 0

    def capture(self):
        ix = self.index
        rows, ids, user, org, live = ix.export_raw() if hasattr(ix, "export_raw") else ix.export()
        ids = np.array(ids, dtype=np.int64)
        live = np.asarray(live).astype(np.uint8)
        prev = self._ids
        if prev is not None and (len(ids) < len(prev) or not np.array_equal(ids[:len(prev)], prev)):
            self._compactions += 1
        self._ids = ids
        self._snap = (np.asarray(rows), ids, np.asarray(user, dtype=np.int32), np.asarray(org, dtype=np.int32))
        return len(ids), pack_bits(live > 0), pack_bits(live == 2), self._compactions

    def export_rows(self, row0: int, n: int):
        rows, ids, user, org = self._snap
        sl = slice(int(row0), int(row0) + int(n))
        return rows[sl], ids[sl], user[sl], org[sl]


class Shards:
    """The vector shards of a knowledge base's index as a checkpoint reads them: ``capture()`` and
    ``export_rows(ranges)`` give one result per shard.  A ``MultiIndex`` of CUDA shards runs both on every shard at
    once; an index without ``capture`` goes through ``ExportCapture``."""

    def __init__(self, index):
        self.index = index
        self.parts = list(getattr(index, "shards", None) or [index])
        self.native = all(hasattr(p, "capture") and hasattr(p, "export_rows") for p in self.parts)
        self._fallback = None if self.native else [ExportCapture(p) for p in self.parts]

    def capture(self) -> list:
        if not self.native:
            return [f.capture() for f in self._fallback]
        return self.index.capture() if hasattr(self.index, "shards") else [self.index.capture()]

    def export_rows(self, ranges) -> list:
        if not self.native:
            return [f.export_rows(*r) for f, r in zip(self._fallback, ranges)]
        if hasattr(self.index, "shards"):
            return self.index.export_rows(ranges)
        return [self.index.export_rows(*ranges[0])]


def new_tag(gen: int) -> str:
    """A file-name tag no earlier checkpoint used: a crashed write never overwrites a file a manifest names."""
    return f"{int(gen)}-{uuid.uuid4().hex[:12]}"


def fsync_dir(directory: str) -> None:
    fd = os.open(directory, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def write_file(path: str, fill: Callable[[Any], None]) -> int:
    """``fill(file)`` into ``path`` beside its final name, fsync'd, then renamed into place.  Returns its bytes."""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        fill(f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)
    return os.path.getsize(path)


def write_npz(path: str, **arrays) -> int:
    return write_file(path, lambda f: np.savez(f, **arrays))


def write_jsonl(path: str, records) -> int:
    def fill(f):
        buf = []
        for rec in records:
            buf.append(json.dumps(rec, separators=(",", ":")))
            if len(buf) >= 4096:
                f.write(("\n".join(buf) + "\n").encode("utf-8"))
                buf = []
        if buf:
            f.write(("\n".join(buf) + "\n").encode("utf-8"))
    return write_file(path, fill)


def read_jsonl(path: str):
    with open(path, encoding="utf-8") as f:
        for line in f:
            if line.strip():
                yield json.loads(line)


def referenced(meta: Dict[str, Any]) -> List[str]:
    """Every file a manifest names."""
    base = meta.get("base") or {}
    names = [meta.get("shard"), base.get("rows"), base.get("meta")]
    for d in meta.get("deltas", []):
        names += [*d["shards"], d["meta"]]
    return [n for n in names if n]


def remove_unreferenced(directory: str, meta: Dict[str, Any]) -> None:
    """Delete the checkpoint files of superseded generations (called once ``meta`` is durable)."""
    keep = set(referenced(meta))
    for name in os.listdir(directory):
        if name.startswith(PREFIXES) and name not in keep:
            try:
                os.remove(os.path.join(directory, name))
            except OSError:
                pass


def restore_rows(rows: np.ndarray, nonfinite: np.ndarray) -> np.ndarray:
    """Rows as ``add`` takes them back (``engine._snapshot_rows``'s rule): an int8 row stored from a row holding a NaN or
    inf is re-added as a bf16 row holding a NaN."""
    if len(nonfinite) and np.any(nonfinite):
        from .engine import to_bf16_bits

        rows = to_bf16_bits(np.asarray(rows, dtype=np.float32))
        rows[np.asarray(nonfinite, dtype=bool), 0] = 0x7FC0
    return rows


def apply_deltas(loaded, directory: str, meta: Dict[str, Any]) -> None:
    """Bring ``loaded`` (the index ``index_loader`` restored from the base's ``shard.{gen}.npz``) to the last delta's
    capture through its own ``remove`` and ``add``: base rows dead in the last bitmaps go, delta rows live in them come
    (placed by the loaded index, e.g. by ``id mod n``)."""
    deltas = meta.get("deltas") or []
    if not deltas:
        return
    last = [np.load(os.path.join(directory, name)) for name in deltas[-1]["shards"]]
    final = [z["live"] for z in last]
    zb = np.load(os.path.join(directory, meta["base"]["rows"]))
    alive = np.ones(len(zb["ids"]), dtype=bool)
    for s, words in enumerate(final):
        on = zb["part"] == s
        alive[on] = bits_at(words, zb["row"][on])
    dead = zb["ids"][~alive]
    if len(dead):
        loaded.remove(np.ascontiguousarray(dead, dtype=np.int64))
    parts = {"rows": [], "ids": [], "user": [], "org": [], "nonfinite": []}
    for d in deltas:
        for s, name in enumerate(d["shards"]):
            z = np.load(os.path.join(directory, name))
            keep = bits_at(final[s], z["row"])
            for key in parts:
                parts[key].append(z[key][keep])
    ids = np.concatenate(parts["ids"])
    if not len(ids):
        return
    from .engine import grow_for

    grow_for(loaded, ids)
    loaded.add(restore_rows(np.concatenate(parts["rows"]), np.concatenate(parts["nonfinite"])), ids,
               np.concatenate(parts["user"]), np.concatenate(parts["org"]))


def read_objects(directory: str, meta: Dict[str, Any]):
    """(props {id: properties}, key2id {key: id}) at the last checkpoint: the base's table, then every delta's upserts
    and deletes in order."""
    props: Dict[int, Dict[str, Any]] = {}
    key2id: Dict[str, int] = {}
    for rid, key, p in read_jsonl(os.path.join(directory, meta["base"]["meta"])):
        props[int(rid)] = p
        if key is not None:
            key2id[key] = int(rid)
    for d in meta.get("deltas") or []:
        for rec in read_jsonl(os.path.join(directory, d["meta"])):
            if rec[0] == "put":
                _, rid, key, p = rec
                props[int(rid)] = p
                if key is not None:
                    key2id[key] = int(rid)
            else:
                _, rid, key = rec
                props.pop(int(rid), None)
                if key is not None and key2id.get(key) == int(rid):
                    del key2id[key]
    return props, key2id

"""Engine daemon + client shim (SURVEY.md section 8(f) item 4, hard part D).

A corpus shard in HBM belongs to ONE process per host, but the reference reaches its vector store
from 2 gunicorn workers x 4 threads, 4 Celery children and the chatbot process
(docker-compose.yaml:191, :283-285) -- over gRPC to the Weaviate container.  Here the owner is this
daemon and the other processes talk to it over a Unix-domain socket with the SAME module API:

    server:  python -m aurora_b200.daemon --socket /run/aurora_b200.sock --snapshot /var/lib/aurora_b200
    client:  from aurora_b200.daemon import Client; kb = Client("/run/aurora_b200.sock")
             kb.search_knowledge_base(user_id, query, limit=5)              # weaviate_client.py:215
             kb._get_weaviate_client()                                      # rca_prompt_builder.py:276-298
             kb.search_similar_good_rcas(...)                               # incident_feedback/weaviate_client.py:246

Wire format: 4-byte big-endian length + JSON ``{"fn", "args", "kwargs"}`` -> ``{"ok", "result" | "error"}``.
The client keeps the reference's error conventions when the daemon is unreachable (search -> [],
deletes -> -1, counts -> 0, insert re-raises so the Celery task retries; weaviate_client.py:210-212,
:283-285, :317-319, :369-371).  ``health()`` replaces the Weaviate readiness probe of
routes/health_routes.py:76-91.

Request coalescing.  The reference issues one query per call (weaviate_client.py:252-259), from up to a dozen
threads at once.  One query uses a sliver of the GPU (an encoder forward of one sequence is ~90 launches of almost
empty kernels), so concurrent ``search_knowledge_base`` calls are gathered for at most ``coalesce_us`` microseconds:
their query texts go through ONE encoder batch, and the dense leg runs as one kernel launch per distinct tenant scope
in the window (the scope folds into the row scale, see csrc/capi.cu); each caller gets its own result back.

Durability.  The daemon owns the only copy of the vectors: it snapshots the knowledge base (KnowledgeBase.save:
atomic rename of shard + metadata) after ``save_every`` mutations or ``save_seconds`` seconds with unsaved
mutations, on SIGTERM / shutdown, and on the ``save`` call; it compacts tombstones when more than a quarter of the
shard is dead.  Between snapshots every acknowledged insert / delete is in the mutation log beside the snapshot
(KnowledgeBase.attach_wal, fsync'd before the reply; bootstrap.configure_from_env attaches it): a restart loads the
last snapshot and replays the log.  The socket is created with mode 0600: any local process that can open it can read every tenant.
"""

from __future__ import annotations

import json
import logging
import os
import signal
import socket
import socketserver
import struct
import threading
import time
from types import SimpleNamespace
from typing import Any, Dict, List, Optional

logger = logging.getLogger(__name__)

API = ("insert_chunks", "search_knowledge_base", "delete_document_chunks", "delete_user_chunks",
       "get_document_chunk_count", "delete_discovery_chunks")
LEARN_API = ("store_good_rca", "search_similar_good_rcas", "delete_incident_knowledge", "delete_user_knowledge")


def _send(sock: socket.socket, obj: Any) -> None:
    raw = json.dumps(obj).encode("utf-8")
    sock.sendall(struct.pack(">I", len(raw)) + raw)


def _recv(sock: socket.socket) -> Optional[Any]:
    def read(n: int) -> Optional[bytes]:
        buf = b""
        while len(buf) < n:
            chunk = sock.recv(n - len(buf))
            if not chunk:
                return None
            buf += chunk
        return buf

    head = read(4)
    if head is None:
        return None
    body = read(struct.unpack(">I", head)[0])
    return None if body is None else json.loads(body.decode("utf-8"))


# ----------------------------------------------------------------------------- request coalescing
class _Pending:
    __slots__ = ("args", "event", "result", "error")

    def __init__(self, args):
        self.args, self.event, self.result, self.error = args, threading.Event(), None, None


class SearchCoalescer:
    """Gathers concurrent search_knowledge_base calls into one encoder batch (+ one dense launch per tenant scope)."""

    def __init__(self, module, window_us: int = 200, max_batch: int = 256):
        self.module, self.window, self.max_batch = module, window_us * 1e-6, max_batch
        self._q: List[_Pending] = []
        self._cv = threading.Condition()
        self._stop = False
        self.batches = self.requests = 0
        self._t = threading.Thread(target=self._run, name="aurora-b200-coalescer", daemon=True)
        self._t.start()

    def submit(self, user_id, query, limit=5, alpha=0.5, min_score=0.0, org_id=None):
        if not isinstance(query, str) or not query.strip():
            return []
        p = _Pending((user_id, query, limit, alpha, min_score, org_id))
        with self._cv:
            self._q.append(p)
            self._cv.notify()
        p.event.wait()
        if p.error is not None:
            raise p.error
        return p.result

    def close(self) -> None:
        with self._cv:
            self._stop = True
            self._cv.notify()
        self._t.join(timeout=5)

    def _run(self) -> None:
        while True:
            with self._cv:
                while not self._q and not self._stop:
                    self._cv.wait()
                if self._stop and not self._q:
                    return
                deadline = time.perf_counter() + self.window        # the first request opens the window
                while len(self._q) < self.max_batch:
                    left = deadline - time.perf_counter()
                    if left <= 0:
                        break
                    self._cv.wait(left)
                batch, self._q = self._q[: self.max_batch], self._q[self.max_batch:]
            self.batches += 1
            self.requests += len(batch)
            try:
                batched = getattr(self.module, "search_knowledge_base_batch", None)
                if batched is not None and len(batch) > 1:
                    results = batched([p.args for p in batch])
                else:
                    results = [self.module.search_knowledge_base(*p.args[:2], limit=p.args[2], alpha=p.args[3], min_score=p.args[4],
                                                                 org_id=p.args[5]) for p in batch]
                for p, r in zip(batch, results):
                    p.result = r
            except Exception as e:          # search swallows errors itself (-> []); this is a programming error
                for p in batch:
                    p.error = e
            for p in batch:
                p.event.set()


# ----------------------------------------------------------------------------- snapshot policy
class SnapshotPolicy:
    """Saves the knowledge base after N mutations / T seconds with unsaved mutations, and on demand."""

    def __init__(self, module, directory: Optional[str], save_every: int = 2000, save_seconds: float = 60.0):
        self.module, self.dir, self.every, self.seconds = module, directory, save_every, save_seconds
        self._lock = threading.Lock()
        self._stop = threading.Event()
        self.saves = 0
        self._t = None
        if directory:
            self._t = threading.Thread(target=self._run, name="aurora-b200-snapshots", daemon=True)
            self._t.start()

    def _kb(self):
        get = getattr(self.module, "_get_kb", None)
        return get() if get else None

    def unsaved(self) -> int:
        try:
            kb = self._kb()
            return int(kb.mutations - kb.saved_mutations) if kb is not None else 0
        except Exception:
            return 0

    def save(self) -> dict:
        if not self.dir:
            raise RuntimeError("the daemon was started without --snapshot")
        with self._lock:
            kb = self._kb()
            t0 = time.perf_counter()
            dead = 0
            try:       # reclaim tombstones first when they are a sizeable part of the shard
                st = kb.index.stats()
                if st["rows"] > 1024 and (st["rows"] - st["live"]) * 4 > st["rows"]:
                    dead = kb.index.compact()
            except Exception:
                pass
            try:       # the GPU keyword store by the same rule (the host BM25Index keeps no tombstones)
                if hasattr(kb.sparse, "compact"):
                    ks = kb.sparse.stats()
                    if ks["docs"] > 1024 and (ks["docs"] - ks["live"]) * 4 > ks["docs"]:
                        kb.sparse.compact()
            except Exception:
                pass
            kb.save(self.dir)
            self.saves += 1
            return {"saved": True, "directory": self.dir, "seconds": round(time.perf_counter() - t0, 3), "compacted_rows": dead}

    def _run(self) -> None:
        last = time.perf_counter()
        while not self._stop.wait(1.0):
            n = self.unsaved()
            if n and (n >= self.every or time.perf_counter() - last >= self.seconds):
                try:
                    self.save()
                except Exception as e:      # pragma: no cover
                    logger.error(f"[KB B200 daemon] snapshot failed: {e}")
                last = time.perf_counter()

    def close(self, final_save: bool = True) -> None:
        self._stop.set()
        if self._t is not None:
            self._t.join(timeout=5)
        if final_save and self.dir and self.unsaved():
            try:
                self.save()
            except Exception as e:          # pragma: no cover
                logger.error(f"[KB B200 daemon] final snapshot failed: {e}")


class _Handler(socketserver.BaseRequestHandler):
    def handle(self) -> None:
        srv = self.server
        module = srv.module          # type: ignore[attr-defined]
        while True:
            try:
                req = _recv(self.request)
            except (OSError, ValueError):
                return
            if req is None:
                return
            fn, args, kwargs = req.get("fn"), req.get("args", []), req.get("kwargs", {})
            try:
                if fn == "health":
                    res = {"ready": True, "pid": os.getpid(), "unsaved_mutations": srv.snapshots.unsaved(),
                           "coalesced_batches": srv.coalescer.batches if srv.coalescer else 0,
                           "coalesced_requests": srv.coalescer.requests if srv.coalescer else 0}
                elif fn == "save":
                    res = srv.snapshots.save()
                elif fn == "search_knowledge_base" and srv.coalescer is not None:
                    res = srv.coalescer.submit(*args, **kwargs)
                elif fn in API:
                    res = getattr(module, fn)(*args, **kwargs)
                elif fn in ("hybrid", "near_text"):      # the private facade of rca_prompt_builder.py:276-298, over the wire
                    res = _facade_query(module, fn, kwargs)
                elif fn in LEARN_API:
                    if srv.learn_module is None:
                        raise RuntimeError("Aurora Learn is not configured in this daemon")
                    res = getattr(srv.learn_module, fn)(*args, **kwargs)
                else:
                    raise ValueError(f"unknown function {fn!r}")
                _send(self.request, {"ok": True, "result": res})
            except Exception as e:           # insert_chunks re-raises by design: report it to the caller
                _send(self.request, {"ok": False, "error": f"{type(e).__name__}: {e}"})


def _facade_query(module, fn: str, kw: Dict[str, Any]):
    from .filters import Filter

    _, collection = module._get_weaviate_client()
    flt = Filter.from_json(kw.get("filters"))
    if fn == "hybrid":
        resp = collection.query.hybrid(query=kw["query"], limit=kw.get("limit", 10), alpha=kw.get("alpha", 0.5),
                                       fusion_type=kw.get("fusion_type"), filters=flt)
    else:
        resp = collection.query.near_text(query=kw["query"], limit=kw.get("limit", 10), filters=flt)
    return [{"properties": o.properties, "uuid": o.uuid, "score": o.metadata.score, "distance": o.metadata.distance} for o in resp.objects]


class _Server(socketserver.ThreadingMixIn, socketserver.UnixStreamServer):
    daemon_threads = True
    allow_reuse_address = True
    request_queue_size = 256      # gunicorn threads + Celery children connect at once

    def server_bind(self):
        old = os.umask(0o177)     # the socket is born 0600: whoever can open it can read every tenant's chunks
        try:
            super().server_bind()
        finally:
            os.umask(old)

    def close_all(self, final_save: bool = True):
        if self.coalescer is not None:
            self.coalescer.close()
        self.snapshots.close(final_save)


def serve(socket_path: str, module=None, background: bool = False, learn_module=None, snapshot_dir: Optional[str] = None,
          save_every: int = 2000, save_seconds: float = 60.0, coalesce_us: int = 200):
    """Serve ``module`` (default: aurora_b200.retriever, already ``configure()``d) on ``socket_path``."""
    if module is None:
        from . import retriever as module
    if os.path.exists(socket_path):
        os.unlink(socket_path)
    srv = _Server(socket_path, _Handler)
    srv.module = module                     # type: ignore[attr-defined]
    srv.learn_module = learn_module
    srv.coalescer = SearchCoalescer(module, coalesce_us) if coalesce_us > 0 else None
    srv.snapshots = SnapshotPolicy(module, snapshot_dir, save_every, save_seconds)
    if background:
        t = threading.Thread(target=srv.serve_forever, name="aurora-b200-daemon", daemon=True)
        t.start()
        return srv

    def _term(signum, frame):               # SIGTERM: stop accepting, then the finally block below saves
        threading.Thread(target=srv.shutdown, daemon=True).start()

    signal.signal(signal.SIGTERM, _term)
    try:
        srv.serve_forever()
    finally:
        srv.close_all(final_save=True)
        srv.server_close()
    return srv


class DaemonUnavailable(RuntimeError):
    pass


class _RemoteQuery:
    def __init__(self, client: "Client"):
        self._c = client

    def _objs(self, rows):
        return SimpleNamespace(objects=[SimpleNamespace(properties=r["properties"], uuid=r["uuid"],
                                                        metadata=SimpleNamespace(score=r["score"], distance=r["distance"])) for r in rows])

    def hybrid(self, query: str, limit: int = 10, alpha: float = 0.5, fusion_type=None, filters=None, return_metadata=None, **_):
        return self._objs(self._c._call("hybrid", query=query, limit=limit, alpha=alpha, fusion_type=fusion_type,
                                        filters=None if filters is None else filters.to_json()))

    def near_text(self, query: str, limit: int = 10, filters=None, return_metadata=None, **_):
        return self._objs(self._c._call("near_text", query=query, limit=limit, filters=None if filters is None else filters.to_json()))


class Client:
    """Same names / signatures as routes.knowledge_base.weaviate_client (+ the Aurora Learn module and the private
    ``_get_weaviate_client`` facade); one connection per thread."""

    def __init__(self, socket_path: str, timeout: float = 30.0):
        self._path, self._timeout = socket_path, timeout
        self._local = threading.local()

    def _call(self, fn: str, *args, **kwargs):
        for attempt in (0, 1):               # one reconnect: the daemon may have restarted
            sock = getattr(self._local, "sock", None)
            try:
                if sock is None:
                    sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
                    sock.settimeout(self._timeout)
                    sock.connect(self._path)
                    self._local.sock = sock
                _send(sock, {"fn": fn, "args": list(args), "kwargs": kwargs})
                resp = _recv(sock)
                if resp is None:
                    raise ConnectionError("daemon closed the connection")
                if not resp["ok"]:
                    raise RuntimeError(resp["error"])
                return resp["result"]
            except (OSError, ConnectionError) as e:
                if sock is not None:
                    try:
                        sock.close()
                    except OSError:
                        pass
                self._local.sock = None
                if attempt == 1:
                    raise DaemonUnavailable(str(e)) from e

    def health(self) -> dict:
        try:
            return self._call("health")
        except Exception as e:
            return {"ready": False, "error": str(e)}

    def save(self) -> dict:
        """Ask the daemon for a snapshot now (it also saves by itself, see the module docstring)."""
        return self._call("save")

    # ---- the reference's module API, with its error conventions on transport failure
    def insert_chunks(self, user_id, document_id, source_filename, chunks, org_id=None) -> int:
        if not chunks:
            return 0
        return self._call("insert_chunks", user_id, document_id, source_filename, chunks, org_id=org_id)   # raises -> retry

    def search_knowledge_base(self, user_id, query, limit=5, alpha=0.5, min_score=0.0, org_id=None):
        if not query.strip():
            return []
        try:
            return self._call("search_knowledge_base", user_id, query, limit=limit, alpha=alpha, min_score=min_score, org_id=org_id)
        except Exception as e:
            logger.error(f"[KB B200 client] Error searching: {e}")
            return []

    def delete_document_chunks(self, user_id, document_id) -> int:
        try:
            return self._call("delete_document_chunks", user_id, document_id)
        except Exception as e:
            logger.error(f"[KB B200 client] Error deleting chunks: {e}")
            return -1

    def delete_user_chunks(self, user_id) -> int:
        try:
            return self._call("delete_user_chunks", user_id)
        except Exception as e:
            logger.error(f"[KB B200 client] Error deleting user chunks: {e}")
            return -1

    def get_document_chunk_count(self, user_id, document_id) -> int:
        try:
            return self._call("get_document_chunk_count", user_id, document_id)
        except Exception:
            return 0

    def delete_discovery_chunks(self, org_id, before=None) -> int:
        try:
            return self._call("delete_discovery_chunks", org_id, before=before)
        except Exception:
            return 0

    def _get_weaviate_client(self):
        """(client, collection) facades for chat/background/rca_prompt_builder.py:276-317: ``collection.query.hybrid``
        and ``near_text`` run in the daemon; raises when it is unreachable (the caller returns "" then, :326-328)."""
        if not self.health().get("ready"):
            raise DaemonUnavailable(self._path)
        return SimpleNamespace(is_ready=lambda: True, close=lambda: None), SimpleNamespace(name="KnowledgeBaseChunk", query=_RemoteQuery(self))

    # ---- Aurora Learn (routes/incident_feedback/weaviate_client.py:165-386), same conventions
    def store_good_rca(self, user_id, incident_id, feedback_id, alert_title, alert_service, source_type, severity, aurora_summary,
                       thoughts, citations, org_id=None) -> bool:
        try:
            return bool(self._call("store_good_rca", user_id, incident_id, feedback_id, alert_title, alert_service, source_type, severity,
                                   aurora_summary, thoughts, citations, org_id=org_id))
        except Exception as e:
            logger.error(f"[AURORA LEARN B200 client] Error storing good RCA: {e}")
            return False

    def search_similar_good_rcas(self, user_id, alert_title, alert_service, source_type, limit=2, min_score=0.7):
        try:
            return self._call("search_similar_good_rcas", user_id, alert_title, alert_service, source_type, limit=limit, min_score=min_score)
        except Exception as e:
            logger.error(f"[AURORA LEARN B200 client] Error searching: {e}")
            return []

    def delete_incident_knowledge(self, user_id, incident_id) -> bool:
        try:
            return bool(self._call("delete_incident_knowledge", user_id, incident_id))
        except Exception:
            return False

    def delete_user_knowledge(self, user_id) -> int:
        try:
            return self._call("delete_user_knowledge", user_id)
        except Exception:
            return -1


if __name__ == "__main__":       # pragma: no cover
    import argparse

    ap = argparse.ArgumentParser(description="aurora_b200 engine daemon (configure the retriever first via AURORA_B200_BOOT)")
    ap.add_argument("--socket", default=os.getenv("AURORA_B200_SOCKET", "/tmp/aurora_b200.sock"))
    ap.add_argument("--boot", default=os.getenv("AURORA_B200_BOOT"), help="module:function that calls retriever.configure(...)")
    ap.add_argument("--snapshot", default=os.getenv("AURORA_B200_SNAPSHOT"), help="directory for periodic / shutdown snapshots")
    ap.add_argument("--save-every", type=int, default=2000, help="snapshot after this many inserts + deletes")
    ap.add_argument("--save-seconds", type=float, default=60.0, help="... or this long with unsaved mutations")
    ap.add_argument("--coalesce-us", type=int, default=200, help="gather concurrent searches for this long (0 = off)")
    a = ap.parse_args()
    if a.snapshot:
        os.environ["AURORA_B200_SNAPSHOT"] = a.snapshot      # the bootstrap restores from it and keeps the mutation log there
    if a.boot:
        mod, fn = a.boot.split(":")
        getattr(__import__(mod, fromlist=[fn]), fn)()
    from . import incident_knowledge as _learn

    serve(a.socket, learn_module=_learn, snapshot_dir=a.snapshot, save_every=a.save_every, save_seconds=a.save_seconds,
          coalesce_us=a.coalesce_us)

"""Drop-in for ``server/routes/incident_feedback/weaviate_client.py`` ("Aurora Learn") on the H100 engine.

Same four public functions, keyword arguments, return shapes and error conventions as the reference
(file:line cited on each).  This is the consumer whose score IS the engine's cosine: the reference runs
``collection.query.near_text(...)`` and reports ``similarity = 1 - distance`` (``:286-297``), keeps
matches with ``similarity >= min_score`` (``:302``, default 0.7) and rounds to three decimals (``:318``).

Underneath: a second chunk store (``aurora_b200.retriever.KnowledgeBase``, collection
``IncidentKnowledge``) -- vectors in an HBM shard searched by the fused similarity + top-k kernels, the
properties in a host table.  The org / user scope is a metadata pre-filter resolved to the set of allowed
rows before the kernel runs, as in Weaviate.

Documented deviation: the embedded text is the concatenation of the vectorised properties the reference
declares (``alert_title, alert_service, source_type, severity, aurora_summary``; the others carry
``skip_vectorization=True``, ``:139-152``) in declaration order; Weaviate's text2vec module also prepends
the class name and lower-cases, which only that container defines.
"""

from __future__ import annotations

import json
import logging
import os
import threading
from datetime import datetime, timezone
from typing import Any, Callable, Dict, List, Optional

from .filters import Filter
from .retriever import KnowledgeBase, _sanitize, generate_uuid5

logger = logging.getLogger(__name__)

COLLECTION_NAME = "IncidentKnowledge"   # incident_feedback/weaviate_client.py:25
_VECTORISED = ("alert_title", "alert_service", "source_type", "severity", "aurora_summary")


def _parse_json_field(value: str) -> list:
    """incident_feedback/weaviate_client.py:28-33: a JSON string field, [] on failure."""
    try:
        return json.loads(value)
    except (json.JSONDecodeError, TypeError):
        return []


def _embedded_text(props: Dict[str, Any]) -> str:
    return " ".join(str(props.get(name, "")) for name in _VECTORISED)


# ---------------------------------------------------------------------- module state
_kb: Optional[KnowledgeBase] = None
_kb_factory: Optional[Callable[[], KnowledgeBase]] = None
_org_resolver: Optional[Callable[[str], Optional[str]]] = None
_client_lock = threading.Lock()          # the reference guards client creation the same way (:44, :63-81)


def configure(encoder=None, capacity: Optional[int] = None, device: Optional[int] = None, index_factory=None,
              factory: Optional[Callable[[], KnowledgeBase]] = None,
              org_resolver: Optional[Callable[[str], Optional[str]]] = None) -> None:
    """Install the backend.  ``org_resolver(user_id) -> org_id | None`` stands in for
    ``utils.auth.stateless_auth.get_org_id_for_user`` (``:276-277``); when omitted that function is
    imported lazily, exactly like the reference does."""
    global _kb, _kb_factory, _org_resolver
    with _client_lock:
        _kb = None
        _org_resolver = org_resolver
        if factory is not None:
            _kb_factory = factory
            return
        cap = capacity if capacity is not None else int(os.getenv("AURORA_B200_LEARN_CAPACITY", str(1 << 16)))
        dev = device if device is not None else int(os.getenv("AURORA_B200_DEVICE", "0"))
        _kb_factory = lambda: KnowledgeBase(encoder, capacity=cap, device=dev, index_factory=index_factory)  # noqa: E731


def _get_kb() -> KnowledgeBase:
    global _kb
    with _client_lock:
        if _kb is None:
            if _kb_factory is None:
                raise RuntimeError("aurora_b200.incident_knowledge is not configured: call configure(encoder=...) first")
            _kb = _kb_factory()
        return _kb


def _org_of(user_id: str) -> Optional[str]:
    if _org_resolver is not None:
        return _org_resolver(user_id)
    from utils.auth.stateless_auth import get_org_id_for_user   # the reference's own lookup (:276)

    return get_org_id_for_user(user_id)


# ---------------------------------------------------------------------- public API (reference signatures)
def store_good_rca(user_id: str, incident_id: str, feedback_id: str, alert_title: str, alert_service: str,
                   source_type: str, severity: str, aurora_summary: str, thoughts: List[Dict[str, Any]],
                   citations: List[Dict[str, Any]], org_id: str = None) -> bool:
    """incident_feedback/weaviate_client.py:165-243.  One object per (user, incident) -- deterministic
    uuid5 (``:214``) so a second positive rating replaces the first; True on success, False on any error."""
    try:
        kb = _get_kb()
        now = datetime.now(timezone.utc).isoformat()
        thoughts_text = "\n".join([t.get("content", "") for t in thoughts])
        full_context = (f"Alert: {alert_title}\nService: {alert_service}\nSource: {source_type}\nSeverity: {severity}\n\n"
                        f"Summary:\n{aurora_summary}\n\nInvestigation:\n{thoughts_text}").strip()       # :199-211
        key = generate_uuid5(f"{user_id}:{incident_id}")
        props = {
            "user_id": user_id, "org_id": org_id or "", "incident_id": incident_id, "feedback_id": feedback_id,
            "alert_title": alert_title, "alert_service": alert_service or "unknown", "source_type": source_type,
            "severity": severity or "unknown", "aurora_summary": aurora_summary, "thoughts": json.dumps(thoughts),
            "citations": json.dumps(citations), "full_context": full_context, "created_at": now,
        }
        kb.insert_objects([(key, props, _embedded_text(props))], user_id, org_id or None)
        logger.info(f"[AURORA LEARN B200] Stored good RCA for incident {_sanitize(incident_id)} (user: {_sanitize(user_id)})")
        return True
    except Exception as e:
        logger.error(f"[AURORA LEARN B200] Error storing good RCA: {e}")
        return False


def search_similar_good_rcas(user_id: str, alert_title: str, alert_service: str, source_type: str, limit: int = 2,
                             min_score: float = 0.7) -> List[Dict[str, Any]]:
    """incident_feedback/weaviate_client.py:246-328.  Pure dense cosine top-``limit`` inside the caller's
    org (user when it has none); ``similarity = 1 - distance``; matches under ``min_score`` dropped;
    ``round(similarity, 3)``; any exception -> []."""
    try:
        kb = _get_kb()
        search_query = f"Alert: {alert_title} Service: {alert_service} Source: {source_type}"          # :274
        org_id = _org_of(user_id)
        if org_id:
            search_filter = Filter.by_property("org_id").equal(org_id)                                  # :279-280
        else:
            logger.warning("No org_id found for user %s, falling back to user_id filter", _sanitize(user_id))
            search_filter = Filter.by_property("user_id").equal(user_id)                                # :283
        objs = kb.query(search_query, limit, filters=search_filter)                                     # near_text, :286-291
        results = []
        for obj in objs:
            distance = obj.metadata.distance if obj.metadata and obj.metadata.distance is not None else 1.0
            similarity = 1.0 - distance                                                                 # :296-297
            if similarity < min_score:                                                                  # :302
                continue
            p = obj.properties
            results.append({
                "incident_id": p.get("incident_id", ""), "alert_title": p.get("alert_title", ""),
                "alert_service": p.get("alert_service", ""), "source_type": p.get("source_type", ""),
                "severity": p.get("severity", ""), "aurora_summary": p.get("aurora_summary", ""),
                "thoughts": _parse_json_field(p.get("thoughts", "[]")),
                "citations": _parse_json_field(p.get("citations", "[]")),
                "similarity": round(similarity, 3),                                                     # :318
            })
        logger.info(f"[AURORA LEARN B200] Search for '{_sanitize(alert_title)[:30]}...' returned {len(results)} matches "
                    f"(min_score={min_score})")
        return results
    except Exception as e:
        logger.error(f"[AURORA LEARN B200] Error searching for similar RCAs: {e}")
        return []


def delete_incident_knowledge(user_id: str, incident_id: str) -> bool:
    """incident_feedback/weaviate_client.py:331-361.  True unless the backend failed."""
    try:
        f = Filter.by_property("user_id").equal(user_id) & Filter.by_property("incident_id").equal(incident_id)
        n = _get_kb().delete_where(f)
        logger.info(f"[AURORA LEARN B200] Deleted {n} knowledge entries for incident {_sanitize(incident_id)}")
        return True
    except Exception as e:
        logger.error(f"[AURORA LEARN B200] Error deleting incident knowledge: {e}")
        return False


def delete_user_knowledge(user_id: str) -> int:
    """incident_feedback/weaviate_client.py:364-386.  Deleted count; -1 on error."""
    try:
        n = _get_kb().delete_where(Filter.by_property("user_id").equal(user_id))
        logger.info(f"[AURORA LEARN B200] Deleted {n} knowledge entries for user {_sanitize(user_id)}")
        return n
    except Exception as e:
        logger.error(f"[AURORA LEARN B200] Error deleting user knowledge: {e}")
        return -1

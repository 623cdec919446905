"""Title similarity of alert correlation: the reference's ``SimilarityStrategy``
(server/services/correlation/strategies/similarity.py) restated over ``aurora_b200.encoder``'s embedding client, plus
batched scoring of many candidates in one device call.

``score`` keeps the reference's per-candidate behaviour: an empty title scores 0.0; otherwise the title similarity is
the clamped cosine of the two titles' embeddings (two ``embed`` calls and a pure-Python cosine), or the Jaccard index of
their word sets when either embedding is None; the service similarity is 1.0 for an exact match, else the Jaccard index
of the service names' tokens; the score is 0.7 * title + 0.3 * service.

``score_many`` / ``score_alerts`` give the same numbers (to within fp64 rounding of the cosine) for all the candidates of
one alert / of many alerts with ONE ``EmbeddingClient.similarities`` call: every distinct title encoded once, every
cosine computed on the device.  A client without ``similarities`` (a reference-style HTTP client) is scored pair by pair
through ``score``; a client with ``similarity_scores`` (``aurora_b200.daemon.Client``) hands the whole call to the
engine daemon, which batches it there.
"""

from __future__ import annotations

import logging
import math
import re
from typing import List, Optional, Sequence, Set, Tuple

from .encoder import get_embedding_client

logger = logging.getLogger(__name__)

STOPWORDS: Set[str] = {"the", "a", "an", "is", "are", "was", "for", "in", "on", "at"}   # similarity.py:19
TOKEN_RE = re.compile(r"[a-z0-9]+")                                                        # similarity.py:20

Candidate = Tuple[str, Sequence[str]]                       # (incident title, incident services)
Alert = Tuple[str, str, Sequence[Candidate]]               # (alert title, alert service, candidates)


class SimilarityStrategy:
    """Vector similarity of titles with service-name overlap (similarity.py:23-153)."""

    TITLE_WEIGHT = 0.7
    SERVICE_WEIGHT = 0.3

    def score(self, alert_title: str, alert_service: str, incident_title: str, incident_services: List[str]) -> float:
        """similarity.py:29-64: 0.0 when either title is empty, else TITLE_WEIGHT * title + SERVICE_WEIGHT * service."""
        if not alert_title or not incident_title:
            logger.warning("[SimilarityStrategy] Empty title input - alert_title=%r, incident_title=%r", bool(alert_title),
                           bool(incident_title))
            return 0.0
        title_sim = self._vector_similarity(alert_title, incident_title)
        if title_sim is None:
            title_sim = self._jaccard_similarity(alert_title, incident_title)
        return self.TITLE_WEIGHT * title_sim + self.SERVICE_WEIGHT * self._service_similarity(alert_service, incident_services)

    def score_many(self, alert_title: str, alert_service: str, candidates: Sequence[Candidate]) -> List[float]:
        """``score`` of every candidate (incident_title, incident_services) of one alert, in one ``similarities`` call."""
        return self.score_alerts([(alert_title, alert_service, candidates)])[0]

    def score_alerts(self, items: Sequence[Alert]) -> List[List[float]]:
        """``score_many`` of several alerts (alert_title, alert_service, candidates), all their pairs in one
        ``similarities`` call; element [i][j] is the score of alert i against its candidate j."""
        try:
            client = get_embedding_client()
        except Exception as e:                     # as _vector_similarity: no client -> every title by Jaccard
            logger.debug("[SimilarityStrategy] Vector similarity failed: %s", e)
            client = None
        remote = getattr(client, "similarity_scores", None)
        if remote is not None:
            return remote(items)
        if getattr(client, "similarities", None) is None:
            return [[self.score(title, service, c[0], c[1]) for c in cands] for title, service, cands in items]
        return self.weigh(items, client.similarities)

    def weigh(self, items: Sequence[Alert], similarities) -> List[List[float]]:
        """``score_alerts`` with the title cosines of the pairs with two non-empty titles from ``similarities(pairs)``
        (a None, or every pair when it raises, falls back to Jaccard)."""
        pairs = [(title, c[0]) for title, _, cands in items if title for c in cands if c[0]]
        sims: List[Optional[float]] = [None] * len(pairs)
        if pairs:
            try:
                sims = list(similarities(pairs))
            except Exception as e:
                logger.debug("[SimilarityStrategy] Vector similarity failed: %s", e)
        it = iter(sims)
        out = []
        for title, service, cands in items:
            row = []
            for inc_title, inc_services in cands:
                if not title or not inc_title:
                    row.append(0.0)
                    continue
                t = next(it)
                if t is None:
                    t = self._jaccard_similarity(title, inc_title)
                row.append(self.TITLE_WEIGHT * t + self.SERVICE_WEIGHT * self._service_similarity(service, inc_services))
            out.append(row)
        return out

    def _vector_similarity(self, text_a: str, text_b: str) -> Optional[float]:
        """similarity.py:66-83: None when an embedding is missing or anything fails."""
        try:
            client = get_embedding_client()
            vec_a = client.embed(text_a)
            vec_b = client.embed(text_b)
            if vec_a is None or vec_b is None:
                return None
            return self._cosine_similarity(vec_a, vec_b)
        except Exception as e:
            logger.debug("[SimilarityStrategy] Vector similarity failed: %s", e)
            return None

    @staticmethod
    def _cosine_similarity(vec_a: List[float], vec_b: List[float]) -> float:
        """similarity.py:84-98: builtin sums in Python floats, 0.0 for unequal or zero lengths and zero norms, clamped
        to [0, 1]."""
        if len(vec_a) != len(vec_b) or len(vec_a) == 0:
            return 0.0
        dot = sum(a * b for a, b in zip(vec_a, vec_b))
        norm_a = math.sqrt(sum(a * a for a in vec_a))
        norm_b = math.sqrt(sum(b * b for b in vec_b))
        if norm_a == 0 or norm_b == 0:
            return 0.0
        return max(0.0, min(1.0, dot / (norm_a * norm_b)))

    def _jaccard_similarity(self, text_a: str, text_b: str) -> float:
        return self._jaccard(self._tokenize(text_a), self._tokenize(text_b))

    @staticmethod
    def _tokenize(text: str) -> Set[str]:
        """Lower-cased [a-z0-9]+ words without stop-words and one-character words."""
        return {t for t in TOKEN_RE.findall(text.lower()) if t not in STOPWORDS and len(t) >= 2}

    @staticmethod
    def _jaccard(set_a: Set[str], set_b: Set[str]) -> float:
        union = set_a | set_b
        return len(set_a & set_b) / len(union) if union else 0.0

    @staticmethod
    def _service_similarity(alert_service: str, incident_services: List[str]) -> float:
        """similarity.py:124-153: 0.0 when either side is empty, 1.0 for an exact match, else the Jaccard index of the
        service names' words (stop-words and one-character words dropped)."""
        if not alert_service or not incident_services:
            logger.warning("[SimilarityStrategy] Empty service input - alert_service=%r, incident_services=%r",
                           bool(alert_service), bool(incident_services))
            return 0.0
        if alert_service in incident_services:
            return 1.0
        alert_tokens = SimilarityStrategy._tokenize(alert_service)
        incident_tokens: Set[str] = set()
        for svc in incident_services:
            incident_tokens |= SimilarityStrategy._tokenize(svc)
        if not alert_tokens or not incident_tokens:
            return 0.0
        return len(alert_tokens & incident_tokens) / len(alert_tokens | incident_tokens)

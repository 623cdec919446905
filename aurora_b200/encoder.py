"""Python handle over the CUDA text encoder (C ABI: aur_encoder_* in include/aurora_b200.h) and
the host-side mirror of the reference's embedding client.

Reference surface mirrored here: ``EmbeddingClient.embed / embed_batch / close`` and
``get_embedding_client()`` (server/services/correlation/embedding_client.py:20-84): ``None`` for
blank text or any failure, a list of floats otherwise.  The reference posts the text to a
t2v-transformers sidecar; here the forward pass runs in-process on the GPU.  Tokenisation is the
caller's (a ``tokenize(text) -> list[int]`` callable): a WordPiece tokenizer needs a vocabulary
file, which is deployment data, not code (SURVEY.md section 8(f) item 2).
"""

from __future__ import annotations

import ctypes as C
import logging
from dataclasses import dataclass
from functools import lru_cache
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _native as N

logger = logging.getLogger(__name__)

POOL = {"cls": 0, "mean": 1}


@dataclass(frozen=True)
class EncoderConfig:
    hidden: int = 768
    layers: int = 12
    heads: int = 12
    inter: int = 3072
    vocab: int = 30522
    max_pos: int = 512
    type_vocab: int = 2
    ln_eps: float = 1e-12
    pool: str = "cls"
    normalize: bool = True


BGE_BASE = EncoderConfig()
MINILM_L6 = EncoderConfig(hidden=384, layers=6, heads=12, inter=1536, pool="mean")   # head dim 32, zero-padded to 64 on the device
BGE_LARGE = EncoderConfig(hidden=1024, layers=24, heads=16, inter=4096)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def pack_sequences(seqs: Sequence[Sequence[int]]):
    """list of token-id lists -> (tokens int32 [total], cu_seqlens int32 [n+1])."""
    lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=len(seqs))
    cu = np.zeros(len(seqs) + 1, dtype=np.int32)
    cu[1:] = np.cumsum(lens)
    tok = np.empty(int(cu[-1]), dtype=np.int32)
    for i, s in enumerate(seqs):
        tok[cu[i]:cu[i + 1]] = s
    return tok, cu


class Encoder:
    """BERT-family encoder resident on one GPU: packed token ids in, pooled vectors out."""

    def __init__(self, cfg: EncoderConfig, max_tokens: int = 32768, max_seqs: int = 2048, device: int = 0):
        self._lib = N.load()
        self.cfg, self.device = cfg, int(device)
        self.max_tokens, self.max_seqs = int(max_tokens), int(max_seqs)
        self._h = C.c_void_p()
        c = N.AurEncoderConfig(device=self.device, hidden=cfg.hidden, layers=cfg.layers, heads=cfg.heads, inter=cfg.inter,
                               vocab=cfg.vocab, max_pos=cfg.max_pos, type_vocab=cfg.type_vocab, pool=POOL[cfg.pool],
                               normalize=int(cfg.normalize), max_tokens=self.max_tokens, max_seqs=self.max_seqs,
                               ln_eps=cfg.ln_eps, reserved=0)
        N.check(self._lib.aur_encoder_open(C.byref(c), C.byref(self._h)))

    def replicate(self, device: int) -> "Encoder":
        """A second encoder on ``device`` (this one's too) with this one's parameters, copied device to device
        (aur_encoder_replicate): its forward is this one's bit for bit, and it outlives this one."""
        h = C.c_void_p()
        N.check(self._lib.aur_encoder_replicate(self._h, int(device), C.byref(h)))
        r = Encoder.__new__(Encoder)
        r._lib, r.cfg, r.device, r.max_tokens, r.max_seqs, r._h = self._lib, self.cfg, int(device), self.max_tokens, self.max_seqs, h
        return r

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.aur_encoder_close(self._h)
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

    # -------------------------------------------------------------- parameters
    def load_weights(self, weights: Dict[str, np.ndarray]) -> None:
        """Names and shapes as documented at aur_encoder_load (torch.nn.Linear layout)."""
        for name, w in weights.items():
            a = np.ascontiguousarray(w, dtype=np.float32)
            N.check(self._lib.aur_encoder_load(self._h, name.encode(), _ptr(a), a.size))

    # -------------------------------------------------------------- forward
    def _check_batch(self, tokens, cu):
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        cu = np.ascontiguousarray(cu, dtype=np.int32)
        if cu.ndim != 1 or cu.size < 2 or tokens.ndim != 1 or tokens.size != int(cu[-1]):
            raise ValueError("tokens [total] and cu_seqlens [n_seq + 1] with cu[-1] == total are required")
        return tokens, cu

    def encode_packed(self, tokens: np.ndarray, cu_seqlens: np.ndarray, bf16: bool = False) -> np.ndarray:
        """[n_seq, hidden] float32 (or raw bf16 bits as uint16 when ``bf16``)."""
        tokens, cu = self._check_batch(tokens, cu_seqlens)
        n = cu.size - 1
        out = np.empty((n, self.cfg.hidden), dtype=np.uint16 if bf16 else np.float32)
        N.check(self._lib.aur_encode(self._h, _ptr(tokens), _ptr(cu), n, None if bf16 else _ptr(out),
                                     _ptr(out) if bf16 else None))
        return out

    def encode_texts(self, tokens: np.ndarray, cu_seqlens: np.ndarray, cu_texts: np.ndarray, bf16: bool = False) -> np.ndarray:
        """aur_encode_texts: [n_texts, hidden] float32 (raw bf16 bits as uint16 when ``bf16``), text j the vector of windows
        cu_texts[j] .. cu_texts[j + 1] - 1 (its one window's, or their mean, DESIGN.md section 4.5); any number of
        windows, batched through the workspace inside the library."""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        cu = np.ascontiguousarray(cu_seqlens, dtype=np.int32)
        ct = np.ascontiguousarray(cu_texts, dtype=np.int32)
        if cu.ndim != 1 or cu.size < 1 or ct.ndim != 1 or ct.size < 1 or tokens.ndim != 1 or tokens.size != int(cu[-1]):
            raise ValueError("tokens [total], cu_seqlens [n_seq + 1] with cu[-1] == total and cu_texts [n_texts + 1] are required")
        out = np.empty((ct.size - 1, self.cfg.hidden), dtype=np.uint16 if bf16 else np.float32)
        N.check(self._lib.aur_encode_texts(self._h, _ptr(tokens), _ptr(cu), cu.size - 1, _ptr(ct), ct.size - 1,
                                           None if bf16 else _ptr(out), _ptr(out) if bf16 else None))
        return out

    def pair_cosines(self, tokens: np.ndarray, cu_seqlens: np.ndarray, cu_texts: np.ndarray, pair_a, pair_b,
                     clamp: bool = True, vectors: bool = False):
        """aur_encode_pair_cosines: [n_pairs] float64 cosines of texts pair_a[p] and pair_b[p] (texts packed as for
        ``encode_texts``), equal bit for bit to ``engine.cosine_pairs`` over ``encode_texts``' vectors with the same
        ``clamp``; one call, the vectors never leave the device.  ``vectors``: also return those vectors,
        (cosines, [n_texts, hidden] float32)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        cu = np.ascontiguousarray(cu_seqlens, dtype=np.int32)
        ct = np.ascontiguousarray(cu_texts, dtype=np.int32)
        if cu.ndim != 1 or cu.size < 1 or ct.ndim != 1 or ct.size < 1 or tokens.ndim != 1 or tokens.size != int(cu[-1]):
            raise ValueError("tokens [total], cu_seqlens [n_seq + 1] with cu[-1] == total and cu_texts [n_texts + 1] are required")
        pa = np.ascontiguousarray(pair_a, dtype=np.int32)
        pb = np.ascontiguousarray(pair_b, dtype=np.int32)
        if pa.ndim != 1 or pa.shape != pb.shape:
            raise ValueError("pair_a and pair_b must be 1-d and of one length")
        cos = np.empty(pa.size, dtype=np.float64)
        vec = np.empty((ct.size - 1, self.cfg.hidden), dtype=np.float32) if vectors else None
        N.check(self._lib.aur_encode_pair_cosines(self._h, _ptr(tokens), _ptr(cu), cu.size - 1, _ptr(ct), ct.size - 1, _ptr(pa),
                                                  _ptr(pb), pa.size, int(bool(clamp)), _ptr(cos), _ptr(vec)))
        return (cos, vec) if vectors else cos

    def encode(self, seqs: Sequence[Sequence[int]]) -> np.ndarray:
        """Token-id lists of any count, [len(seqs), hidden] float32: one ``encode_texts`` call with one window per text,
        cut into workspace batches inside the library."""
        for i, s in enumerate(seqs):
            if len(s) > self.max_tokens:
                raise ValueError(f"sequence {i} has {len(s)} tokens: more than max_tokens={self.max_tokens}")
        tok, cu = pack_sequences(seqs)
        return self.encode_texts(tok, cu, np.arange(len(seqs) + 1, dtype=np.int32))

    def encode_append(self, index, tokens: np.ndarray, cu_seqlens: np.ndarray, ids: np.ndarray,
                      user_codes: Optional[np.ndarray] = None, org_codes: Optional[np.ndarray] = None) -> None:
        """Fused ingest: encode and append to ``index`` (engine.Index) without leaving the device."""
        tokens, cu = self._check_batch(tokens, cu_seqlens)
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        u = None if user_codes is None else np.ascontiguousarray(user_codes, dtype=np.int32)
        o = None if org_codes is None else np.ascontiguousarray(org_codes, dtype=np.int32)
        N.check(self._lib.aur_encode_append(self._h, index._h, _ptr(tokens), _ptr(cu), cu.size - 1, _ptr(ids), _ptr(u), _ptr(o)))

    def stats(self) -> dict:
        st = N.AurEncoderStats()
        N.check(self._lib.aur_encoder_get_stats(self._h, C.byref(st)))
        return {k: getattr(st, k) for k, _ in st._fields_}

    def hidden_states(self) -> np.ndarray:
        """Final hidden states [tokens, hidden] (bf16 bits) of the last call (test hook)."""
        t = self.stats()["tokens"]
        out = np.empty((t, self.cfg.hidden), dtype=np.uint16)
        N.check(self._lib.aur_debug_encoder_hidden(self._h, _ptr(out), out.size))
        return out


def encode_append_multi(encoders: Sequence[Encoder], shards, tokens: np.ndarray, cu_seqlens: np.ndarray, ids: np.ndarray,
                        user_codes: Optional[np.ndarray] = None, org_codes: Optional[np.ndarray] = None,
                        max_tokens_per_call: int = 0, max_seqs_per_call: int = 0, cu_texts: Optional[np.ndarray] = None) -> None:
    """aur_encode_append_multi: packed sequences encoded and appended to ``shards`` (``engine.Index`` on their encoders'
    devices) placed by ``id mod len(shards)``, sequence i by ``encoders[ids[i] % n]``; every shard's share at once,
    in workspace batches (0 = the encoder's workspace).  With ``cu_texts`` (aur_encode_append_texts_multi) the unit is
    the text: text j is windows cu_texts[j] .. cu_texts[j + 1] - 1, stored as ``Encoder.encode_texts`` gives it, and
    ids / user_codes / org_codes are per text."""
    n = len(shards)
    if len(encoders) != n:
        raise ValueError(f"{len(encoders)} encoders for {n} shards")
    tokens = np.ascontiguousarray(tokens, dtype=np.int32)
    cu = np.ascontiguousarray(cu_seqlens, dtype=np.int32)
    if cu.ndim != 1 or cu.size < 1 or tokens.ndim != 1 or tokens.size != int(cu[-1]):
        raise ValueError("tokens [total] and cu_seqlens [n_seq + 1] with cu[-1] == total are required")
    ct = None if cu_texts is None else np.ascontiguousarray(cu_texts, dtype=np.int32)
    n_units = cu.size - 1 if ct is None else ct.size - 1
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    if ids.shape != (n_units,):
        raise ValueError("ids must be [n_seq] ([n_texts] with cu_texts)")
    u = None if user_codes is None else np.ascontiguousarray(user_codes, dtype=np.int32)
    o = None if org_codes is None else np.ascontiguousarray(org_codes, dtype=np.int32)
    encs = (C.c_void_p * n)(*[e._h.value for e in encoders])
    hs = (C.c_void_p * n)(*[sh._h.value for sh in shards])
    lib = N.load()
    if ct is None:
        N.check(lib.aur_encode_append_multi(encs, hs, n, _ptr(tokens), _ptr(cu), cu.size - 1, _ptr(ids), _ptr(u), _ptr(o),
                                            int(max_tokens_per_call), int(max_seqs_per_call)))
    else:
        N.check(lib.aur_encode_append_texts_multi(encs, hs, n, _ptr(tokens), _ptr(cu), cu.size - 1, _ptr(ct), n_units, _ptr(ids),
                                                  _ptr(u), _ptr(o), int(max_tokens_per_call), int(max_seqs_per_call)))


class TextEncoder:
    """Adapter for aurora_b200.retriever.KnowledgeBase: ``dim`` + ``encode(texts)`` over a tokenizer and the CUDA
    ``Encoder``; ``encode_append`` is the fused ingest path (vectors never leave the device between the forward
    pass and the shard append).  ``replicate(devices)`` adds one encoder per further device, so that the fused path
    also serves an ``engine.MultiIndex`` with every shard's share encoded on the shard's own GPU; queries
    (``encode``) stay on the primary encoder.

    ``tokenizer``: an ``aurora_b200.wordpiece.NativeTokenizer`` (C++, multi-threaded -- then a whole batch is tokenised
    in ONE C call, with no Python per text) or any ``tokenize(text) -> list[int]`` callable.

    Texts longer than the position table (the reference's chunker can emit a 4 000-character chunk,
    document_processor.py:266-267) are not cut off: they are split into windows of ``max_pos`` tokens, each window is
    encoded, and the text's vector is the L2-normalised mean of its windows -- the same idea as the t2v sidecar's
    sentence batching + averaging (that container's exact splitting rule is not in the reference tree).  Windows,
    forward, mean and append all stay in the library and on the device (``aur_tokenize_windows``, ``aur_encode_texts``,
    ``aur_encode_append_texts_multi``; the arithmetic is in DESIGN.md section 4.5)."""

    def __init__(self, encoder: Encoder, tokenizer, max_len: Optional[int] = None):
        self._enc, self._tok = encoder, tokenizer
        self._native = hasattr(tokenizer, "encode_packed")
        self.dim = encoder.cfg.hidden
        self.max_len = int(max_len or encoder.cfg.max_pos)
        self._encs: Dict[int, Encoder] = {encoder.device: encoder}    # device -> the encoder that appends there

    def replicate(self, devices) -> "TextEncoder":
        """Keep one encoder on each of ``devices``: the primary for its own device, a replica (``Encoder.replicate``,
        the same parameters copied device to device) for every other.  Returns self."""
        for d in devices:
            if int(d) not in self._encs:
                self._encs[int(d)] = self._enc.replicate(int(d))
        return self

    @staticmethod
    def _shards(index) -> list:
        from .engine import MultiIndex

        return list(index.shards) if isinstance(index, MultiIndex) else [index]

    def can_append(self, index) -> bool:
        """Whether ``encode_append`` takes ``index``: an ``engine.Index``, or a ``MultiIndex`` of them, bf16 or int8,
        ``dim`` wide, with an encoder on every shard's device."""
        from .engine import Index

        shards = self._shards(index)
        return bool(shards) and all(isinstance(sh, Index) and sh.dtype != N.AUR_F32 and sh.dim == self.dim
                                    and sh.device in self._encs for sh in shards)

    # ------------------------------------------------------------------ tokenisation
    def _tokenize_windows(self, texts: Sequence[str]):
        """(tokens, cu_seqlens over windows, cu_texts): one C call with the native tokenizer, ``_windows`` per text
        with a callable one."""
        if self._native:
            return self._tok.encode_windows(list(texts), self.max_len)
        wins = [self._windows(t) for t in texts]
        cu_texts = np.zeros(len(texts) + 1, dtype=np.int32)
        cu_texts[1:] = np.cumsum([len(w) for w in wins])
        tok, cu = pack_sequences([s for w in wins for s in w])
        return tok, cu, cu_texts

    def _windows(self, text: str):
        """Token windows of one text: [CLS] body[i : i + max_len - 2] [SEP] for i = 0, max_len - 2, ... (one window
        when the text fits).  The Python statement of aur_tokenize_windows' rule."""
        if self._native:
            tok, cu = self._tok.encode_packed([text], int(self._tok.lengths([text], max_len=0x7FFFFFFF)[0]))   # the whole text
        else:
            tok, cu = pack_sequences([list(self._tok(text))])
        ids = tok[cu[0]:cu[1]]
        cls, sep, body = ids[0], ids[-1], ids[1:-1]
        step = self.max_len - 2
        return [np.concatenate(([cls], body[i:i + step], [sep])).astype(np.int32) for i in range(0, max(len(body), 1), step)]

    # ------------------------------------------------------------------ API used by the retriever
    def encode(self, texts: Sequence[str]) -> np.ndarray:
        """[len(texts), dim] float32: one tokenisation and one aur_encode_texts call (windows, batches and the mean of
        an over-long text's windows inside the library)."""
        return self._enc.encode_texts(*self._tokenize_windows(texts))

    def encode_append(self, index, texts: Sequence[str], ids: np.ndarray, user_codes=None, org_codes=None) -> None:
        """Tokenise once (one multi-threaded C call with the native tokenizer), then ONE aur_encode_append_texts_multi
        call: workspace batches, encoder forward, the mean of an over-long text's windows and the shard append inside
        the library, each shard's share on its own device in input order (``can_append`` says which indexes qualify);
        nothing runs per text or per batch in Python and no vector leaves the device."""
        if not self.can_append(index):
            raise ValueError("encode_append needs bf16 or int8 engine.Index shards on devices this encoder has replicas on")
        tok, cu, cu_texts = self._tokenize_windows(texts)
        shards = self._shards(index)
        encode_append_multi([self._encs[sh.device] for sh in shards], shards, tok, cu, ids, user_codes, org_codes,
                            cu_texts=cu_texts)


# ----------------------------------------------------------------------------- reference mirror
class EmbeddingClient:
    """Drop-in for server/services/correlation/embedding_client.py:20-78 backed by ``Encoder``."""

    def __init__(self, encoder: Encoder, tokenize: Callable[[str], List[int]]):
        self._enc, self._tok = encoder, tokenize

    def embed(self, text: str) -> Optional[List[float]]:
        if not text or not text.strip():                      # embedding_client.py:48-49
            return None
        try:
            return self._enc.encode([self._tok(text)])[0].tolist()
        except Exception as e:                                  # embedding_client.py:66-70: any failure -> None
            logger.warning("[EmbeddingClient] embed failed: %s", e)
            return None

    def embed_batch(self, texts: List[str]) -> List[Optional[List[float]]]:
        """One batched forward instead of the reference's per-text loop (embedding_client.py:72-74);
        blank texts and failures still map to None per element."""
        idx = [i for i, t in enumerate(texts) if t and t.strip()]
        out: List[Optional[List[float]]] = [None] * len(texts)
        if not idx:
            return out
        try:
            vecs = self._enc.encode([self._tok(texts[i]) for i in idx])
            for j, i in enumerate(idx):
                out[i] = vecs[j].tolist()
        except Exception as e:
            logger.warning("[EmbeddingClient] embed_batch failed: %s", e)
        return out

    def similarities(self, pairs: Sequence[Tuple[str, str]]) -> List[Optional[float]]:
        """Clamped cosine of each pair's two texts, from the vectors ``embed`` would return for them, in ONE
        ``Encoder.pair_cosines`` call instead of two ``embed`` calls and a Python cosine per pair: every distinct text
        is tokenised and encoded once.  A pair holding a text ``embed`` answers None for (blank, a tokenizer error, a
        sequence of 0 or more than max_pos tokens, a token id outside the vocabulary) is None, and the other pairs are
        unaffected; a failed device call makes every pair None, as the serial path is when every ``embed`` fails."""
        cfg = self._enc.cfg
        limit = min(cfg.max_pos, self._enc.max_tokens)
        seq: Dict[str, Optional[np.ndarray]] = {}          # text -> its one sequence, None when embed would give None
        for pair in pairs:
            for t in pair:
                if t in seq:
                    continue
                seq[t] = None
                if not t or not t.strip():
                    continue
                try:
                    ids = np.asarray(self._tok(t), dtype=np.int64)
                except Exception as e:                          # embed: any failure -> None
                    logger.warning("[EmbeddingClient] tokenize failed: %s", e)
                    continue
                if ids.ndim == 1 and 1 <= ids.size <= limit and ids.min() >= 0 and ids.max() < cfg.vocab:
                    seq[t] = ids.astype(np.int32)
        out: List[Optional[float]] = [None] * len(pairs)
        live = [p for p, (a, b) in enumerate(pairs) if seq[a] is not None and seq[b] is not None]
        if not live:
            return out
        row: Dict[str, int] = {}
        for p in live:
            for t in pairs[p]:
                row.setdefault(t, len(row))
        try:
            tok, cu = pack_sequences([seq[t] for t in row])
            cos = self._enc.pair_cosines(tok, cu, np.arange(len(row) + 1, dtype=np.int32), [row[pairs[p][0]] for p in live],
                                         [row[pairs[p][1]] for p in live], clamp=True)
        except Exception as e:
            logger.warning("[EmbeddingClient] similarities failed: %s", e)
            return out
        for p, c in zip(live, cos.tolist()):
            out[p] = c
        return out

    def close(self) -> None:                                   # embedding_client.py:76-78
        self._enc.close()


_factory: Optional[Callable[[], EmbeddingClient]] = None


def configure_embedding_client(factory: Callable[[], EmbeddingClient]) -> None:
    """Deployment hook: how to build the process-wide client (weights, tokenizer, device)."""
    global _factory
    _factory = factory
    get_embedding_client.cache_clear()


@lru_cache(maxsize=1)
def get_embedding_client() -> EmbeddingClient:                 # embedding_client.py:81-84
    if _factory is None:
        raise RuntimeError("call aurora_b200.encoder.configure_embedding_client(factory) first")
    return _factory()


# ----------------------------------------------------------------------------- checkpoint loading
def read_safetensors(path: str) -> Dict[str, np.ndarray]:
    """Minimal safetensors reader (8-byte little-endian header length, JSON header, raw tensors):
    F32 / F16 / BF16 tensors come back as float32 arrays.  No third-party dependency."""
    import json
    import struct

    out: Dict[str, np.ndarray] = {}
    with open(path, "rb") as f:
        (hlen,) = struct.unpack("<Q", f.read(8))
        header = json.loads(f.read(hlen))
        base = 8 + hlen
        for name, info in header.items():
            if name == "__metadata__":
                continue
            lo, hi = info["data_offsets"]
            f.seek(base + lo)
            raw = f.read(hi - lo)
            dt = info["dtype"]
            if dt == "F32":
                a = np.frombuffer(raw, dtype=np.float32)
            elif dt == "F16":
                a = np.frombuffer(raw, dtype=np.float16).astype(np.float32)
            elif dt == "BF16":
                a = (np.frombuffer(raw, dtype=np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32)
            else:
                continue                                   # integer buffers (position_ids) are not parameters
            out[name] = a.reshape(info["shape"]).copy()
    return out


def from_hf_bert(state: Dict[str, np.ndarray], cfg: EncoderConfig) -> Dict[str, np.ndarray]:
    """HuggingFace BertModel parameter names (with or without a ``bert.`` prefix) -> the names
    ``aur_encoder_load`` expects; query / key / value matrices are stacked into ``wqkv``."""
    def g(name: str) -> np.ndarray:
        for prefix in ("", "bert."):
            if prefix + name in state:
                return np.asarray(state[prefix + name], dtype=np.float32)
        raise KeyError(name)

    w = {"word_emb": g("embeddings.word_embeddings.weight"), "pos_emb": g("embeddings.position_embeddings.weight"),
         "type_emb": g("embeddings.token_type_embeddings.weight"), "emb_ln_g": g("embeddings.LayerNorm.weight"),
         "emb_ln_b": g("embeddings.LayerNorm.bias")}
    for l in range(cfg.layers):
        p, q = f"l{l}.", f"encoder.layer.{l}."
        w[p + "wqkv"] = np.concatenate([g(q + f"attention.self.{n}.weight") for n in ("query", "key", "value")], axis=0)
        w[p + "bqkv"] = np.concatenate([g(q + f"attention.self.{n}.bias") for n in ("query", "key", "value")], axis=0)
        w[p + "wo"], w[p + "bo"] = g(q + "attention.output.dense.weight"), g(q + "attention.output.dense.bias")
        w[p + "ln1_g"], w[p + "ln1_b"] = g(q + "attention.output.LayerNorm.weight"), g(q + "attention.output.LayerNorm.bias")
        w[p + "wi"], w[p + "bi"] = g(q + "intermediate.dense.weight"), g(q + "intermediate.dense.bias")
        w[p + "wo2"], w[p + "bo2"] = g(q + "output.dense.weight"), g(q + "output.dense.bias")
        w[p + "ln2_g"], w[p + "ln2_b"] = g(q + "output.LayerNorm.weight"), g(q + "output.LayerNorm.bias")
    return w

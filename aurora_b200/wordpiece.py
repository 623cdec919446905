"""WordPiece tokenisation for the uncased BERT vocabularies the reference's encoders use
(all-MiniLM-L6-v2, bge-base-en): text -> token ids for ``aurora_b200.encoder``.

In the reference this happens inside the t2v-transformers sidecar (embedding_client.py:52-59 posts
raw text to it); the algorithm is the published BERT one: basic tokenisation (clean, lower-case,
strip accents, split on whitespace and punctuation, isolate CJK characters) followed by greedy
longest-match-first WordPiece with ``##`` continuation pieces.  tests/test_wordpiece.py holds it to
``transformers.BertTokenizer`` on the same vocabulary.  The vocabulary file itself is deployment
data (SURVEY.md section 8(f) item 2).
"""

from __future__ import annotations

import unicodedata
from typing import Dict, Iterable, List


def load_vocab(path: str) -> Dict[str, int]:
    vocab: Dict[str, int] = {}
    with open(path, encoding="utf-8") as f:
        for i, line in enumerate(f):
            vocab[line.rstrip("\n")] = i
    return vocab


def _is_whitespace(ch: str) -> bool:
    return ch in " \t\n\r" or unicodedata.category(ch) == "Zs"


def _is_control(ch: str) -> bool:
    if ch in "\t\n\r":
        return False
    return unicodedata.category(ch).startswith("C")


def _is_punctuation(ch: str) -> bool:
    cp = ord(ch)
    if 33 <= cp <= 47 or 58 <= cp <= 64 or 91 <= cp <= 96 or 123 <= cp <= 126:
        return True
    return unicodedata.category(ch).startswith("P")


def _is_cjk(cp: int) -> bool:
    return (0x4E00 <= cp <= 0x9FFF or 0x3400 <= cp <= 0x4DBF or 0x20000 <= cp <= 0x2A6DF or 0x2A700 <= cp <= 0x2B73F or
            0x2B740 <= cp <= 0x2B81F or 0x2B820 <= cp <= 0x2CEAF or 0xF900 <= cp <= 0xFAFF or 0x2F800 <= cp <= 0x2FA1F)


def basic_tokenize(text: str, lower: bool = True) -> List[str]:
    out = []
    for ch in text:                                   # clean + put spaces around CJK characters
        cp = ord(ch)
        if cp == 0 or cp == 0xFFFD or _is_control(ch):
            continue
        if _is_cjk(cp):
            out.append(f" {ch} ")
        else:
            out.append(" " if _is_whitespace(ch) else ch)
    words = []
    for tok in "".join(out).split():
        if lower:
            tok = tok.lower()
            tok = "".join(c for c in unicodedata.normalize("NFD", tok) if unicodedata.category(c) != "Mn")
        cur = []
        for ch in tok:                                # split on punctuation, each mark its own token
            if _is_punctuation(ch):
                if cur:
                    words.append("".join(cur)); cur = []
                words.append(ch)
            else:
                cur.append(ch)
        if cur:
            words.append("".join(cur))
    return words


class WordPieceTokenizer:
    def __init__(self, vocab: Dict[str, int], lower: bool = True, unk: str = "[UNK]", cls: str = "[CLS]",
                 sep: str = "[SEP]", max_chars_per_word: int = 100):
        self.vocab, self.lower, self.max_chars = vocab, lower, max_chars_per_word
        self.unk_id, self.cls_id, self.sep_id = vocab[unk], vocab[cls], vocab[sep]

    def wordpiece(self, word: str) -> List[int]:
        if len(word) > self.max_chars:
            return [self.unk_id]
        ids, start = [], 0
        while start < len(word):
            end, cur = len(word), None
            while start < end:
                piece = word[start:end] if start == 0 else "##" + word[start:end]
                if piece in self.vocab:
                    cur = self.vocab[piece]
                    break
                end -= 1
            if cur is None:
                return [self.unk_id]                 # one unknown piece makes the whole word [UNK]
            ids.append(cur)
            start = end
        return ids

    def tokenize_ids(self, text: str) -> List[int]:
        ids: List[int] = []
        for w in basic_tokenize(text, self.lower):
            ids.extend(self.wordpiece(w))
        return ids

    def encode(self, text: str, max_len: int = 512) -> List[int]:
        """[CLS] pieces [SEP], truncated to ``max_len`` ids (the sidecar's truncation=True)."""
        body = self.tokenize_ids(text)[: max(0, max_len - 2)]
        return [self.cls_id] + body + [self.sep_id]

    __call__ = encode

    def encode_batch(self, texts: Iterable[str], max_len: int = 512) -> List[List[int]]:
        return [self.encode(t, max_len) for t in texts]


class NativeTokenizer:
    """The same tokenisation in C++ behind the C ABI (csrc/tokenizer.cpp, ``aur_tokenize``): multi-threaded, GIL-free,
    ids identical to ``transformers.BertTokenizer``.  This is what the ingest path uses; the pure-Python class above
    stays as the readable restatement the tests cross-check it with.

    ``vocab``: path of a vocab.txt, or a ``{piece: id}`` dict / list of pieces (ids must be 0..n-1)."""

    def __init__(self, vocab, lower: bool = True):
        import ctypes as C

        from . import _native as N

        self._N, self._lib, self._h = N, N.load(), C.c_void_p()
        if isinstance(vocab, (str, bytes)):
            path = vocab if isinstance(vocab, bytes) else vocab.encode()
            N.check(self._lib.aur_tokenizer_open(path, int(lower), C.byref(self._h)))
        else:
            pieces = list(vocab) if not isinstance(vocab, dict) else [p for p, _ in sorted(vocab.items(), key=lambda kv: kv[1])]
            if isinstance(vocab, dict) and sorted(vocab.values()) != list(range(len(vocab))):
                raise ValueError("vocabulary ids must be 0 .. n-1")
            blob = "\n".join(pieces).encode("utf-8")
            N.check(self._lib.aur_tokenizer_open_mem(blob, len(blob), int(lower), C.byref(self._h)))
        vs, unk, cls, sep = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        N.check(self._lib.aur_tokenizer_info(self._h, C.byref(vs), C.byref(unk), C.byref(cls), C.byref(sep)))
        self.vocab_size, self.unk_id, self.cls_id, self.sep_id = vs.value, unk.value, cls.value, sep.value

    @staticmethod
    def _pack(texts):
        import numpy as np

        enc = [t.encode("utf-8", "replace") for t in texts]
        offs = np.zeros(len(enc) + 1, dtype=np.int64)
        if enc:
            offs[1:] = np.cumsum([len(b) for b in enc])
        return b"".join(enc), offs

    def encode_packed(self, texts, max_len: int = 512, threads: int = 0):
        """(tokens int32 [total], cu_seqlens int32 [n + 1]) -- the layout ``Encoder.encode_packed`` takes."""
        import ctypes as C

        import numpy as np

        blob, offs = self._pack(texts)
        n = len(offs) - 1
        tokens = np.empty(max(1, n * max_len), dtype=np.int32)
        cu = np.zeros(n + 1, dtype=np.int32)
        self._N.check(self._lib.aur_tokenize(self._h, blob, offs.ctypes.data_as(C.c_void_p), n, int(max_len),
                                             tokens.ctypes.data_as(C.c_void_p), tokens.size, cu.ctypes.data_as(C.c_void_p), int(threads)))
        return tokens[: int(cu[-1])], cu

    def lengths(self, texts, max_len: int = 1 << 20, threads: int = 0):
        """Token counts ([CLS] / [SEP] included, capped at ``max_len``) of every text, one C call, no ids returned."""
        import ctypes as C

        import numpy as np

        blob, offs = self._pack(texts)
        n = len(offs) - 1
        cu = np.zeros(n + 1, dtype=np.int32)
        self._N.check(self._lib.aur_tokenize(self._h, blob, offs.ctypes.data_as(C.c_void_p), n, int(max_len), None, 0,
                                             cu.ctypes.data_as(C.c_void_p), int(threads)))
        return np.diff(cu)

    def encode_windows(self, texts, max_len: int = 512, threads: int = 0):
        """(tokens int32 [total], cu_seqlens int32 [windows + 1], cu_texts int32 [n + 1]): every text's whole
        tokenisation [CLS] b [SEP] as windows for a position table of ``max_len`` (``aur_tokenize_windows``): one window,
        ``encode_packed``'s, when it fits; otherwise [CLS] b[i : i + max_len - 2] [SEP] for i = 0, max_len - 2, ...
        Text j is windows cu_texts[j] .. cu_texts[j + 1] - 1.  One C call (two if a text tokenises to more ids than it
        has bytes, which the first call's buffers assume it does not)."""
        import ctypes as C

        import numpy as np

        blob, offs = self._pack(texts)
        n = len(offs) - 1
        seqs = 2 * n + len(blob) // max(1, int(max_len) - 2)
        toks = len(blob) + 2 * seqs
        cu_texts = np.zeros(n + 1, dtype=np.int32)
        totals = np.zeros(2, dtype=np.int64)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)      # noqa: E731
        for _ in range(2):
            tokens, cu = np.empty(max(1, toks), dtype=np.int32), np.zeros(seqs + 1, dtype=np.int32)
            rc = self._lib.aur_tokenize_windows(self._h, blob, vp(offs), n, int(max_len), vp(tokens), tokens.size, vp(cu), seqs,
                                                vp(cu_texts), vp(totals), int(threads))
            if rc != self._N.AUR_ERR_NOMEM:
                break
            seqs, toks = int(totals[0]), int(totals[1])
        self._N.check(rc)
        return tokens[: int(totals[1])], cu[: int(totals[0]) + 1], cu_texts

    def encode_batch(self, texts, max_len: int = 512) -> List[List[int]]:
        tok, cu = self.encode_packed(texts, max_len)
        return [tok[cu[i]:cu[i + 1]].tolist() for i in range(len(cu) - 1)]

    def encode(self, text: str, max_len: int = 512) -> List[int]:
        return self.encode_batch([text], max_len)[0]

    __call__ = encode

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.aur_tokenizer_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

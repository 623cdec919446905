"""The byte rule the device analyzer implements (csrc/kw_text.cu), derived from Python's str.lower at run time, and the
argument checks of aur_kw_vocab_* / aur_kw_add_text / aur_kw_read_rows that need no device."""

import ctypes as C
import re
import sys

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200 import bm25


def _byte_words(data: bytes):
    """The analyzer's rule on UTF-8 bytes (include/aurora_b200.h, aur_kw_vocab): ASCII letters (lowered) and digits are
    word characters, E2 84 AA is "k" inside a word, C4 B0 is "i" and then a break, every other byte breaks."""
    out, cur, i = [], [], 0
    while i < len(data):
        c = data[i]
        if 48 <= c <= 57 or 97 <= c <= 122 or 65 <= c <= 90:
            cur.append(chr(c).lower()); i += 1; continue
        if data[i:i + 3] == b"\xe2\x84\xaa":
            cur.append("k"); i += 3; continue
        if data[i:i + 2] == b"\xc4\xb0":
            cur.append("i")
        if cur:
            out.append("".join(cur)); cur = []
        i += 1
    if cur:
        out.append("".join(cur))
    return out


def test_only_two_non_ascii_characters_lower_to_word_characters():
    found = [c for c in range(128, sys.maxunicode + 1)
             if not (0xD800 <= c <= 0xDFFF) and re.search(r"[0-9a-z]", chr(c).lower())]
    assert found == [0x130, 0x212A]


def test_the_byte_rule_is_tokenize():
    rng = np.random.default_rng(2)
    alphabet = [chr(c) for c in range(32, 127)] + ["İ", "K", "\x00", "é", "ß", "̇", "日", "\U0001f600"]
    texts = ["".join(rng.choice(alphabet, size=int(rng.integers(0, 80)))) for _ in range(3000)]
    texts += ["İ", "K", "abİcd", "aKb", "İKİ", "xİİy", "lone\ud83dsurrogate", "\udc00x\ud800"]
    for t in texts:   # engine._add_text encodes with surrogatepass: a lone surrogate reaches the device as ED xx xx
        assert _byte_words(t.encode("utf-8", "surrogatepass")) == bm25.tokenize(t), t


def test_text_calls_reject_bad_arguments_without_a_device():
    lib = N.load()
    h = C.c_void_p()
    assert lib.aur_kw_vocab_open(0, None) == N.AUR_ERR_INVALID
    assert lib.aur_kw_vocab_close(None) == N.AUR_OK
    assert lib.aur_kw_vocab_size(None, None, None) == N.AUR_ERR_INVALID
    off = np.zeros(2, np.int64)
    assert lib.aur_kw_vocab_read(None, 0, 1, None, 0, off.ctypes.data_as(C.c_void_p)) == N.AUR_ERR_INVALID
    assert lib.aur_kw_vocab_set_option(None, b"hash_bits", 4) == N.AUR_ERR_INVALID
    assert lib.aur_kw_add_text(None, 1, None, None, None, None, None, None, 1) == N.AUR_ERR_INVALID
    total = C.c_int64(0)
    assert lib.aur_kw_read_rows(None, 0, 1, None, off.ctypes.data_as(C.c_void_p), None, None, 0, C.byref(total)) == N.AUR_ERR_INVALID
    if lib.aur_device_count() == 0:
        assert lib.aur_kw_vocab_open(0, C.byref(h)) == N.AUR_ERR_NO_DEVICE


def test_vocabulary_needs_a_device():
    lib = N.load()
    if lib.aur_device_count() > 0:
        pytest.skip("a GPU is present; the no-device behaviour is exercised on the CPU box")
    from aurora_b200.engine import KeywordVocab

    with pytest.raises(N.AuroraError) as e:
        KeywordVocab(0)
    assert e.value.code == N.AUR_ERR_NO_DEVICE
    with pytest.raises(N.AuroraError) as e:
        bm25.DeviceBM25(128)
    assert e.value.code == N.AUR_ERR_NO_DEVICE


def test_a_store_without_add_text_is_fed_build_csr():
    calls = []

    class Store:    # a recording double of engine.KeywordIndex without the device analyzer
        def add(self, ids, terms, tfs, offsets, user_codes=None, org_codes=None):
            calls.append((ids.tolist(), terms.tolist(), tfs.tolist(), offsets.tolist()))

    sp = bm25.DeviceBM25(store=Store())
    sp.add_many([4, 9], ["Disk disk full", "node İ"])
    want = {}
    t, f, o = bm25.build_csr(want, ["Disk disk full", "node İ"])
    assert calls == [([4, 9], t.tolist(), f.tolist(), o.tolist())]
    assert sp.vocab == want and len(sp) == 2


def test_a_failed_text_add_reports_its_own_error_and_syncs_the_mirror():
    import threading

    class Vocab:    # the surface of engine.KeywordVocab that DeviceBM25 reads
        def __init__(self, fail):
            self.words, self.fail = [], fail

        def read(self, id0=0, n=None):
            if self.fail:
                raise RuntimeError("mirror read failed")
            return self.words[id0:]

    class Store:
        def add_text(self, vocab, ids, texts, user_codes=None, org_codes=None):
            vocab.words.extend(["alpha", "beta"])        # words added before the failure, as the device may
            raise MemoryError("posting growth failed")

    sp = bm25.DeviceBM25.__new__(bm25.DeviceBM25)        # without a device: the doubles stand in for it
    sp.store, sp.vocab, sp._docs, sp._lock = Store(), {}, set(), threading.RLock()
    sp._dvocab = Vocab(fail=False)
    with pytest.raises(MemoryError):
        sp.add_many([1], ["alpha beta"])
    assert sp.vocab == {"alpha": 0, "beta": 1}           # the mirror holds what the vocabulary holds
    sp._dvocab = Vocab(fail=True)
    with pytest.raises(MemoryError):                     # the add's error, not the mirror's
        sp.add_many([2], ["gamma"])
    assert not sp._docs

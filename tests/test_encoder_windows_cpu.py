"""Texts longer than the position table, without a GPU: the window rule of aur_tokenize_windows (C++) against
TextEncoder._windows and the pure-Python WordPieceTokenizer, and oracle/window_mean.py (the arithmetic that folds a
text's window vectors into one vector on the device) against fp64 and hand-worked cases."""

import ctypes as C
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.encoder import TextEncoder
from aurora_b200.wordpiece import NativeTokenizer, WordPieceTokenizer, basic_tokenize
from oracle.window_mean import fold_texts, fold_windows

U = lambda *cps: "".join(chr(c) for c in cps)      # noqa: E731
HERE = os.path.dirname(os.path.abspath(__file__))

# the Unicode edge cases of test_tokenizer_native.py
EDGE = [U(0x39f, 0x394, 0x3a5, 0x3a3, 0x3a3, 0x395, 0x3a5, 0x3a3), U(0x130), U(0x1e9e), U(0x1c5), U(0xc5), U(0x61, 0xad, 0x62), U(0x78, 0x200b, 0x79),
        U(0xfeff, 0x62), U(0x61, 0x20, 0x62, 0xfffd, 0x63), U(0xff46, 0xff55), U(0x2460), U(0xd55c, 0xae00), U(0x61, 0xa0, 0x62),
        U(0x61, 0x2028, 0x62), U(0xac00), U(0x61, 0x7f, 0x62), U(0x61, 0x85, 0x62), U(0x61, 0x378, 0x62), U(0x65, 0x301), U(0x1e69),
        U(0x61, 0x20dd, 0x62), U(0x61, 0x903, 0x62), U(0x61, 0x0, 0x62), U(0x61, 0xe000, 0x62), U(0x61, 0x1f600, 0x62), U(0x61, 0xb7, 0x62),
        U(0x61, 0x2d, 0x62), U(0x61, 0x60, 0x62), U(0x61, 0x5e, 0x62), U(0x61, 0x24, 0x62), U(0x61, 0xa2, 0x62), U(0x61, 0x3001, 0x62),
        U(0x4e2d, 0x6587), U(0x1e9b, 0x323), U(0xf900, 0x61), U(0x2f800), U(0x301, 0x61), U(0x1100, 0x1161), U(0x3b1, 0x345, 0x301)]
WORDS = ["restart", "the", "payment", "service", "node", "disk", "pressure", "kafka", "lag", "10", ".", "0", "/", ":"]


def _golden_chunks():
    gold = json.load(open(os.path.join(HERE, "golden", "chunker_ref.json"), encoding="utf-8"))
    return [(c["heading_context"] + "\n" if c["heading_context"] else "") + c["content"]
            for d in gold["documents"] for c in d["chunks"]]


def _vocab(texts):
    """[specials] + every word of the texts (up to 100 characters) + every character as a word-initial and a ## piece."""
    pieces = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    words = set()
    for t in texts:
        words.update(basic_tokenize(t))
    chars = sorted({c for w in words for c in w})
    pieces += sorted(w for w in words if len(w) <= 100 and len(w) > 1) + chars + ["##" + c for c in chars]
    seen, uniq = set(), []
    for p in pieces:
        if p not in seen:
            seen.add(p); uniq.append(p)
    return {p: i for i, p in enumerate(uniq)}


def _body(n, seed=0):
    """A text of exactly n word pieces under _vocab (every WORDS entry is one piece)."""
    rng = np.random.default_rng(seed)
    return " ".join(rng.choice(WORDS, size=n))


def _texts(step):
    return ["", "kafka", _body(step), _body(step + 1, 1), _body(3 * step, 2), _body(7 * step + 5, 3)] + EDGE + _golden_chunks()


@pytest.fixture(scope="module")
def toks():
    big = _body(220_000, 9)                                        # about 1 MB of text
    assert len(big.encode()) > 1_000_000
    vocab = _vocab(_texts(10) + [big])
    return NativeTokenizer(vocab), WordPieceTokenizer(vocab), big


def _text_encoder(tok, max_len):
    stub = SimpleNamespace(cfg=SimpleNamespace(hidden=32, max_pos=512), device=0)   # _windows needs no encoder
    return TextEncoder(stub, tok, max_len=max_len)


def _split(tok, cu, cu_texts):
    return [[tok[cu[w]:cu[w + 1]].tolist() for w in range(cu_texts[j], cu_texts[j + 1])] for j in range(len(cu_texts) - 1)]


@pytest.mark.parametrize("max_len", [64, 512])
def test_native_windows_follow_the_python_rule(toks, max_len):
    nat, py, big = toks
    step = max_len - 2
    texts = _texts(step) + [big]
    tok, cu, cu_texts = nat.encode_windows(texts, max_len)
    got = _split(tok, cu, cu_texts)
    te_nat = _text_encoder(nat, max_len)
    te_py = _text_encoder(lambda t: py.encode(t, max_len=1 << 40), max_len)
    for t, g in zip(texts, got):
        assert g == [w.tolist() for w in te_nat._windows(t)]
        full = py.encode(t, max_len=1 << 40)                       # [CLS] b [SEP], whole
        body = full[1:-1]
        want = [[full[0]] + body[i:i + step] + [full[-1]] for i in range(0, max(len(body), 1), step)]
        if full == nat.encode(t, max_len=1 << 30):                 # (where the Python restatement tokenises as the C++ one)
            assert g == want == [w.tolist() for w in te_py._windows(t)]
        assert all(2 <= len(w) <= max_len for w in g)
        if 2 + len(body) <= max_len:                               # a text that fits is aur_tokenize's one window
            assert g == [nat.encode(t, max_len)]
    lens = [len(g) for g in got]
    assert lens[:6] == [1, 1, 1, 2, 3, 8]                          # empty, one piece, exactly max_len, max_len + 1, 3 steps, 7 steps + 5
    assert [len(w) for w in got[2]] == [max_len] and [len(w) for w in got[3]] == [max_len, 3]
    assert [len(w) for w in got[4]] == [max_len] * 3
    assert lens[-1] == -(-220_000 // step)
    # the Python callable route packs the same windows
    ptok, pcu, pct = te_py._tokenize_windows(texts[:6] + _golden_chunks())
    ntok, ncu, nct = nat.encode_windows(texts[:6] + _golden_chunks(), max_len)
    assert np.array_equal(ptok, ntok) and np.array_equal(pcu, ncu) and np.array_equal(pct, nct)


def test_golden_chunks_really_span_windows(toks):
    nat, _, _ = toks
    _, _, cu_texts = nat.encode_windows(_golden_chunks(), 512)
    assert np.diff(cu_texts).max() >= 2                           # the 4 196-character chunk


def _raw(nat, texts, max_len, tokens_cap, seqs_cap, threads=0, null=False):
    blob, offs = nat._pack(texts)
    n = len(texts)
    tok = np.zeros(max(1, tokens_cap), np.int32)
    cu = np.zeros(seqs_cap + 1, np.int32)
    ct = np.full(n + 1, -7, np.int32)
    tot = np.zeros(2, np.int64)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)      # noqa: E731
    rc = nat._lib.aur_tokenize_windows(nat._h, blob, vp(offs), n, max_len, None if null else vp(tok), tokens_cap,
                                       None if null else vp(cu), seqs_cap, vp(ct), vp(tot), threads)
    return rc, tok, cu, ct, tot


def test_threads_count_mode_and_capacity_errors(toks):
    nat, _, _ = toks
    texts = _texts(62) * 6
    t1 = nat.encode_windows(texts, 64, threads=1)
    ta = nat.encode_windows(texts, 64, threads=0)
    assert all(np.array_equal(a, b) for a, b in zip(t1, ta))
    tok, cu, cu_texts = t1
    need_w, need_t = int(cu_texts[-1]), int(cu[-1])
    rc, _, _, ct, tot = _raw(nat, texts, 64, 0, 0, null=True)     # count mode
    assert rc == N.AUR_OK and np.array_equal(ct, cu_texts) and tot.tolist() == [need_w, need_t]
    for tcap, scap in ((need_t - 1, need_w), (need_t, need_w - 1)):
        rc, _, _, ct, tot = _raw(nat, texts, 64, tcap, scap)
        assert rc == N.AUR_ERR_NOMEM and np.array_equal(ct, cu_texts) and tot.tolist() == [need_w, need_t]
    rc, t2, c2, ct, _ = _raw(nat, texts, 64, need_t, need_w)       # exactly enough
    assert rc == N.AUR_OK and np.array_equal(t2, tok) and np.array_equal(c2, cu) and np.array_equal(ct, cu_texts)
    assert _raw(nat, texts, 2, need_t, need_w)[0] == N.AUR_ERR_INVALID   # no room for a piece between [CLS] and [SEP]
    assert _raw(nat, texts, 64, -1, need_w)[0] == N.AUR_ERR_INVALID


# ---------------------------------------------------------------------- the fold arithmetic
def _unit_rows(rng, w, h):
    v = rng.standard_normal((w, h)).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("w", [2, 3, 5, 8, 17])
@pytest.mark.parametrize("h", [128, 768])
def test_fold_is_the_fp64_mean_and_norm_within_fp32_rounding(w, h):
    rng = np.random.default_rng(w * 1000 + h)
    u = 2.0 ** -24
    for _ in range(4):
        v = _unit_rows(rng, w, h)
        got = fold_windows(v, True).astype(np.float64)
        m64 = v.astype(np.float64).mean(axis=0)
        want = m64 / np.linalg.norm(m64)
        # the fp32 sum rounds w - 1 times, the division once: |m - m64| <= e elementwise, then normalised
        e = (w - 1) * u * np.abs(v).astype(np.float64).sum(axis=0) / w + u * np.abs(m64)
        tol = 2.0 * np.linalg.norm(e) / np.linalg.norm(m64) + 2.0 * u
        assert np.max(np.abs(got - want)) <= tol
        raw = fold_windows(v, False).astype(np.float64)
        assert np.max(np.abs(raw - m64)) <= np.max(e) * 2
    one = _unit_rows(rng, 1, h)
    assert fold_windows(one, True).tobytes() == one[0].tobytes()   # one window: the window's vector, bit for bit


def test_fold_hand_cases():
    h = 32
    e = np.zeros((2, h), np.float32)
    e[0, 0], e[1, 1] = 1.0, 1.0                                    # w = 2: (e0 + e1) / 2, normalised
    got = fold_windows(e, True)
    assert got[0] == got[1] == np.float32(0.5 / np.sqrt(0.5)) and not got[2:].any()
    assert fold_windows(e, False)[:2].tolist() == [0.5, 0.5]
    # w = 3: the sum runs in window order in fp32, 1 + 2^-24 rounds back to 1 twice (the exact sum is 1 + 2^-23)
    v = np.zeros((3, h), np.float32)
    v[:, 0] = [1.0, 2.0 ** -24, 2.0 ** -24]
    v[:, 5] = [0.1, 0.2, 0.4]
    raw = fold_windows(v, False)
    assert raw[0] == np.float32(1.0) / np.float32(3.0)
    assert raw[5] == ((np.float32(0.1) + np.float32(0.2)) + np.float32(0.4)) / np.float32(3.0)
    q = float(np.float64(raw[0]) ** 2 + np.float64(raw[5]) ** 2)    # lanes 0 and 5; every other lane sum is 0
    norm = fold_windows(v, True)
    assert norm[0] == np.float32(np.float64(raw[0]) / np.sqrt(q)) and norm[5] == np.float32(np.float64(raw[5]) / np.sqrt(q))
    # zero vectors: q = 0 leaves the mean (zeros), never NaN
    z = np.zeros((4, h), np.float32)
    assert fold_windows(z, True).tobytes() == np.zeros(h, np.float32).tobytes()
    # opposite windows cancel exactly: the mean is zero, so is the text's vector
    o = np.stack([e[0], -e[0]])
    assert not fold_windows(o, True).any()


def test_fold_texts_splits_by_cu_texts():
    rng = np.random.default_rng(3)
    v = _unit_rows(rng, 7, 64)
    ct = np.array([0, 1, 4, 5, 7])
    out = fold_texts(v, ct, True)
    for j in range(4):
        assert out[j].tobytes() == fold_windows(v[ct[j]:ct[j + 1]], True).tobytes()

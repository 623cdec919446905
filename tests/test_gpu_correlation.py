"""aur_encode_pair_cosines (Encoder.pair_cosines) and EmbeddingClient.similarities on the GPU: the text vectors are
aur_encode_texts' bit for bit and the cosines aur_cosine_pairs' over them bit for bit, across workspace batches and
windows left open between them; malformed calls are rejected before any device work; the client's pairs agree with the
serial embed + Python cosine of the reference's path."""

import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from aurora_b200 import _native as N
from aurora_b200.correlation import SimilarityStrategy
from aurora_b200.encoder import EmbeddingClient, Encoder, EncoderConfig, pack_sequences
from aurora_b200.engine import cosine_pairs
from oracle import bert_encoder as B
from oracle import ref_cosine

# bge-base and MiniLM widths (head dim 64 with CLS pooling; head dim 32 with mean pooling), two layers to keep it short
CFGS = {
    "bge-base": B.BertConfig(hidden=768, layers=2, heads=12, inter=3072, vocab=1000, max_pos=512, pool="cls"),
    "minilm": B.BertConfig(hidden=384, layers=2, heads=12, inter=1536, vocab=1000, max_pos=512, pool="mean"),
}
_WEIGHTS = {}


def _encoder(name, max_tokens=32768, max_seqs=2048) -> Encoder:
    c = CFGS[name]
    if name not in _WEIGHTS:
        _WEIGHTS[name] = B.init_weights(c, seed=7, bf16=True)
    enc = Encoder(EncoderConfig(hidden=c.hidden, layers=c.layers, heads=c.heads, inter=c.inter, vocab=c.vocab,
                                max_pos=c.max_pos, type_vocab=c.type_vocab, ln_eps=c.ln_eps, pool=c.pool,
                                normalize=c.normalize), max_tokens=max_tokens, max_seqs=max_seqs)
    enc.load_weights(_WEIGHTS[name])
    return enc


def _texts(rng, window_counts, vocab, max_len=200):
    """Packed windows: text j has window_counts[j] windows of 1 .. max_len tokens."""
    wins = [rng.integers(0, vocab, int(rng.integers(1, max_len + 1))).astype(np.int32) for w in window_counts for _ in range(w)]
    tok, cu = pack_sequences(wins)
    ct = np.zeros(len(window_counts) + 1, np.int32)
    ct[1:] = np.cumsum(window_counts)
    return tok, cu, ct


def _pairs(rng, n_texts, n):
    pa = rng.integers(0, n_texts, n).astype(np.int32)
    pb = rng.integers(0, n_texts, n).astype(np.int32)
    pa[:3], pb[:3] = 0, 0                 # a self-pair ...
    pa[3:5], pb[3:5] = 1, n_texts - 1     # ... and a repeated pair
    return pa, pb


@pytest.mark.parametrize("name", sorted(CFGS))
@pytest.mark.parametrize("clamp", [0, 1])
def test_vectors_and_cosines_are_bit_identical_across_batches(name, clamp):
    rng = np.random.default_rng(11 + clamp)
    # a workspace of 384 tokens / 3 sequences: the 40 texts take many batches, and the 4-window texts of up to 200 tokens
    # a window are left open across batch boundaries
    enc = _encoder(name, max_tokens=384, max_seqs=3)
    counts = [1] * 40
    counts[5], counts[17], counts[30] = 4, 2, 3
    tok, cu, ct = _texts(rng, counts, CFGS[name].vocab)
    assert int(cu[-1]) >= 3 * 384 and len(cu) - 1 >= 9
    pa, pb = _pairs(rng, len(counts), 500)
    cos, vec = enc.pair_cosines(tok, cu, ct, pa, pb, clamp=bool(clamp), vectors=True)
    want_vec = enc.encode_texts(tok, cu, ct)
    assert np.array_equal(vec.view(np.uint32), want_vec.view(np.uint32))
    want = cosine_pairs(want_vec[pa], want_vec[pb], clamp=bool(clamp))
    assert np.array_equal(cos.view(np.uint64), want.view(np.uint64))
    ref = np.array([ref_cosine.cosine_similarity(want_vec[a].tolist(), want_vec[b].tolist(), clamp=bool(clamp)) for a, b in zip(pa, pb)])
    assert np.max(np.abs(cos - ref)) <= 1e-12
    assert np.array_equal(enc.pair_cosines(tok, cu, ct, pa, pb, clamp=bool(clamp)).view(np.uint64), cos.view(np.uint64))
    enc.close()


def test_single_text_no_pairs_and_ten_thousand_pairs():
    rng = np.random.default_rng(3)
    enc = _encoder("minilm")
    tok, cu, ct = _texts(rng, [1], 1000)
    cos, vec = enc.pair_cosines(tok, cu, ct, [0], [0], vectors=True)
    assert cos.tolist() == [1.0] or abs(cos[0] - 1.0) <= 1e-15
    assert np.array_equal(vec, enc.encode_texts(tok, cu, ct))
    cos0, vec0 = enc.pair_cosines(tok, cu, ct, [], [], vectors=True)
    assert cos0.shape == (0,) and np.array_equal(vec0, vec)
    assert enc.pair_cosines(tok, cu, ct, [], []).shape == (0,)
    tok, cu, ct = _texts(rng, [1] * 300, 1000, max_len=40)
    pa, pb = _pairs(rng, 300, 10000)
    cos, vec = enc.pair_cosines(tok, cu, ct, pa, pb, vectors=True)
    assert np.array_equal(cos.view(np.uint64), cosine_pairs(vec[pa], vec[pb], clamp=True).view(np.uint64))
    enc.close()


def test_rejections_leave_outputs_and_stats_untouched():
    rng = np.random.default_rng(5)
    enc = _encoder("minilm", max_tokens=4096, max_seqs=64)
    tok, cu, ct = _texts(rng, [1, 2, 1], 1000, max_len=60)
    pa, pb = np.array([0, 1, 2], np.int32), np.array([2, 1, 0], np.int32)
    enc.pair_cosines(tok, cu, ct, pa, pb)
    before = enc.stats()
    lib = N.load()
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def call(pa_, pb_, n_pairs, clamp=1, ct_=ct, cos=True, vec=True):
        out = np.full(max(n_pairs, 1), 7.0)
        v = np.full((len(ct_) - 1, CFGS["minilm"].hidden), 7.0, np.float32)
        rc = lib.aur_encode_pair_cosines(enc._h, p(tok), p(cu), len(cu) - 1, p(ct_), len(ct_) - 1, p(pa_), p(pb_), n_pairs,
                                         clamp, p(out) if cos else None, p(v) if vec else None)
        return rc, bool(np.all(out == 7.0) and np.all(v == 7.0))

    bad_ct = np.array([0, 2, 2, 4], np.int32)                           # text 1 has no window
    for args in [(np.array([0, 3, 1], np.int32), pb, 3), (np.array([0, -1, 1], np.int32), pb, 3), (pa, np.array([0, 1, 9], np.int32), 3),
                 (None, pb, 3), (pa, None, 3), (pa, pb, -1)]:
        rc, untouched = call(*args)
        assert rc == N.AUR_ERR_INVALID and untouched, (args, lib.aur_last_error())
    for kw in [dict(clamp=2), dict(clamp=-1), dict(ct_=bad_ct), dict(cos=False)]:
        rc, untouched = call(pa, pb, 3, **kw)
        assert rc == N.AUR_ERR_INVALID and untouched, (kw, lib.aur_last_error())
    assert enc.stats() == before
    enc.close()


def _tokenizer(vocab):
    """[CLS] word ids [SEP]; "oov<n>" maps to id n (outside the vocabulary when n >= vocab)."""
    def tok(text):
        ids = [int(w[3:]) if w.startswith("oov") else 5 + (sum(map(ord, w)) % (vocab - 5)) for w in text.split()]
        return [2] + ids + [3]
    return tok


def test_similarities_match_the_serial_path_and_none_only_where_embed_fails():
    enc = _encoder("bge-base")
    client = EmbeddingClient(enc, _tokenizer(CFGS["bge-base"].vocab))
    long_text = " ".join(["word"] * 600)                                 # 602 tokens > max_pos
    titles = ["High CPU usage on api-server", "API server CPU is high", "Disk pressure on node-3", "kafka consumer lag",
              "payment 5xx errors", "Café latency über p99", "", "   ", long_text, "cpu oov1000 high"]
    bad = {"", "   ", long_text, "cpu oov1000 high"}
    pairs = [(a, b) for a in titles for b in titles] + [(titles[0], titles[1])] * 3
    got = client.similarities(pairs)
    s = SimilarityStrategy()
    for (a, b), g in zip(pairs, got):
        va, vb = client.embed(a), client.embed(b)
        if a in bad or b in bad:
            assert g is None and (va is None or vb is None), (a, b)
        else:
            assert g is not None and abs(g - s._cosine_similarity(va, vb)) <= 1e-12, (a, b)
    assert client.similarities([]) == [] and client.similarities([("", "x")]) == [None]
    enc.close()


def test_pair_cosines_and_encode_on_two_threads():
    rng = np.random.default_rng(9)
    enc = _encoder("minilm", max_tokens=512, max_seqs=8)
    tok, cu, ct = _texts(rng, [1, 3, 1, 1, 2, 1] * 4, 1000, max_len=150)
    pa, pb = _pairs(rng, len(ct) - 1, 200)
    want_cos = enc.pair_cosines(tok, cu, ct, pa, pb)
    seqs = [rng.integers(0, 1000, int(rng.integers(1, 200))).astype(np.int32) for _ in range(20)]
    want_enc = enc.encode(seqs)
    errs = []

    def run(fn, want):
        try:
            for _ in range(10):
                got = fn()
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
        except Exception as e:      # pragma: no cover
            errs.append(e)

    ts = [threading.Thread(target=run, args=(lambda: enc.pair_cosines(tok, cu, ct, pa, pb), want_cos)),
          threading.Thread(target=run, args=(lambda: enc.encode(seqs), want_enc))]
    [t.start() for t in ts]; [t.join() for t in ts]
    assert not errs, errs[0]
    enc.close()

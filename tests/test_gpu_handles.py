"""Handles whose open fails part-way (csrc owners: DevBuf, Stream, Event) give back what they had taken: the open returns
AUR_ERR_NOMEM, and every handle type then opens, adds, searches and closes normally on the same device.  The failing
requests are far larger than any card, so cudaMalloc refuses them outright and nothing is held."""

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index, KeywordIndex, KeywordVocab
from oracle import cosine_topk as O

pytestmark = pytest.mark.gpu


def _nomem(make):
    with pytest.raises(N.AuroraError) as ei:
        make()
    assert ei.value.code == N.AUR_ERR_NOMEM


def test_index_rows_allocation_failure_then_normal_use():
    _nomem(lambda: Index(8192, 2**31 - 64))      # 32 TiB of rows, after the streams were made
    rng = np.random.default_rng(0)
    C = O.round_to_bf16(rng.standard_normal((300, 256)).astype(np.float32))
    Q = O.round_to_bf16(rng.standard_normal((5, 256)).astype(np.float32))
    with Index(256, 512) as ix:
        ix.add(C, np.arange(300, dtype=np.int64))
        ids, _ = ix.search(Q, 7)
        assert np.array_equal(ids, O.cosine_topk(Q, C, 7)[0])


def test_keyword_postings_allocation_failure_then_normal_use():
    _nomem(lambda: KeywordIndex(1000, postings_capacity=2**42))   # 32 TiB of postings, after the row arrays
    vocab = KeywordVocab(0)
    store = KeywordIndex(16)
    try:
        store.add_text(vocab, [0, 1], ["alpha beta", "gamma alpha delta"])   # term ids 0 .. 3 by first occurrence
        ids, _, snap = store.search(np.array([0, 2], np.int32), np.array([0, 1, 2], np.int64), 2)
        assert snap == 2
        assert sorted(ids[0].tolist()) == [0, 1]
        assert ids[1].tolist() == [1, -1]
    finally:
        store.close()
        vocab.close()


def test_closing_handles_gives_their_memory_back():
    """Open, use and close every handle type several times over: the device's free memory comes back each time.  Each
    round holds well over a GiB, so a handle that kept any of its big arrays would lose more than the tolerance."""
    import torch

    from aurora_b200.encoder import Encoder, EncoderConfig

    rng = np.random.default_rng(1)
    C = O.round_to_bf16(rng.standard_normal((1000, 1024)).astype(np.float32))
    cfg = EncoderConfig(hidden=128, layers=1, heads=2, inter=256, vocab=120, max_pos=512, pool="mean")

    def round_trip():
        with Index(1024, 1 << 19) as ix:                      # 1 GiB of rows
            ix.add(C, np.arange(1000, dtype=np.int64))
            ix.search(C[:3], 5)
        vocab, store = KeywordVocab(0), KeywordIndex(1 << 20, postings_capacity=1 << 26)   # 512 MiB of postings
        store.add_text(vocab, [0, 1], ["alpha beta", "gamma alpha delta"])
        store.search(np.array([0], np.int32), np.array([0, 1], np.int64), 2)
        store.close(); vocab.close()
        with Encoder(cfg, max_tokens=1 << 19, max_seqs=8):    # 128 MiB per activation buffer
            pass

    torch.cuda.synchronize()
    round_trip()                                              # modules load and contexts appear once
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(4):
        round_trip()
    assert free0 - torch.cuda.mem_get_info()[0] < (256 << 20)

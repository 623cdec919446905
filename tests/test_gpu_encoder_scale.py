"""The encoder at the batch the benchmark runs (bench.py's encoder leg and cfg3: 192 chunks of about N(384, 96) tokens,
71 331 tokens) and at the shapes the project serves, checked per token and one layer at a time.

Teacher forcing: the device's hidden states after L layers are compared with the fp64 bf16-store oracle's layer L run
on the device's own output after L - 1 layers, so every layer is held to the same per-token criterion
(BD.HIDDEN_ULPS bf16 ulps of max(|ref|, row RMS)) at any depth.  Free-running, the error of a correct encoder grows with
depth and the criterion would have to grow with it; teacher-forced, it does not, and a corrupted tile or a duplicated
row in any one layer still scores far above it (tests/test_bounds.py holds the emulation and those mutants to it).

The fp64 oracle runs on a sample of the batch: its first two and last two synthetic sequences, sequences of every
edge length appended to it, and the sequence that straddles token 65 536."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dataclasses import replace

from aurora_b200.encoder import Encoder
from oracle import bert_encoder as B
from oracle.cosine_topk import bf16_bits_to_f32
from tests import bounds as BD
from tests.test_gpu_encoder import _check_pooled, _mirror

# attention key-block and query-block edges, and the position table's end
EDGE_LENS = [1, 2, 127, 128, 129, 511, 512]

MODELS = {   # name: (config, synthetic sequences before the edge lengths, layers checked)
    "bge_base": (B.BGE_BASE, 192, 12),      # LayerNorm with 3 chunks per lane, BN 256
    "minilm_l6": (B.MINILM_L6, 192, 6),     # head dim 32 zero-padded to 64, BN 128 with 6 ring slots, mean pooling
    "bge_large": (B.BGE_LARGE, 62, 2),      # 4 chunks per lane, I 4096; 24 413 tokens
}

E2E_ABS_TOL = 6e-3     # per component of a 12-layer pooled vector (see test_bge_base_end_to_end_and_batch_invariance)


def _batch(cfg, n_seq):
    """bench.py's chunk batch (B.synth_batch with seed 1003) followed by one sequence of each edge length.  The total
    is odd, so layernorm_kernel's last warp has no second row."""
    tok, cu = B.synth_batch(cfg, n_seq, 1003)
    rng = np.random.default_rng(1004)
    edges = [rng.integers(1000, cfg.vocab, n).astype(np.int32) for n in EDGE_LENS]
    for e in edges:
        e[0], e[-1] = 101, 102
    tok = np.concatenate([tok, *edges])
    cu = np.concatenate([cu, cu[-1] + np.cumsum(EDGE_LENS)]).astype(np.int32)
    assert cu[-1] % 2 == 1
    return tok, cu


def _sample(cu, n_seq):
    """(sequence indices, their packed rows, their cu_seqlens) of the sequences the oracle checks."""
    seqs = {0, 1, n_seq - 2, n_seq - 1, *range(n_seq, len(cu) - 1)}
    if cu[-1] > 65536:
        s = int(np.searchsorted(cu, 65536, side="right")) - 1
        assert cu[s] < 65536 < cu[s + 1]
        seqs.add(s)
    seqs = sorted(seqs)
    rows = np.concatenate([np.arange(cu[s], cu[s + 1]) for s in seqs])
    sub_cu = np.zeros(len(seqs) + 1, np.int32)
    sub_cu[1:] = np.cumsum([cu[s + 1] - cu[s] for s in seqs])
    return seqs, rows, sub_cu


def _weights(cfg):
    # init_weights draws the parameters in weight_names order from one generator, so these are the full model's first
    # cfg.layers layers
    return B.init_weights(cfg, seed=7, bf16=True)


@pytest.mark.parametrize("model", list(MODELS))
def test_hidden_states_layer_by_layer(model):
    """For each depth L, a fresh encoder with L layers encodes the whole batch; its hidden states on the sampled
    sequences must be within BD.HIDDEN_ULPS ulps of the oracle's layer L applied to the device's hidden states after
    L - 1 layers (to the oracle's embedding for L = 1).  The worst and the 99.9th percentile are printed per layer."""
    cfg, n_seq, depth = MODELS[model]
    cfg = replace(cfg, layers=depth)
    w = _weights(cfg)
    tok, cu = _batch(cfg, n_seq)
    seqs, rows, sub_cu = _sample(cu, n_seq)
    x_in = B.embed_tokens(cfg, w, tok[rows], sub_cu, bf16_stores=True)
    worst = []
    for L in range(1, depth + 1):
        cfg_l = replace(cfg, layers=L)
        with Encoder(_mirror(cfg_l), max_tokens=int(cu[-1]), max_seqs=len(cu) - 1) as enc:
            enc.load_weights({k: w[k] for k in B.weight_names(cfg_l)})
            enc.encode_packed(tok, cu)
            got = bf16_bits_to_f32(enc.hidden_states()[rows]).astype(np.float64)
        ref = B.encoder_layer(cfg, w, L - 1, x_in, sub_cu, bf16_stores=True)
        e = BD.bf16_ulps(got, ref)
        worst.append(float(e.max()))
        print(f"{model} layer {L}: max {e.max():.2f}, p99.9 {np.quantile(e, 0.999):.2f} ulps of max(|ref|, row RMS) "
              f"({len(seqs)} sequences, {len(rows)} of {int(cu[-1])} tokens)")
        x_in = got
    assert max(worst) <= BD.HIDDEN_ULPS, worst


def test_bge_base_end_to_end_and_batch_invariance():
    """Each sampled sequence encoded alone in the same encoder, whose workspace still holds the big batch's rows: its
    hidden states and pooled vector must be bit-identical to its rows in the big batch (every GEMM row, attention row
    and LayerNorm row is computed the same way wherever it sits in the batch).  Then the 12-layer pooled vectors of the
    sampled sequences against the fp64 oracle: cosine >= COS_TOL as in test_gpu_encoder, and every component within
    E2E_ABS_TOL.

    E2E_ABS_TOL is 6e-3 here rather than test_gpu_encoder's 4e-3.  Measured on an H100 80GB HBM3 (700 W limit): the
    per-sequence max |d| of the 12 sampled sequences runs from 1.47e-3 to 4.06e-3 (the largest on the 128-token
    sequence), with cosine >= 0.999927.  The excess is not traced to any kernel.  The fp32 bf16-store emulation on the
    CPU gives 1.59e-3 to 4.03e-3 on the same sequences, the largest on the same 128-token sequence.  That emulation is
    B.encode_tokens in float32 with bf16_stores, so no kernel takes part.  Its error comes from the bf16 hidden states
    between kernels compounding over 12 layers.  test_hidden_states_layer_by_layer holds each layer on its own to
    BD.HIDDEN_ULPS."""
    cfg, n_seq, _ = MODELS["bge_base"]
    w = _weights(cfg)
    tok, cu = _batch(cfg, n_seq)
    seqs, rows, sub_cu = _sample(cu, n_seq)
    with Encoder(_mirror(cfg), max_tokens=int(cu[-1]), max_seqs=len(cu) - 1) as enc:
        enc.load_weights(w)
        pooled = enc.encode_packed(tok, cu)
        hidden = enc.hidden_states()
        for s in seqs:
            lo, hi = int(cu[s]), int(cu[s + 1])
            alone = enc.encode_packed(tok[lo:hi], np.array([0, hi - lo], np.int32))
            assert np.array_equal(alone[0].view(np.uint32), pooled[s].view(np.uint32)), f"sequence {s}: pooled vector"
            assert np.array_equal(enc.hidden_states(), hidden[lo:hi]), f"sequence {s}: hidden states"
    got, ref = pooled[seqs].astype(np.float64), B.encode(cfg, w, tok[rows], sub_cu)
    cos = (got * ref).sum(axis=1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    for s, c, d in zip(seqs, cos, np.abs(got - ref).max(axis=1)):
        print(f"bge_base 12 layers, sequence {s} ({cu[s + 1] - cu[s]} tokens): cosine {c:.6f}, max |d| {d:.2e}")
    _check_pooled(got, ref, E2E_ABS_TOL)

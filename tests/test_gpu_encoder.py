"""GPU parity of the encoder path (SURVEY.md section 8 a6/a11) through the C ABI: the wgmma GEMM
and attention kernels against numpy, the whole forward against oracle/bert_encoder.py and against
the HF-BertModel golden vectors, and the fused encode -> append -> search ingest path.

Tolerance (floating point, stated here as the tier asks): the GPU keeps activations in bf16
between kernels (fp32 accumulation inside them) while the oracle runs fp64 on the same
bf16-rounded weights.  A pooled, L2-normalised vector must have cosine >= 0.9995 with the oracle's
and every component within 1e-2; single kernels must keep every output element within its own error bound, derived
from the arithmetic the kernel does (tests/bounds.py)."""

import ctypes as C
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from aurora_b200 import _native as N
from aurora_b200.encoder import EmbeddingClient, Encoder, EncoderConfig
from aurora_b200.engine import Index, to_bf16_bits
from oracle import bert_encoder as B
from oracle.cosine_topk import bf16_bits_to_f32
from tests import bounds as BD
from tests.test_oracle_bert import constant_row_weights

# Floating-point tolerance of the encoder path (bf16 activations between kernels, fp32 accumulation) against the fp64
# oracle on the same bf16-rounded weights: pooled unit vectors must agree to cosine >= 0.9999 and 4e-3 per component
# (a regression of either shows up here).
COS_TOL, ABS_TOL = 0.9999, 4e-3


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _mirror(cfg_o: B.BertConfig) -> EncoderConfig:
    return EncoderConfig(hidden=cfg_o.hidden, layers=cfg_o.layers, heads=cfg_o.heads, inter=cfg_o.inter, vocab=cfg_o.vocab,
                         max_pos=cfg_o.max_pos, type_vocab=cfg_o.type_vocab, ln_eps=cfg_o.ln_eps, pool=cfg_o.pool,
                         normalize=cfg_o.normalize)


SMALL = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")


GEMM_SHAPES = [(128, 256, 64, 0), (130, 128, 192, 0), (1000, 768, 768, 2), (777, 3072, 768, 1), (640, 768, 3072, 2),
               (500, 384, 384, 1), (1, 256, 64, 0),
               # the pair-tile boundary (256 rows), single-CTA tile boundary (128), bge-large wo2 (K 4096), N = 384 (BN 128,
               # three tiles) and 2304 (qkv of bge-base)
               (255, 768, 768, 0), (256, 768, 768, 2), (257, 768, 768, 1), (127, 384, 256, 0), (129, 384, 256, 2),
               (257, 1024, 4096, 2), (300, 2304, 768, 0)]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k,epi", GEMM_SHAPES)
def test_gemm_matches_numpy(m, n, k, epi, cta_group):
    _gemm_case(m, n, k, epi, cta_group)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("case", ["gelu_spread", "resid_large"])
def test_gemm_epilogue_edges(case, cta_group):
    """GELU inputs over [-6, 6] (both tails of the erf approximation) and a residual 2^10 times the product (catches
    a residual added after the bf16 rounding of the product)."""
    if case == "gelu_spread":
        _gemm_case(257, 384, 64, 1, cta_group, spread=True)
    else:
        _gemm_case(129, 768, 192, 2, cta_group, big_resid=True)


def _gemm_case(m, n, k, epi, cta_group, spread=False, big_resid=False, rows=None):
    """rows: check only these output rows against the fp64 reference (for a shape whose full reference is too large
    to compute); the residual is then only made when the epilogue reads it."""
    lib = N.load()
    a, w, bias, resid = BD.gemm_inputs(m, n, k, seed=m * 7 + n + k + epi, spread=spread, big_resid=big_resid,
                                       with_resid=rows is None or epi == 2)
    out = np.zeros((m, n), dtype=np.uint16)
    N.check(lib.aur_debug_gemm(0, _ptr(to_bf16_bits(a)), _ptr(to_bf16_bits(w)), _ptr(bias),
                               None if resid is None else _ptr(to_bf16_bits(resid)), m, n, k, epi, cta_group, _ptr(out), None))
    sel = slice(None) if rows is None else rows
    ref, bound = BD.gemm_reference(a[sel], w, bias, None if resid is None else resid[sel], epi)
    BD.assert_within(f"gemm m={m} n={n} k={k} epi={epi} cta_group={cta_group}", bf16_bits_to_f32(out[sel]), ref, bound)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _many_tile_rows(n_tiles, groups, tile_m, last_round):
    """Rows m, not a multiple of 128, whose m_tiles x n_tiles tiles give each of ``groups`` CTA groups at least 3
    tiles.  last_round: "full" (every group takes the same number of tiles), "short" (a few groups take one more) or
    "long" (all but a few groups take one more)."""
    ok = {"full": lambda r: r == 0, "short": lambda r: 0 < r <= n_tiles, "long": lambda r: r >= groups - n_tiles}[last_round]
    m_tiles = -(-3 * groups // n_tiles)
    while not ok(m_tiles * n_tiles % groups):
        m_tiles += 1
    return m_tiles * tile_m - 37


# (bn, cta_group, epi, k, last_round): K 64, 320, 448 and 1088 are 1, 5, 7 and 17 k-blocks, none a multiple of the
# ring's 4 (BN 256) or 6 (BN 128) slots, so tiles after the first start mid-lap; K 768 (12 k-blocks) is aligned
MANY_TILE_CASES = [(bn, g, epi, (64, 320, 448, 1088)[i % 4], ("short", "long")[i % 2])
                   for i, (bn, g, epi) in enumerate((bn, g, epi) for bn in (128, 256) for g in (1, 2) for epi in (0, 1, 2))]
MANY_TILE_CASES += [(256, 2, 2, 768, "short"), (128, 1, 0, 320, "full")]


@pytest.mark.parametrize("bn,cta_group,epi,k,last_round", MANY_TILE_CASES)
def test_gemm_many_tiles_per_cta(bn, cta_group, epi, k, last_round):
    """The persistent schedule with at least 3 tiles per CTA group: the TMA ring's stage / phase and the full / empty
    barriers carry over from tile to tile, and the producer streams the next tile's k-blocks during the epilogue.
    Every element is checked against the fp64 reference.  The shape is chosen from the device's SM count; the
    premise (tiles per group, ring laps per tile) is computed with launch_one's formulas and printed."""
    n = 3 * bn                                  # three N tiles; 384 keeps aur_debug_gemm's BN at 128
    groups_max = _sm_count() // cta_group
    m = _many_tile_rows(n // bn, groups_max, 128 * cta_group, last_round)
    bn_, stages, tiles, groups, kb = BD.gemm_schedule(m, n, k, cta_group, _sm_count())
    q, r = divmod(tiles, groups)
    print(f"gemm m={m} n={n} k={k} bn={bn_} cta_group={cta_group}: {tiles} tiles over {groups} groups = {q} rounds + "
          f"{r}; {kb} k-blocks per tile in a {stages}-slot ring = {kb / stages:.2f} laps")
    assert bn_ == bn and m % 128 and q >= 3 and (r == 0) == (last_round == "full")
    assert (kb % stages == 0) == (k == 768)
    _gemm_case(m, n, k, epi, cta_group)


def test_gemm_benchmark_scale():
    """bge-base's FFN up-projection over the benchmark's 192-chunk batch: 71 331 rows (odd, more than 65 535), N 3072,
    K 768, GELU, CTA pairs: about 50 tiles per pair.  Checked on the first and last 300 rows and every 97th row between
    (97 is coprime with the 256-row tile, so the checked rows land on every row position of a tile)."""
    m, n, k = 71331, 3072, 768
    bn, stages, tiles, groups, kb = BD.gemm_schedule(m, n, k, 2, _sm_count())
    print(f"gemm m={m} n={n} k={k}: {tiles} tiles over {groups} pairs = {tiles / groups:.1f} per pair")
    assert tiles // groups >= 3
    rows = np.unique(np.r_[0:300, 300:m - 300:97, m - 300:m])
    _gemm_case(m, n, k, 1, 2, rows=rows)


def _attention(heads, lens, kind="random", seed=None):
    lib = N.load()
    hidden = heads * 64
    qkv, cu = BD.attention_inputs(heads, lens, seed=sum(lens) + heads if seed is None else seed, kind=kind)
    out = np.zeros((int(cu[-1]), hidden), dtype=np.uint16)
    N.check(lib.aur_debug_attention(0, _ptr(to_bf16_bits(qkv)), _ptr(cu), len(lens), heads, hidden, _ptr(out), None))
    ref, bound = BD.attention_reference(qkv, cu, heads, hidden)
    BD.assert_within(f"attention heads={heads} kind={kind} lens={list(lens)[:8]}", bf16_bits_to_f32(out), ref, bound)


@pytest.mark.parametrize("heads,lens", [(2, [1]), (2, [5]), (2, [128]), (2, [129, 1, 64]), (12, [300, 17, 512, 384, 200]),
                                        (4, [512, 512, 511]), (1, [127, 256, 257]),
                                        # every key-block count and query-block boundary
                                        (2, [1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512])])
def test_attention_matches_numpy(heads, lens):
    _attention(heads, lens)


@pytest.mark.parametrize("kind,lens", [("onehot", [129, 385, 512]), ("lastmax", [1, 2, 128, 129, 257, 511]),
                                       ("leak", [129, 300, 128, 40, 512, 257])])
def test_attention_edges(kind, lens):
    """Nearly one-hot rows (exp underflows), every query's largest logit on the last valid key (a key dropped by the
    mask shows), and neighbours in the packed batch whose keys are 8x larger (a key leaking across the mask shows)."""
    _attention(4, lens, kind)


def test_attention_large_batch():
    """A large batch (2 000 sequences x 2 query blocks x 12 heads = 48 000 work units, far more than the GPU holds at
    once).  Checked against numpy on a sample of sequences from the start, the middle and the end of the batch."""
    lib = N.load()
    heads, hidden, n_seq = 12, 768, 2000
    rng = np.random.default_rng(2024)
    lens = rng.integers(129, 150, n_seq)
    cu = np.zeros(n_seq + 1, dtype=np.int32)
    cu[1:] = np.cumsum(lens)
    T = int(cu[-1])
    qkv_bits = to_bf16_bits((rng.standard_normal((T, 3 * hidden), dtype=np.float32) * 1.5))
    out = np.zeros((T, hidden), dtype=np.uint16)
    N.check(lib.aur_debug_attention(0, _ptr(qkv_bits), _ptr(cu), n_seq, heads, hidden, _ptr(out), None))
    worst = 0.0
    for s in list(range(0, 6)) + list(range(990, 1000)) + list(range(n_seq - 6, n_seq)):
        a, b = int(cu[s]), int(cu[s + 1])
        ref, bound = BD.attention_reference(bf16_bits_to_f32(qkv_bits[a:b]), np.array([0, b - a]), heads, hidden)
        r = BD.ratio(bf16_bits_to_f32(out[a:b]), ref, bound)
        assert r <= 1.0, (s, r)
        worst = max(worst, r)
    print(f"attention large batch: max(err / bound) = {worst:.4f}")


# ------------------------------------------------------------------ per-token hidden states and pooling
MINILM_SHAPE = B.BertConfig(hidden=384, layers=1, heads=12, inter=1536, vocab=120, max_pos=512, pool="mean")


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("shape", ["small", "minilm"])
def test_hidden_states_match_the_bf16_store_oracle(shape, layers):
    """Encoder.hidden_states() token by token against the oracle that rounds to bf16 exactly where the GPU stores bf16
    (embedding LayerNorm, LayerNorm, attention with the zero-padded head dim 32 of the MiniLM shape included).

    Every element is within 8 bf16 ulps of max(|ref|, RMS of its token's row) (measured on an H100: at most 5).  A LayerNorm output inherits the error
    of its input's bf16 stores, whose ulps are set by the row's magnitude, not by the element's: one store that
    rounds the other way (fp32 accumulation sits on the other side of a rounding boundary than fp64) moves small
    elements of an O(1) row by many of their own ulps.  Counted in ulps of max(|ref|, 1/16) the head-dim-64 shape
    stays within 2 ulps for 99.9 % of the elements and 8 for all; the MiniLM shape (H 384, I 1536) does not, and
    the figures are printed."""
    base = SMALL if shape == "small" else MINILM_SHAPE
    cfg_o = B.BertConfig(**{**base.__dict__, "layers": layers})
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 7, 17 + layers, mean_len=150, std_len=140, min_len=1, max_len=400)
    with Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=16) as enc:
        enc.load_weights(w)
        enc.encode_packed(tok, cu)
        got = bf16_bits_to_f32(enc.hidden_states()).astype(np.float64)
    ref = B.encode_tokens(cfg_o, w, tok, cu, bf16_stores=True)
    e = BD.bf16_ulps(got, ref, 1.0 / 16)
    within2, worst = float((e <= 2).mean()), float(e.max())
    e_row = BD.bf16_ulps(got, ref)
    print(f"hidden states {shape} layers={layers}: {100 * within2:.3f} % within 2 ulps of max(|ref|, 1/16), "
          f"{100 * float((e == 0).mean()):.2f} % exact, max {worst:.1f} ulps; max {float(e_row.max()):.2f} ulps of "
          f"max(|ref|, row RMS); {e.size} elements")
    assert float(e_row.max()) <= BD.HIDDEN_ULPS
    if shape == "small":
        assert within2 >= 0.999 and worst <= 8


@pytest.mark.parametrize("pool,normalize", [("cls", False), ("cls", True), ("mean", False), ("mean", True)])
@pytest.mark.parametrize("hidden", [128, 768, 1024])
def test_pool_kernel_against_fp64_pool_of_its_own_hidden_states(hidden, pool, normalize):
    """The pool kernel alone: the GPU's fp32 pooled vectors against an fp64 pool of the GPU's own hidden states.  A
    mean of n bf16 values summed in fp32 is within (n + 4) u max|x| per component; normalising divides that by |v|
    and adds the error of |v| (an H-term fp32 sum of squares, a square root and a division).  One thread per pair of
    dims: H 768 is 12 warps, H 1024 all 16 warps of the 512-thread block in the norm's reduction."""
    cfg_o = B.BertConfig(**{**SMALL.__dict__, "hidden": hidden, "heads": hidden // 64, "inter": 2 * hidden, "layers": 1,
                            "pool": pool, "normalize": normalize})
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 9, 5, mean_len=150, std_len=140, min_len=1, max_len=512)
    with Encoder(_mirror(cfg_o), max_tokens=8192, max_seqs=16) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(tok, cu).astype(np.float64)
        hs = bf16_bits_to_f32(enc.hidden_states()).astype(np.float64)
    H = cfg_o.hidden
    for s in range(len(cu) - 1):
        x = hs[cu[s]:cu[s + 1]] if pool == "mean" else hs[cu[s]:cu[s] + 1]
        n = x.shape[0]
        v = x.mean(axis=0)
        bound = (n + 4) * BD.U * np.abs(x).max(axis=0)
        ref = v
        if normalize:
            nv = np.linalg.norm(v)
            ref = v / nv
            bound = bound / nv * (1 + np.sqrt(H) * np.abs(ref)) + (H + 4) * BD.U * np.abs(ref)
        BD.assert_within(f"pool {pool} normalize={normalize} seq {s} (n={n})", got[s], ref, bound)


def test_constant_row_layernorm_is_exact_on_gpu():
    """A token whose embedding-LayerNorm input is a constant row (pos / type rows zero, constant word row, eps 1e-12)
    and whose later LayerNorm inputs are constant too (zero layer weights, constant LN biases) comes out as exactly
    bf16(ln2_b): each LayerNorm must return exactly its bias for a zero-variance row, with no NaN."""
    cfg_o = B.BertConfig(**{**SMALL.__dict__, "layers": 1})
    w = constant_row_weights(cfg_o)
    tok, cu = np.array([1, 5, 5, 9, 5, 2], np.int32), np.array([0, 6], np.int32)
    with Encoder(_mirror(cfg_o), max_tokens=256, max_seqs=2) as enc:
        enc.load_weights(w)
        enc.encode_packed(tok, cu)
        got = bf16_bits_to_f32(enc.hidden_states())
    assert np.array_equal(got[tok == 5], np.broadcast_to(w["l0.ln2_b"], (3, cfg_o.hidden)))


def _check_pooled(got, ref, abs_tol=ABS_TOL):
    cos = (got * ref).sum(axis=1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    print(f"pooled parity: min cosine {cos.min():.6f}, max |d| {np.abs(got - ref).max():.2e}")     # (pytest -s / on failure)
    assert cos.min() >= COS_TOL, cos.min()
    assert np.abs(got - ref).max() <= abs_tol, np.abs(got - ref).max()


@pytest.mark.parametrize("pool,normalize", [("cls", True), ("mean", True), ("mean", False)])
def test_small_encoder_matches_oracle(pool, normalize):
    cfg_o = B.BertConfig(**{**SMALL.__dict__, "pool": pool, "normalize": normalize})
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 9, 21, mean_len=150, std_len=140, min_len=1, max_len=512)
    with Encoder(_mirror(cfg_o), max_tokens=8192, max_seqs=16) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(tok, cu)
        bits = enc.encode_packed(tok, cu, bf16=True)
        st = enc.stats()
    ref = B.encode(cfg_o, w, tok, cu)
    if normalize:
        _check_pooled(got, ref)
    else:
        assert np.abs(got - ref).max() <= 2e-2 * np.abs(ref).max() + 1e-2
    np.testing.assert_array_equal(bits, to_bf16_bits(got))          # both outputs are the same vector
    assert st["tokens"] == len(tok) and st["seqs"] == 9 and st["launches"] == 2 + 7 * cfg_o.layers


def test_bge_base_matches_hf_golden():
    """bge-base-en architecture (random-init, seed 7) against transformers.BertModel's output."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "bert_ref.json")) as f:
        case = next(c for c in json.load(f)["cases"] if c["name"] == "bge_base")
    cfg_o = B.BertConfig(**case["cfg"])
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    with Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=8) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(np.asarray(case["tokens"], np.int32), np.asarray(case["cu_seqlens"], np.int32))
    _check_pooled(got, np.asarray(case["pooled"]))


def test_bge_large_matches_hf_golden():
    """bge-large-en architecture (H1024 / L24 / 16 heads / I4096: the encoder behind BASELINE config 4's 1024-d vectors),
    random-init, against transformers.BertModel's output, then a longer ragged batch against the oracle."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "bert_ref.json")) as f:
        case = next(c for c in json.load(f)["cases"] if c["name"] == "bge_large")
    cfg_o = B.BertConfig(**case["cfg"])
    assert (cfg_o.hidden, cfg_o.layers, cfg_o.heads, cfg_o.inter) == (1024, 24, 16, 4096)
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    with Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=8) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(np.asarray(case["tokens"], np.int32), np.asarray(case["cu_seqlens"], np.int32))
        _check_pooled(got, np.asarray(case["pooled"]))
        tok, cu = B.synth_batch(cfg_o, 3, 44, mean_len=120, std_len=60, min_len=8, max_len=300)
        got2 = enc.encode_packed(tok, cu)
        assert enc.stats()["launches"] == 2 + 7 * 24
    _check_pooled(got2, B.encode(cfg_o, w, tok, cu, dtype=np.float32).astype(np.float64))


def test_minilm_l6_matches_hf_golden():
    """all-MiniLM-L6-v2 architecture (H384 / 12 heads = head dim 32, masked-mean pooling; the model the
    reference deploys, docker-compose.yaml:528), random-init, against transformers.BertModel."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "bert_ref.json")) as f:
        case = next(c for c in json.load(f)["cases"] if c["name"] == "minilm_l6")
    cfg_o = B.BertConfig(**case["cfg"])
    assert cfg_o.hidden // cfg_o.heads == 32
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    with Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=8) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(np.asarray(case["tokens"], np.int32), np.asarray(case["cu_seqlens"], np.int32))
    _check_pooled(got, np.asarray(case["pooled"]))
    # and a longer ragged batch against the oracle
    tok, cu = B.synth_batch(cfg_o, 7, 33, mean_len=180, std_len=150, min_len=1, max_len=512)
    with Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=8) as enc:
        enc.load_weights(w)
        got = enc.encode_packed(tok, cu)
    _check_pooled(got, B.encode(cfg_o, w, tok, cu, dtype=np.float32).astype(np.float64))


def test_batch_invariance_and_split_calls():
    """A sequence's vector does not depend on what else is in the batch (packed, no padding)."""
    cfg_o = SMALL
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 6, 5, mean_len=60, std_len=50, min_len=1, max_len=300)
    seqs = [tok[cu[i]:cu[i + 1]].tolist() for i in range(6)]
    with Encoder(_mirror(cfg_o), max_tokens=512, max_seqs=4) as enc:      # forces several calls
        enc.load_weights(w)
        together = enc.encode(seqs)
        alone = np.stack([enc.encode([s])[0] for s in seqs])
    np.testing.assert_array_equal(together, alone)


def test_encode_append_then_search_finds_the_chunk():
    cfg_o = SMALL
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    tok, cu = B.synth_batch(cfg_o, 40, 9, mean_len=40, std_len=20, min_len=4, max_len=128)
    ids = np.arange(1000, 1040, dtype=np.int64)
    with Encoder(_mirror(cfg_o), max_tokens=8192, max_seqs=64) as enc, Index(cfg_o.hidden, 256) as ix:
        enc.load_weights(w)
        enc.encode_append(ix, tok, cu, ids)
        assert ix.stats()["live"] == 40
        q = enc.encode_packed(tok, cu, bf16=True)
        got_ids, got_sc = ix.search(q, 3)
        # re-ingesting the same ids is an upsert, not a duplicate (weaviate_client.py:172)
        enc.encode_append(ix, tok, cu, ids)
        assert ix.stats()["live"] == 40
    ref = B.encode(cfg_o, w, tok, cu)
    np.testing.assert_array_equal(got_ids[:, 0], ids)
    assert np.all(got_sc[:, 0] > 0.9999)
    # the runner-up's score agrees with the oracle's embedding geometry (random-init embeddings are
    # all close together, so the runner-up's identity is not stable under bf16 noise; its score is)
    sims = ref @ ref.T
    np.fill_diagonal(sims, -1)
    assert np.abs(got_sc[:, 1] - sims.max(axis=1)).max() <= 2e-3


def test_encoder_error_paths():
    cfg_o = SMALL
    with Encoder(_mirror(cfg_o), max_tokens=256, max_seqs=2) as enc:
        tok, cu = np.array([1, 5, 2], np.int32), np.array([0, 3], np.int32)
        with pytest.raises(N.AuroraError) as e:
            enc.encode_packed(tok, cu)                                  # parameters not loaded
        assert e.value.code == N.AUR_ERR_INVALID
        enc.load_weights(B.init_weights(cfg_o, seed=7, bf16=True))
        with pytest.raises(N.AuroraError):
            enc.load_weights({"l0.wo": np.zeros((3, 3), np.float32)})  # wrong shape
        with pytest.raises(N.AuroraError):
            enc.load_weights({"nope": np.zeros(1, np.float32)})
        with pytest.raises(N.AuroraError):
            enc.encode_packed(np.array([1, 500, 2], np.int32), cu)      # token id out of range
        with pytest.raises(N.AuroraError) as e:
            enc.encode_packed(np.ones(300, np.int32), np.array([0, 300], np.int32))
        assert e.value.code == N.AUR_ERR_NOMEM
        with pytest.raises(N.AuroraError):
            enc.encode_packed(np.ones(3, np.int32), np.array([0, 1, 2, 3], np.int32))   # > max_seqs
        with pytest.raises(N.AuroraError):
            enc.encode_packed(np.ones(2, np.int32), np.array([0, 0, 2], np.int32))      # empty sequence
        assert enc.encode_packed(tok, cu).shape == (1, cfg_o.hidden)   # still usable afterwards
    with pytest.raises(N.AuroraError) as e:
        Encoder(EncoderConfig(hidden=256, layers=1, heads=16, inter=512))               # head dim 16
    assert e.value.code == N.AUR_ERR_UNSUPPORTED


def test_embedding_client_mirror():
    cfg_o = SMALL
    enc = Encoder(_mirror(cfg_o), max_tokens=1024, max_seqs=8)
    enc.load_weights(B.init_weights(cfg_o, seed=7, bf16=True))
    tokenize = lambda t: [1] + [3 + (hash(w) % 100) for w in t.lower().split()][:60] + [2]
    client = EmbeddingClient(enc, tokenize)
    assert client.embed("") is None and client.embed("   ") is None     # embedding_client.py:48-49
    v = client.embed("disk pressure on node-3")
    assert isinstance(v, list) and len(v) == cfg_o.hidden and abs(sum(x * x for x in v) - 1.0) < 1e-3
    batch = client.embed_batch(["disk pressure on node-3", "", "pod crashloop"])
    assert batch[1] is None and batch[0] == v and len(batch[2]) == cfg_o.hidden
    client.close()
    assert client.embed("after close") is None                           # any failure -> None (:66-70)


def test_retriever_with_cuda_encoder_end_to_end():
    """search_knowledge_base / insert_chunks (weaviate_client.py:136-285 signatures) running on the
    CUDA encoder + CUDA shard, fused ingest included."""
    from aurora_b200 import retriever as R
    from aurora_b200.encoder import TextEncoder

    cfg_o = SMALL
    enc = Encoder(_mirror(cfg_o), max_tokens=4096, max_seqs=64)
    enc.load_weights(B.init_weights(cfg_o, seed=7, bf16=True))
    vocab = {}
    tokenize = lambda t: [1] + [vocab.setdefault(w, 3 + len(vocab) % 110) for w in t.lower().split()][:100] + [2]
    R.configure(encoder=TextEncoder(enc, tokenize), capacity=1024, device=0)
    try:
        chunks = [{"content": f"runbook step {i}: restart service alpha-{i} and check queue depth", "heading_context": "Recovery",
                   "chunk_index": i} for i in range(12)]
        assert R.insert_chunks("u1", "doc1", "runbook.md", chunks, org_id="o1") == 12
        assert R.insert_chunks("u2", "doc2", "other.md", [{"content": "unrelated billing notes", "chunk_index": 0}]) == 1
        assert R.get_document_chunk_count("u1", "doc1") == 12
        q7 = "Recovery\nrunbook step 7: restart service alpha-7 and check queue depth"
        hits = R.search_knowledge_base("u1", q7, limit=3, alpha=1.0)                  # pure vector: score = cosine
        assert hits and hits[0]["chunk_index"] == 7 and hits[0]["document_id"] == "doc1" and hits[0]["score"] > 0.999
        hy = R.search_knowledge_base("u1", q7, limit=3)                               # default alpha=0.5: ranked fusion
        assert hy[0]["chunk_index"] == 7 and hy[0]["score"] == pytest.approx(1.0 / 60.0)
        assert set(hits[0]) == {"content", "heading_context", "source_filename", "document_id", "chunk_index", "score"}
        assert all(h["document_id"] == "doc1" for h in R.search_knowledge_base("u1", "billing", limit=5))   # tenant scope
        assert R.search_knowledge_base("u1", "   ") == []
        assert R.delete_document_chunks("u1", "doc1") == 12
        assert R.search_knowledge_base("u1", "runbook step 7", limit=3) == []
    finally:
        R.configure(encoder=None)
        enc.close()


def test_reference_chunker_output_through_tokenizer_encoder_and_shard():
    """SURVEY.md 8 a9 -> a4: the chunks the REAL reference chunker produced (tests/golden/chunker_ref.json, generated by
    oracle/gen_golden_chunks.py from document_processor.py) go through insert_chunks -> C++ WordPiece -> CUDA encoder ->
    shard, one aur_encode_text_append call per document; every chunk is then found again by its own text.  The
    4 196-character chunk (document_processor.py:266-267) exceeds the 512-token position table: it is embedded as the
    normalised mean of its token windows instead of being cut off."""
    from aurora_b200 import retriever as R
    from aurora_b200.encoder import TextEncoder
    from aurora_b200.wordpiece import NativeTokenizer, basic_tokenize

    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "chunker_ref.json"), encoding="utf-8"))
    docs = [d for d in gold["documents"] if d["chunks"]]
    words = sorted({w for d in docs for c in d["chunks"] for w in basic_tokenize(c["heading_context"] + " " + c["content"])})
    pieces = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + [w for w in words if len(w) <= 100]
    cfg_o = B.BertConfig(hidden=128, layers=2, heads=2, inter=256, vocab=len(pieces), max_pos=512, pool="cls")
    enc = Encoder(_mirror(cfg_o), max_tokens=8192, max_seqs=64)
    enc.load_weights(B.init_weights(cfg_o, seed=11, bf16=True))
    tok = NativeTokenizer(pieces)
    te = TextEncoder(enc, tok)
    R.configure(encoder=te, capacity=1024, device=0)
    try:
        total = 0
        for d in docs:
            n = R.insert_chunks("user-1", f"doc-{d['name']}", d["name"], d["chunks"], org_id="org-1")
            assert n == len(d["chunks"])
            assert R.get_document_chunk_count("user-1", f"doc-{d['name']}") == n
            total += n
        big = next(c for d in docs for c in d["chunks"] if len(c["content"]) > 4000)
        assert len(te._windows(big["content"])) >= 2                                   # really longer than the position table
        for d in docs:
            for c in d["chunks"]:
                text = (c["heading_context"] + "\n" if c["heading_context"] else "") + c["content"]
                if len(set(basic_tokenize(text))) < 3:
                    continue                                                        # ('xxxx...' chunks: all [UNK], identical vectors)
                hits = R.search_knowledge_base("user-1", text, limit=1, alpha=1.0)
                assert hits and hits[0]["document_id"] == f"doc-{d['name']}" and hits[0]["chunk_index"] == c["chunk_index"], (d["name"], c["chunk_index"])
                assert hits[0]["score"] > 0.999
        # the over-long chunk's stored vector is the normalised mean of its windows' vectors
        wins = te._windows(big["content"])
        from aurora_b200.encoder import pack_sequences
        wv = enc.encode_packed(*pack_sequences(wins))
        mean = wv.mean(axis=0); mean /= np.linalg.norm(mean)
        got = te.encode([big["content"]])[0]
        assert float(np.dot(got, mean)) > 0.9999
    finally:
        R.configure(encoder=None)
        tok.close()
        enc.close()


def test_bootstrap_from_environment_end_to_end(tmp_path, monkeypatch):
    """aurora_b200.bootstrap.configure_from_env: safetensors checkpoint (HF names) + vocab.txt -> CUDA encoder
    + shard behind the reference's module API, then snapshot -> restore.  all-MiniLM-L6-v2 dimensions
    (the model the reference deploys), random-init weights written to a temporary checkpoint."""
    import json
    import struct

    from aurora_b200 import bootstrap, retriever as R

    cfg_o = B.MINILM_L6
    w = B.init_weights(cfg_o, seed=7, bf16=True)
    h = cfg_o.hidden
    hf = {"embeddings.word_embeddings.weight": w["word_emb"], "embeddings.position_embeddings.weight": w["pos_emb"],
          "embeddings.token_type_embeddings.weight": w["type_emb"], "embeddings.LayerNorm.weight": w["emb_ln_g"],
          "embeddings.LayerNorm.bias": w["emb_ln_b"]}
    for l in range(cfg_o.layers):
        p, q = f"l{l}.", f"encoder.layer.{l}."
        for i, n in enumerate(("query", "key", "value")):
            hf[q + f"attention.self.{n}.weight"] = w[p + "wqkv"][i * h:(i + 1) * h]
            hf[q + f"attention.self.{n}.bias"] = w[p + "bqkv"][i * h:(i + 1) * h]
        for a, b in (("attention.output.dense.weight", "wo"), ("attention.output.dense.bias", "bo"),
                     ("attention.output.LayerNorm.weight", "ln1_g"), ("attention.output.LayerNorm.bias", "ln1_b"),
                     ("intermediate.dense.weight", "wi"), ("intermediate.dense.bias", "bi"), ("output.dense.weight", "wo2"),
                     ("output.dense.bias", "bo2"), ("output.LayerNorm.weight", "ln2_g"), ("output.LayerNorm.bias", "ln2_b")):
            hf[q + a] = w[p + b]
    header, blobs, off = {}, [], 0
    for name, arr in hf.items():
        raw = np.ascontiguousarray(arr, dtype="<f4").tobytes()
        header[name] = {"dtype": "F32", "shape": list(arr.shape), "data_offsets": [off, off + len(raw)]}
        blobs.append(raw); off += len(raw)
    hj = json.dumps(header).encode()
    ckpt = tmp_path / "model.safetensors"
    with open(ckpt, "wb") as f:
        f.write(struct.pack("<Q", len(hj))); f.write(hj)
        for b_ in blobs:
            f.write(b_)
    words = ["restart", "the", "payment", "service", "when", "latency", "spikes", "rotate", "database", "credentials",
             "kafka", "consumer", "lag", "alert", "runbook", "every", "ninety", "days"]
    vocab = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + words
    vocab += [f"[unused{i}]" for i in range(cfg_o.vocab - len(vocab))]
    (tmp_path / "vocab.txt").write_text("\n".join(vocab) + "\n", encoding="utf-8")
    snap = tmp_path / "snap"
    for k_, v_ in {"AURORA_B200_MODEL": "minilm-l6", "AURORA_B200_ENCODER_WEIGHTS": str(ckpt), "AURORA_B200_VOCAB": str(tmp_path / "vocab.txt"),
                   "AURORA_B200_CAPACITY": "512", "AURORA_B200_MAX_TOKENS": "4096", "AURORA_B200_MAX_SEQS": "32",
                   "AURORA_B200_SNAPSHOT": str(snap)}.items():
        monkeypatch.setenv(k_, v_)
    try:
        bootstrap.configure_from_env()
        chunks = [{"content": "restart the payment service when latency spikes", "heading_context": "", "chunk_index": 0},
                  {"content": "rotate database credentials every ninety days", "heading_context": "", "chunk_index": 1},
                  {"content": "kafka consumer lag alert runbook", "heading_context": "", "chunk_index": 2}]
        assert R.insert_chunks("u1", "doc", "runbook.md", chunks) == 3
        top = R.search_knowledge_base("u1", "kafka consumer lag alert runbook", limit=2, alpha=1.0)
        assert top[0]["chunk_index"] == 2 and top[0]["score"] > 0.999
        R._get_kb().save(str(snap))
        bootstrap.configure_from_env()                     # restores the snapshot
        again = R.search_knowledge_base("u1", "kafka consumer lag alert runbook", limit=2, alpha=1.0)
        assert [(r["chunk_index"], round(r["score"], 5)) for r in again] == [(r["chunk_index"], round(r["score"], 5)) for r in top]
        assert R.get_document_chunk_count("u1", "doc") == 3
    finally:
        R.configure(encoder=None)

"""The per-element bounds of tests/bounds.py have teeth: a numpy emulation of each tensor-core kernel (fp32
accumulation, bf16 stores where the kernel makes them) stays within its bound at the shapes the GPU tests use, and each
deliberately broken emulation -- a bug of the kind a kernel rewrite introduces -- fails it.  CPU only."""

import numpy as np
import pytest

from oracle import bert_encoder as B
from oracle.cosine_topk import bf16_bits_to_f32, f32_to_bf16_bits, round_to_bf16
from tests import bounds as BD

F32 = np.float32


def _rtz_bf16(x):
    return bf16_bits_to_f32((np.asarray(x, F32).view(np.uint32) >> np.uint32(16)).astype(np.uint16))


# ------------------------------------------------------------------------------------------------------ GEMM
def _gelu_erf_f32(x):
    """gelu_erf of gemm_tc.cu in fp32: Abramowitz-Stegun 7.1.26 erf."""
    x = np.asarray(x, F32)
    z = np.abs(x) * F32(0.70710678118654752)
    t = F32(1) / (F32(0.3275911) * z + F32(1))
    poly = F32(1.061405429) * t - F32(1.453152027)
    poly = poly * t + F32(1.421413741)
    poly = poly * t - F32(0.284496736)
    poly = poly * t + F32(0.254829592)
    e = np.exp2(z * F32(-1.4426950408889634) * z)
    erf_abs = F32(1) - poly * t * e
    h = F32(0.5) * x
    return h * np.copysign(erf_abs, x) + h


def _gelu_tanh_f32(x):
    x = np.asarray(x, F32)
    return F32(0.5) * x * (F32(1) + np.tanh(F32(0.7978845608) * (x + F32(0.044715) * x * x * x)))


def _scheduled_product(a, w, groups, bm, bn, stages, mutant=None):
    """a . w^T as gemm_tc_kernel's persistent schedule computes it: (bm x bn) tiles in row-major tile order, group g
    takes tiles g, g + groups, ... and accumulates each in fp32 over the 64-wide k-blocks it streams through a ring of
    ``stages`` slots.  Mutants: acc_carry (the accumulator is not zeroed between a group's tiles); stale_kblock (one
    k-block of group 0's second tile reads its slot one ring lap stale: the block loaded ``stages`` loads earlier)."""
    m, k = a.shape
    a = np.concatenate([a, np.zeros((-m % bm, k), F32)])          # the zero rows a partial last row of tiles covers
    m_tiles, n_tiles, kb = a.shape[0] // bm, w.shape[0] // bn, k // 64
    out = np.empty((a.shape[0], w.shape[0]), F32)
    for g in range(groups):
        loads, d = [], None                                        # (rows, cols, k-block) of each load, in ring order
        for i, t in enumerate(range(g, m_tiles * n_tiles, groups)):
            r = slice(t // n_tiles * bm, t // n_tiles * bm + bm)
            c = slice(t % n_tiles * bn, t % n_tiles * bn + bn)
            blocks = [(r, c, j) for j in range(kb)]
            read = list(blocks)
            if mutant == "stale_kblock" and g == 0 and i == 1:
                j = max(0, stages - kb)
                assert j < kb, "the ring never wraps inside the second tile"
                read[j] = (loads + blocks)[len(loads) + j - stages]
            acc = d if (mutant == "acc_carry" and d is not None) else np.zeros((bm, bn), F32)
            for rr, cc, j in read:
                acc = acc + a[rr, 64 * j:64 * j + 64] @ w[cc, 64 * j:64 * j + 64].T
            out[r, c] = d = acc
            loads += blocks
    return out[:m]


def emulate_gemm(a, w, bias, resid, epi, mutant=None, groups=None, bm=256, bn=256, stages=4):
    """gemm_tc.cu in numpy; groups: run its persistent tile schedule (``_scheduled_product``) over that many groups
    of (bm x bn) tiles with a ``stages``-slot ring, instead of one product."""
    a, w = a.astype(F32), w.astype(F32)
    if mutant == "drop_last_k16":
        a, w = a[:, :-16], w[:, :-16]
    prod = a @ w.T if groups is None else _scheduled_product(a, w, groups, bm, bn, stages, mutant)
    x = prod + (np.roll(bias, -1) if mutant == "bias_shift" else bias).astype(F32)
    if epi == 1:
        x = _gelu_tanh_f32(x) if mutant == "tanh_gelu" else _gelu_erf_f32(x)
    if epi == 2:
        x = x + resid.astype(F32)
    return _rtz_bf16(x) if mutant == "rtz_store" else round_to_bf16(x)


GEMM_CASES = {   # name: (m, n, k, epi, spread, big_resid)
    "bias": (256, 384, 768, 0, False, False),
    "gelu": (257, 384, 4096, 1, False, False),
    "gelu_spread": (129, 384, 64, 1, True, False),
    "resid": (255, 256, 768, 2, False, False),
    "resid_large": (127, 384, 192, 2, False, True),
}


def _gemm(case, mutant=None):
    m, n, k, epi, spread, big = GEMM_CASES[case]
    a, w, bias, resid = BD.gemm_inputs(m, n, k, seed=m + n + k, spread=spread, big_resid=big)
    ref, bound = BD.gemm_reference(a, w, bias, resid, epi)
    return BD.ratio(emulate_gemm(a, w, bias, resid, epi, mutant), ref, bound)


@pytest.mark.parametrize("case", sorted(GEMM_CASES))
def test_gemm_emulation_within_bound(case):
    assert _gemm(case) <= 1.0


@pytest.mark.parametrize("mutant,case", [("tanh_gelu", "gelu_spread"), ("bias_shift", "bias"), ("bias_shift", "resid"),
                                         ("drop_last_k16", "bias"), ("drop_last_k16", "gelu"),
                                         ("rtz_store", "bias"), ("rtz_store", "resid_large")])
def test_gemm_mutant_fails_bound(mutant, case):
    assert _gemm(case, mutant) > 1.0


SCHEDULE_CASES = {   # name: (m, n, k, epi, cta_group, sm_count); every group takes 3 tiles plus a partial last round
    "pair_bn256": (1263, 512, 320, 0, 2, 6),      # 10 tiles over 3 groups, 5 k-blocks in a 4-slot ring
    "single_bn128": (1115, 384, 448, 1, 1, 8),    # 27 tiles over 8 groups, 7 k-blocks in a 6-slot ring
    "pair_resid": (1436, 768, 1088, 2, 2, 10),    # 18 tiles over 5 groups, 17 k-blocks in a 4-slot ring
}


def _scheduled_gemm(case, mutant=None):
    m, n, k, epi, g, sm = SCHEDULE_CASES[case]
    bn, stages, tiles, groups, kb = BD.gemm_schedule(m, n, k, g, sm)
    assert tiles // groups >= 3 and 0 < tiles % groups and kb % stages
    a, w, bias, resid = BD.gemm_inputs(m, n, k, seed=m + n + k)
    ref, bound = BD.gemm_reference(a, w, bias, resid, epi)
    return BD.ratio(emulate_gemm(a, w, bias, resid, epi, mutant, groups, 128 * g, bn, stages), ref, bound)


@pytest.mark.parametrize("case", sorted(SCHEDULE_CASES))
def test_scheduled_gemm_emulation_within_bound(case):
    assert _scheduled_gemm(case) <= 1.0


@pytest.mark.parametrize("mutant", ["acc_carry", "stale_kblock"])
@pytest.mark.parametrize("case", sorted(SCHEDULE_CASES))
def test_scheduled_gemm_mutant_fails_bound(mutant, case):
    assert _scheduled_gemm(case, mutant) > 1.0


# -------------------------------------------------------------------------------------------------- attention
def emulate_attention(qkv, cu, heads, hidden, head_dim=64, mutant=None):
    """attn_tc.cu in numpy: 128-key blocks, fp32 logits in log2 units, running max with rescale, P rounded to bf16
    for P V, normaliser from the unrounded P, bf16 output."""
    x = np.concatenate([qkv.astype(F32), np.zeros((512, qkv.shape[1]), F32)])   # the packed buffer's padding rows
    scale = 1.0 / np.sqrt(64 if mutant == "scale_for_dim64" else head_dim)
    sc = F32(np.log2(np.e) * scale)
    out = np.zeros((qkv.shape[0], hidden), F32)
    for s in range(len(cu) - 1):
        t0, n = int(cu[s]), int(cu[s + 1] - cu[s])
        lim = n + {"mask_plus1": 1, "mask_minus1": -1}.get(mutant, 0)
        for h in range(heads):
            c = slice(h * head_dim, (h + 1) * head_dim)
            q = x[t0:t0 + n, c]
            m = np.full(n, -np.inf, F32)
            l = np.zeros(n, F32)
            o = np.zeros((n, head_dim), F32)
            for j in range((n + 127) // 128):
                k = x[t0 + 128 * j:t0 + 128 * (j + 1), hidden:][:, c]
                v = x[t0 + 128 * j:t0 + 128 * (j + 1), 2 * hidden:][:, c]
                sv = (q @ k.T) * sc
                sv[:, np.arange(128 * j, 128 * (j + 1)) >= lim] = -np.inf
                m_new = np.maximum(m, sv.max(axis=1))
                alpha = np.ones(n, F32) if mutant == "no_rescale" else np.exp2(m - m_new)
                m = m_new
                p = np.exp2(sv - m[:, None])
                l = l * alpha + p.sum(axis=1, dtype=F32)
                o = o * alpha[:, None] + round_to_bf16(p) @ v
            out[t0:t0 + n, c] = round_to_bf16(o / l[:, None])
    return out


ATTN_CASES = {   # name: (heads, lens, kind, head_dim)
    "ragged": (2, [129, 1, 64], "random", 64),
    "blocks": (1, [127, 256, 257], "random", 64),
    "lastmax": (2, [129, 255, 2], "lastmax", 64),
    "leak": (2, [129, 300, 128, 40], "leak", 64),
    "onehot": (2, [385, 128], "onehot", 64),
    "dim32": (4, [129, 33], "random", 32),
}


def _attn(case, mutant=None):
    heads, lens, kind, dh = ATTN_CASES[case]
    qkv, cu = BD.attention_inputs(heads, lens, seed=sum(lens) + heads, kind=kind, head_dim=dh)
    ref, bound = BD.attention_reference(qkv, cu, heads, heads * dh, dh)
    return BD.ratio(emulate_attention(qkv, cu, heads, heads * dh, dh, mutant), ref, bound)


@pytest.mark.parametrize("case", sorted(ATTN_CASES))
def test_attention_emulation_within_bound(case):
    assert _attn(case) <= 1.0


@pytest.mark.parametrize("mutant,case", [("mask_plus1", "leak"), ("mask_minus1", "lastmax"), ("mask_minus1", "ragged"),
                                         ("no_rescale", "blocks"), ("no_rescale", "ragged"),
                                         ("scale_for_dim64", "dim32")])
def test_attention_mutant_fails_bound(mutant, case):
    assert _attn(case, mutant) > 1.0


# ------------------------------------------------------------------------------------------- similarity scores
def emulate_sim(Q, C, mutant=None):
    """simtopk_tc.cu's debug tile: fp32 dot of bf16 rows times the fp32 inverse norm of row_inv_norm_kernel."""
    Q, C = Q.astype(F32), C.astype(F32)
    inv = np.sqrt((C * C).sum(axis=1, dtype=F32))
    inv = np.divide(F32(1), inv, out=np.zeros_like(inv), where=inv > 0)
    Cm = C.copy()
    if mutant == "neighbour_norm":
        inv = np.roll(inv, -1)
    if mutant == "skip_kblock":
        Cm[:, 64:128 if C.shape[1] > 64 else 64] = 0
        if C.shape[1] == 64:
            Cm[:] = 0
    if mutant == "unswizzled":   # 16-byte chunk c of row r read from chunk c ^ (r & 7) of every 128-byte k-block
        chunks = Cm.reshape(C.shape[0], -1, 8, 8)
        perm = np.arange(8)[None, :] ^ (np.arange(C.shape[0]) % 8)[:, None]
        Cm = np.take_along_axis(chunks, perm[:, None, :, None], axis=2).reshape(C.shape)
    return (Q @ Cm.T) * inv[None, :]


SIM_DIMS = [64, 128, 192, 576, 768, 1024]


def _sim(dim, mutant=None):
    rng = np.random.default_rng(dim)
    Q = round_to_bf16(rng.standard_normal((16, dim)).astype(F32))
    C = round_to_bf16(rng.standard_normal((150, dim)).astype(F32))
    C[5] = 0.0
    ref, bound = BD.sim_reference(Q, C)
    return BD.ratio(emulate_sim(Q, C, mutant), ref, bound)


@pytest.mark.parametrize("dim", SIM_DIMS)
def test_sim_emulation_within_bound(dim):
    assert _sim(dim) <= 1.0


@pytest.mark.parametrize("mutant", ["neighbour_norm", "skip_kblock", "unswizzled"])
@pytest.mark.parametrize("dim", SIM_DIMS)
def test_sim_mutant_fails_bound(mutant, dim):
    assert _sim(dim, mutant) > 1.0


# ------------------------------------------------------------------------------------- encoder, one layer at a time
TF_CFG = B.BertConfig(hidden=128, layers=4, heads=2, inter=256, vocab=120, max_pos=512, pool="cls")
MUTANT_LAYER = 2


def _mutated_gelu(mutant):
    """B.gelu with one defect in the first sequence of at least 129 tokens: ``tile`` copies the 128 x 128 block of
    GELU outputs at (0, 0) from its neighbour at (0, 128); ``row`` gives the middle token the GELU row of the token
    before it."""
    gelu, done = B.gelu, []

    def g(x):
        y = gelu(x)
        if not done and len(y) > 128:
            if mutant == "tile":
                y[:128, :128] = y[:128, 128:256]
            else:
                y[len(y) // 2] = y[len(y) // 2 - 1]
            done.append(True)
        return y
    return g


def _teacher_forced_worst(monkeypatch=None, mutant=None):
    """Worst bf16 ulps (BD.bf16_ulps) per layer of the fp32 bf16-store emulation of the encoder, each layer checked
    against the fp64 bf16-store oracle of that layer run on the emulation's own output of the layer before (the
    first layer on the oracle's own embedding)."""
    w = B.init_weights(TF_CFG, seed=7, bf16=True)
    tok, cu = B.synth_batch(TF_CFG, 6, 29, mean_len=200, std_len=120, min_len=1, max_len=512)
    x32 = B.embed_tokens(TF_CFG, w, tok, cu, F32, bf16_stores=True)
    x_in = B.embed_tokens(TF_CFG, w, tok, cu, bf16_stores=True)
    worst = []
    for l in range(TF_CFG.layers):
        ref = B.encoder_layer(TF_CFG, w, l, x_in, cu, bf16_stores=True)
        if mutant and l == MUTANT_LAYER:
            monkeypatch.setattr(B, "gelu", _mutated_gelu(mutant))
        x32 = B.encoder_layer(TF_CFG, w, l, x32, cu, F32, bf16_stores=True)
        if mutant and l == MUTANT_LAYER:
            monkeypatch.undo()
        worst.append(float(BD.bf16_ulps(x32, ref).max()))
        x_in = x32
    print(f"teacher-forced emulation, mutant {mutant}: worst ulps per layer {[round(e, 2) for e in worst]}")
    return worst


def test_teacher_forced_emulation_within_hidden_ulps():
    assert max(_teacher_forced_worst()) <= BD.HIDDEN_ULPS


@pytest.mark.parametrize("mutant", ["tile", "row"])
def test_teacher_forced_mutant_fails_hidden_ulps(mutant, monkeypatch):
    worst = _teacher_forced_worst(monkeypatch, mutant)
    assert worst[MUTANT_LAYER] > BD.HIDDEN_ULPS


def test_bf16_helpers_round_to_nearest_and_toward_zero():
    x = np.array([1.0 + 2 ** -8 + 2 ** -10, -(1.0 + 2 ** -8 + 2 ** -10)], F32)
    assert round_to_bf16(x).tolist() == [1.0 + 2 ** -7, -(1.0 + 2 ** -7)]
    assert _rtz_bf16(x).tolist() == [1.0, -1.0]
    assert f32_to_bf16_bits(np.array([1.0], F32))[0] == 0x3F80


# --------------------------------------------------------------------------------- int8 first pass (tensor cores)
def emulate_int8_first_pass(q_bits, R, mutant=None):
    """simtopk_tc.cu's int8 first pass as the kernel computes it: the query image of query_image_i8_kernel (fp32 amax,
    fp64 product and division, rint), int32 MMAs over hi and lo, fmaf(acc_hi, 256, acc_lo) in fp32, times the row's
    fp32 inverse norm.  Mutants: drop_lo (acc_lo never added); logical_hi (hi taken from a logical shift of the 16-bit
    image, i.e. read as the unsigned byte, so a negative q16 gets hi + 256)."""
    q = bf16_bits_to_f32(q_bits).astype(np.float64)
    amax = np.abs(q).max(axis=1, initial=0.0)
    v = np.where(amax[:, None] > 0, np.rint(q * 32512.0 / np.where(amax > 0, amax, 1.0)[:, None]), 0).astype(np.int64)
    hi = (v + 128) >> 8
    lo = v - 256 * hi
    if mutant == "logical_hi":
        hi = ((v + 128) & 0xFFFF) >> 8
    R = np.asarray(R, np.int64)
    acc_hi, acc_lo = (hi @ R.T).astype(F32), (lo @ R.T).astype(F32)
    if mutant == "drop_lo":
        acc_lo = np.zeros_like(acc_lo)
    s = (acc_hi.astype(np.float64) * 256 + acc_lo.astype(np.float64)).astype(F32)   # fmaf: one rounding
    ss = (R * R).sum(axis=1).astype(F32)
    inv = np.divide(F32(1), np.sqrt(ss), out=np.zeros_like(ss), where=ss > 0)
    return s * inv[None, :]


def _int8_case(dim):
    from aurora_b200.engine import to_bf16_bits
    from oracle.quantize import quantize_rows

    rng = np.random.default_rng(dim)
    Q = rng.standard_normal((6, dim))
    Q[1] = 0.0
    Q[2, 3] = 40.0
    C = rng.standard_normal((90, dim))
    C[4] = 0.0
    R, _ = quantize_rows(to_bf16_bits(C.astype(F32)))
    return to_bf16_bits(Q.astype(F32)), R


@pytest.mark.parametrize("dim", [128, 384, 1024])
def test_int8_emulation_matches_the_exact_reference_and_the_cosine_bound(dim):
    q_bits, R = _int8_case(dim)
    got = emulate_int8_first_pass(q_bits, R)
    assert np.array_equal(got, BD.int8_tc_reference(q_bits, R))
    ref, bound, scale = BD.int8_cosine_reference(q_bits, R)
    assert BD.ratio(got * scale[:, None], ref, bound) <= 1.0


@pytest.mark.parametrize("mutant", ["drop_lo", "logical_hi"])
@pytest.mark.parametrize("dim", [128, 384, 1024])
def test_int8_mutant_fails_the_exact_reference_and_the_cosine_bound(mutant, dim):
    q_bits, R = _int8_case(dim)
    got = emulate_int8_first_pass(q_bits, R, mutant)
    assert not np.array_equal(got, BD.int8_tc_reference(q_bits, R))
    ref, bound, scale = BD.int8_cosine_reference(q_bits, R)
    assert BD.ratio(got * scale[:, None], ref, bound) > 1.0


# ---------------------------------------------------------------------------------------------- list kernel
def emulate_list_scores(Q, C, lists, q_list, mutant=None):
    """list_scores_kernel as a dense [nq, n] matrix (NaN where a query's list does not reach): the queries of a list in
    groups of up to 64 (stable order), each row scored over ceil(dim / 64) zero-filled 64-dim chunks accumulated in fp32
    (a chunk's products summed exactly: a model of the MMA), times the row's fp32 inverse norm.  Mutants: drop_last_chunk
    (dim // 64 chunks); shifted_partial_group (the queries of a group's last, partial 16-row block read the query one row
    further on, zeros past the group); neighbour_norm (a row takes the inverse norm of the next row of its list)."""
    Q, C = Q.astype(F32), C.astype(F32)
    nq, dim = Q.shape
    inv = np.sqrt((C * C).sum(axis=1, dtype=F32))
    inv = np.divide(F32(1), inv, out=np.zeros_like(inv), where=inv > 0)
    n_kc = dim // 64 if mutant == "drop_last_chunk" else -(-dim // 64)
    out = np.full((nq, C.shape[0]), np.nan)
    order = np.argsort(q_list, kind="stable")
    for l, rows in enumerate(lists):
        rows = np.unique(rows)
        qs = order[q_list[order] == l]
        for g0 in range(0, len(qs), 64):
            grp = qs[g0:g0 + 64]
            Qg = Q[grp].copy()
            full = len(grp) // 16 * 16
            if mutant == "shifted_partial_group" and full < len(grp):
                Qg[full:] = np.concatenate([Q[grp[full + 1:]], np.zeros((1, dim), F32)])
            acc = np.zeros((len(grp), len(rows)), F32)
            for kc in range(n_kc):
                k = slice(kc * 64, min(dim, kc * 64 + 64))
                acc = acc + (Qg[:, k].astype(np.float64) @ C[rows, k].T.astype(np.float64)).astype(F32)
            nv = inv[np.roll(rows, -1)] if mutant == "neighbour_norm" else inv[rows]
            out[np.ix_(grp, rows)] = acc * nv[None, :]
    return out


def _list_case(dim):
    rng = np.random.default_rng(dim)
    C = round_to_bf16(rng.standard_normal((300, dim)).astype(F32))
    lists = [rng.choice(300, size=s, replace=False) for s in (65, 130, 7)]
    q_list = rng.permutation(np.repeat(np.arange(3), [17, 70, 1])).astype(np.int32)
    Q = round_to_bf16(rng.standard_normal((len(q_list), dim)).astype(F32))
    return Q, C, lists, q_list


@pytest.mark.parametrize("dim", [72, 200, 1536])
def test_list_emulation_within_bound(dim):
    Q, C, lists, q_list = _list_case(dim)
    got = emulate_list_scores(Q, C, lists, q_list)
    ref, bound = BD.sim_reference(Q, C)
    m = np.isfinite(got)
    assert m.sum() == sum(len(lists[l]) for l in q_list)
    assert BD.ratio(got[m], ref[m], bound[m]) <= 1.0


@pytest.mark.parametrize("mutant", ["drop_last_chunk", "shifted_partial_group", "neighbour_norm"])
@pytest.mark.parametrize("dim", [72, 200])
def test_list_mutant_fails_bound(mutant, dim):
    Q, C, lists, q_list = _list_case(dim)
    got = emulate_list_scores(Q, C, lists, q_list, mutant)
    ref, bound = BD.sim_reference(Q, C)
    m = np.isfinite(got)
    assert BD.ratio(got[m], ref[m], bound[m]) > 1.0


def test_f32_reference_covers_rounded_products():
    """sim_reference_f32 admits a dot product whose fp32 products each round before an fp32 sum."""
    rng = np.random.default_rng(3)
    Q = rng.standard_normal((8, 1025)).astype(F32)
    C = rng.standard_normal((40, 1025)).astype(F32)
    inv = F32(1) / np.sqrt((C * C).sum(axis=1, dtype=F32))
    got = np.stack([np.stack([np.add.reduce(q * c, dtype=F32) for c in C]) for q in Q]) * inv[None, :]
    ref, bound = BD.sim_reference_f32(Q, C)
    assert BD.ratio(got, ref, bound) <= 1.0

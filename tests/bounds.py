"""Per-element error bounds for the tensor-core kernels, derived from the arithmetic each kernel does.

Every bound is a function of the fp64 reference and the inputs, element by element, so a bug that moves a typical
element by a few per cent cannot hide under the largest element's tolerance.  Notation: u = 2^-24 is the fp32 unit
roundoff.  A bf16 store rounds to nearest and adds at most half an ulp, 2^-8 |x| (just above a power of two), so
outputs whose error is all store rounding come close to max(err / bound) = 1 by design.  Products of
two bf16 values are exact in fp32, so in a dot product only the additions round: K additions add at most K u sum|a b|
whatever the order the tensor core uses.

The CPU tests (tests/test_bounds.py) run numpy emulations of the kernels against these bounds, and deliberately broken
emulations (mutants) that each must fail them; the GPU tests hold the real kernels to the same bounds and print
max(err / bound).
"""

from __future__ import annotations

import numpy as np

from oracle import bert_encoder as B
from oracle import quantize as QZ
from oracle.cosine_topk import round_to_bf16

U = 2.0 ** -24
ERF_AS = 1.5e-7          # |error| of the Abramowitz-Stegun 7.1.26 erf approximation in gelu_erf
GELU_SLOPE = 1.13        # max |d gelu / dx|: an input error reaches the output at most this much larger


def _f64(x):
    return np.asarray(x, dtype=np.float64)


def _bf16(x):
    return round_to_bf16(np.asarray(x, dtype=np.float32))


def ratio(got, ref, bound) -> float:
    """max(|got - ref| / bound) over all elements (inf where got is not finite; a zero bound demands an exact 0)."""
    got, ref = _f64(got), _f64(ref)
    err = np.where(np.isfinite(got), np.abs(got - ref), np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.max(r)) if r.size else 0.0


def assert_within(tag: str, got, ref, bound) -> float:
    r = ratio(got, ref, bound)
    print(f"{tag}: max(err / bound) = {r:.4f}")
    if r > 1.0:
        got, ref = _f64(got), _f64(ref)
        worst = np.unravel_index(np.argmax(np.abs(got - ref) / bound), ref.shape)
        raise AssertionError(f"{tag}: max(err / bound) = {r:.4f} at {worst}: got {got[worst]!r} want {ref[worst]!r} "
                             f"bound {bound[worst]!r}")
    return r


# ------------------------------------------------------------------------------------------- similarity scores
def sim_reference(Q, C):
    """The similarity kernel's debug tile: dot(q, c) * inv_norm_f32(c) (not divided by |q|).  Returns (ref, bound).

    bound = K u (|q| . |c|) / |c|  +  (K / 2 + 4) u |ref|; the second term covers the fp32 inverse norm of
    row_inv_norm_kernel (a K-term sum of squares, a square root and a division)."""
    Q, C = _f64(Q), _f64(C)
    K = Q.shape[1]
    cn = np.sqrt(np.einsum("ij,ij->i", C, C))
    inv = np.divide(1.0, cn, out=np.zeros_like(cn), where=cn > 0)
    ref = (Q @ C.T) * inv[None, :]
    bound = K * U * (np.abs(Q) @ np.abs(C).T) * inv[None, :] + (K / 2 + 4) * U * np.abs(ref)
    return ref, bound


def sim_reference_f32(Q, C):
    """sim_reference for fp32 queries and rows (the generic kernel over an f32 shard).  Returns (ref, bound).

    A product of two fp32 values is no longer exact in fp32.  simt_scores_kernel folds each product into its running sum
    with one fmaf, one rounding per step, which the K u (|q| . |c|) term already covers; an evaluation that rounds the
    product on its own first adds at most u |q_k c_k| per term.  So bound = sim_reference's bound + u (|q| . |c|) / |c|.
    The inverse norm's sum of squares rounds the same way, inside its (K / 2 + 4) u |ref| term."""
    Q, C = _f64(Q), _f64(C)
    ref, bound = sim_reference(Q, C)
    cn = np.sqrt(np.einsum("ij,ij->i", C, C))
    inv = np.divide(1.0, cn, out=np.zeros_like(cn), where=cn > 0)
    return ref, bound + U * (np.abs(Q) @ np.abs(C).T) * inv[None, :]


def int8_inv_norm(R):
    """The fp32 inverse norm of int8 rows as the ingest kernel computes it, bit for bit: the sum of squares is an integer
    below 2^24 (dim <= 1024), exact in fp32 in any order, and sqrtf and the division round once each; 0 for a zero row."""
    ss = (np.asarray(R, np.int64) ** 2).sum(axis=1).astype(np.float32)
    return np.divide(np.float32(1), np.sqrt(ss), out=np.zeros_like(ss), where=ss > 0)


def int8_tc_reference(q_bits, R):
    """The tensor-core kernel's int8 first pass, exactly (float32 [nq, n]).  q16 = 256 hi + lo is the query image
    (oracle/quantize.py:query_image); acc_hi = hi . c and acc_lo = lo . c are exact int32 sums (|acc| < 2^24); the kernel
    forms fmaf(acc_hi, 256, acc_lo) from their exact fp32 conversions, one rounding of 256 acc_hi + acc_lo, and scales it
    by the row's fp32 inverse norm (int8_inv_norm) with one more rounding.  The dump must equal this bit for bit."""
    _, hi, lo = QZ.query_image(q_bits)
    R = np.asarray(R, np.int64)
    acc = 256 * (hi @ R.T) + lo @ R.T
    return acc.astype(np.float32) * int8_inv_norm(R)[None, :]


def int8_cosine_reference(q_bits, R):
    """What the int8 first pass approximates: (ref, bound, scale).  score * scale[:, None] (scale = amax_q / 32512, the
    query image's step) against ref = q . c / |c| in fp64 over the stored int8 rows c.

    The image rounds each query element to the nearest multiple of amax_q / 32512, so it moves q_k by at most
    amax_q / 65024 (the per-dimension bound of the int8 design), and the score by at most amax_q / 65024 . |c| / |c|.  The
    kernel's fp32 work is two roundings of the combination and the final product plus the inverse norm's (sqrtf and a
    division of an exact sum): 4 u of (|q| + amax_q / 65024) . |c| / |c|."""
    q = QZ.bf16_bits_to_f64(np.atleast_2d(q_bits))
    R = _f64(R)
    cn = np.sqrt(np.einsum("ij,ij->i", R, R))
    inv = np.divide(1.0, cn, out=np.zeros_like(cn), where=cn > 0)
    step = np.abs(q).max(axis=1, initial=0.0)[:, None] / 65024
    ref = (q @ R.T) * inv[None, :]
    absc = np.abs(R).T * inv[None, :]
    bound = step * absc.sum(axis=0)[None, :] + 4 * U * ((np.abs(q) + step) @ absc)
    return ref, bound, 2 * step[:, 0]


# ------------------------------------------------------------------------------------------------------ GEMM
def gemm_reference(A, W, bias, resid=None, epi: int = 0):
    """out = epi(A . W^T + bias) (+ resid) in fp64; epi 0 = bias, 1 = bias + erf-GELU, 2 = bias + residual.
    Returns (ref, bound).

    bound = 2^-8 |ref| + 1.13 (K + 2) u (|A| . |W|^T + |bias|) + u |resid|  (+ 1.5e-7 |x| / 2 for GELU, x = its input)."""
    A, W, bias = _f64(A), _f64(W), _f64(bias)
    K = A.shape[1]
    pre = A @ W.T + bias[None, :]
    ref = pre
    bound = GELU_SLOPE * (K + 2) * U * (np.abs(A) @ np.abs(W).T + np.abs(bias)[None, :])
    if epi == 1:
        ref = B.gelu(pre)
        bound = bound + ERF_AS * np.abs(pre) / 2
    if epi == 2:
        ref = pre + _f64(resid)
        bound = bound + U * np.abs(_f64(resid))
    return ref, bound + 2.0 ** -8 * np.abs(ref)


def gemm_schedule(m: int, n: int, k: int, cta_group: int, sm_count: int):
    """gemm_tc.cu's persistent schedule for an aur_debug_gemm call: (bn, stages, tiles, groups, k_blocks).  The N tile
    is 256 when it divides n, else 128 (aur_debug_gemm); the TMA ring has GemmSmem::kStages slots of one 64-wide
    k-block each; tiles are (128 cta_group) x bn; launch_one starts min(tiles, sm_count / cta_group) groups of
    cta_group CTAs, and group g takes tiles g, g + groups, ..."""
    bn = 256 if n % 256 == 0 else 128
    stages = min(8, (192 * 1024) // (128 * 64 * 2 + bn * 64 * 2))
    tiles = -(-m // (128 * cta_group)) * (n // bn)
    return bn, stages, tiles, min(tiles, sm_count // cta_group), k // 64


# ------------------------------------------------------------------------------------------ encoder hidden states
HIDDEN_ULPS = 8          # per-token hidden states, one layer against the bf16-store oracle


def bf16_ulps(got, ref, floor=None):
    """|got - ref| in bf16 ulps (2^(floor(log2 s) - 7)) of s = max(|ref|, floor); floor defaults to the RMS of the
    element's token row.  A LayerNorm output inherits the error of its input's bf16 stores, whose ulps are set by
    the row's magnitude, not by the element's, so small elements of an O(1) row are measured against the row."""
    got, ref = _f64(got), _f64(ref)
    if floor is None:
        floor = np.sqrt((ref * ref).mean(axis=1, keepdims=True))
    return np.abs(got - ref) / 2.0 ** (np.floor(np.log2(np.maximum(np.abs(ref), floor))) - 7)


# -------------------------------------------------------------------------------------------------- attention
def attention_reference(qkv, cu, heads: int, hidden: int, head_dim: int = 64):
    """Softmax(q k^T / sqrt(head_dim)) v per packed sequence and head, fp64.  Returns (ref, bound) [tokens, hidden].

    bound = 2^-8 |ref| + (2^-8 + 2 max_j |ds_ij| + 2^-21) (P |V|)_id, ds_ij = 64 u (|q_i| . |k_j|) scale the fp32
    error of a logit (K = 64: the MMA's depth, also for a zero-padded head dim 32).  The 2^-8 inside the bracket covers
    P rounded to bf16 before the P V MMA (the normaliser sums the unrounded P); 2^-21 the exp2 / reciprocal
    approximations."""
    qkv = _f64(qkv)
    scale = 1.0 / np.sqrt(head_dim)
    ref = np.zeros((qkv.shape[0], hidden))
    bound = np.zeros_like(ref)
    for s in range(len(cu) - 1):
        x = qkv[cu[s]:cu[s + 1]]
        for h in range(heads):
            c = slice(h * head_dim, (h + 1) * head_dim)
            q, k, v = x[:, c], x[:, hidden:][:, c], x[:, 2 * hidden:][:, c]
            a = q @ k.T * scale
            p = np.exp(a - a.max(axis=1, keepdims=True))
            p /= p.sum(axis=1, keepdims=True)
            ds = 64 * U * (np.abs(q) @ np.abs(k).T) * scale
            o = p @ v
            ref[cu[s]:cu[s + 1], c] = o
            bound[cu[s]:cu[s + 1], c] = (2.0 ** -8 * np.abs(o)
                                         + (2.0 ** -8 + 2 * ds.max(axis=1, keepdims=True) + 2.0 ** -21) * (p @ np.abs(v)))
    return ref, bound


# ---------------------------------------------------------------------------------- inputs shared by CPU and GPU
def gemm_inputs(m: int, n: int, k: int, seed: int, spread: bool = False, big_resid: bool = False,
                with_resid: bool = True):
    """bf16-valued A [m, k], W [n, k], resid [m, n] (None unless with_resid) and fp32 bias.  spread: a small product
    and a bias spanning [-6, 6], so GELU inputs reach both tails of the erf approximation; big_resid: a residual 2^10
    times the product."""
    rng = np.random.default_rng(seed)
    a = _bf16(rng.standard_normal((m, k)))
    w = _bf16(rng.standard_normal((n, k)) / np.sqrt(k) * (0.05 if spread else 1.0))
    bias = (rng.uniform(-6, 6, n) if spread else rng.standard_normal(n)).astype(np.float32)
    resid = _bf16(rng.standard_normal((m, n)) * (1024.0 if big_resid else 1.0)) if with_resid else None
    return a, w, bias, resid


def attention_inputs(heads: int, lens, seed: int, kind: str = "random", head_dim: int = 64):
    """Packed bf16-valued qkv [tokens, 3 hidden] and cu_seqlens.  kind: random (entries 1.5 N(0, 1)); onehot (large q
    and k: nearly one-hot rows, exp underflows); lastmax (every query's largest logit on its sequence's last key); leak
    (every other sequence's keys 8x larger, so a key leaking across the mask shows)."""
    rng = np.random.default_rng(seed)
    hidden = heads * head_dim
    cu = np.zeros(len(lens) + 1, dtype=np.int32)
    cu[1:] = np.cumsum(lens)
    x = rng.standard_normal((int(cu[-1]), 3 * hidden)) * 1.5
    if kind == "onehot":
        x[:, :2 * hidden] *= 4.0
    for s in range(len(lens)):
        a, b = int(cu[s]), int(cu[s + 1])
        if kind == "lastmax":
            d = rng.standard_normal(hidden)
            x[a:b, :hidden] = 0.3 * x[a:b, :hidden] + d
            x[b - 1, hidden:2 * hidden] = 2.0 * d
        if kind == "leak" and s % 2 == 1:
            x[a:b, hidden:2 * hidden] *= 8.0
    return _bf16(x), cu


# ------------------------------------------------------------------------- similarity kernel debug tiles
def tc_debug_tile(cta: int, nq: int):
    """(query block, corpus tile) of the [64 queries x 64 rows] score tile CTA ``cta`` returns from
    Index.debug_tc_scores (the first tile of its tile set).  run_tc_block: up to 64 queries make one query block (a
    pair request then runs as single CTAs), so every CTA is its own tile set; 65 to 128 queries make two, and CTA c
    takes query block c % 2 (its rank in a pair, or every other single CTA) and tile set c // 2."""
    n_qblocks = 1 if nq <= 64 else 2
    return cta % n_qblocks, cta // n_qblocks


def tc_debug_rows(cta: int, nq: int, tile_n: int):
    """(query block, corpus rows) of CTA ``cta``'s [64 queries x tile_n rows] tile from Index.debug_tc_tile, tile_n = 64
    or 128 as the call reports: tile set t starts at tile t whatever the width, rows t tile_n .. t tile_n + tile_n - 1."""
    qb, tile = tc_debug_tile(cta, nq)
    return qb, tile * tile_n + np.arange(tile_n)

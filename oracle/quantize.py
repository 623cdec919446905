"""The int8 row format (AUR_I8) restated in numpy: what a shard stores for a bf16 row.

A row of bf16 values x with amax = max |x| (exact) is stored as q = rint(x * 127 / amax): the product is exact in fp64
and the quotient one correctly rounded fp64 division, rint rounds half to even, so |q| <= 127 and a non-zero row has an
element equal to +-127.  An all-zero row stays zero.  A row holding a NaN or +-inf is stored as zeros and is never
returned by a search (``finite`` False).  Re-quantizing a stored row converted to bf16 gives the same bytes back.
"""

from __future__ import annotations

import numpy as np


def bf16_bits_to_f64(bits: np.ndarray) -> np.ndarray:
    """bf16 bit patterns (uint16) -> exact float64 values."""
    u = np.ascontiguousarray(bits, dtype=np.uint16).astype(np.uint32) << np.uint32(16)
    return u.view(np.float32).astype(np.float64)


def quantize_rows(bits: np.ndarray):
    """bf16 rows [n, dim] (uint16 bits) -> (int8 rows [n, dim], finite [n] bool)."""
    x = bf16_bits_to_f64(np.atleast_2d(bits))
    finite = np.isfinite(x).all(axis=1)
    x = np.where(finite[:, None], x, 0.0)
    amax = np.abs(x).max(axis=1, initial=0.0)
    safe = np.where(amax > 0.0, amax, 1.0)
    q = np.rint((x * 127.0) / safe[:, None])
    return q.astype(np.int8), finite


def int8_to_bf16_bits(q: np.ndarray) -> np.ndarray:
    """int8 values -> bf16 bit patterns (every int8 value is exact in bf16)."""
    f = np.ascontiguousarray(q, dtype=np.float32)
    return (f.view(np.uint32) >> np.uint32(16)).astype(np.uint16)


def query_image(bits: np.ndarray):
    """bf16 queries [nq, dim] (uint16 bits) -> (q16, hi, lo) int64 [nq, dim]: the tensor-core kernel's 16-bit query image
    of an int8 shard (query_image_i8_kernel).  q16 = rint(q * 32512 / amax_q): the product is exact in fp64 and the
    quotient one correctly rounded division, half to even; a zero query stays zero.  Split exactly as q16 = 256 hi + lo
    with hi = (q16 + 128) >> 8, an arithmetic shift (floor), so hi in [-127, 127] and lo in [-128, 127], both int8."""
    x = bf16_bits_to_f64(np.atleast_2d(bits))
    amax = np.abs(x).max(axis=1, initial=0.0)
    ok = (amax > 0.0) & np.isfinite(amax)
    safe = np.where(ok, amax, 1.0)
    q16 = np.where(ok[:, None], np.rint((x * 32512.0) / safe[:, None]), 0.0).astype(np.int64)
    hi = (q16 + 128) >> 8
    return q16, hi, q16 - 256 * hi

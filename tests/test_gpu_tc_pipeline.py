"""The similarity kernel's MMA issue at the shapes where a TMA-ring or accumulator hand-off bug would hide: one k-block per
tile (dim 64), a 2-stage ring (dim 1024 at large k), k-block counts that are not a multiple of the stage count, many
tiles per CTA, and CTAs with an odd and an even number of tiles in the same launch.  Every search is held to the fp64
oracle, and the one-CTA and two-CTA-cluster kernels must return the same ids and scores."""

from __future__ import annotations

import numpy as np
import pytest

from aurora_b200 import _native as N
from aurora_b200.engine import Index
from oracle import cosine_topk as O
from tests.gpu_exact import check_exact, dev_search

pytestmark = pytest.mark.gpu

SMEM_OPTIN = 227 * 1024   # sm_90 opt-in shared memory per block
KSLACK, QROWS, TILE_N, MAX_STAGES = 8, 64, 64, 12   # kSlack, kTcQRows, kTcTileN, kTcMaxStages (csrc/internal.h)


def tc_stages(dim: int, ksel: int) -> int:
    """tc_pick_stages (csrc/simtopk_tc.cu): the deepest TMA ring make_layout fits into the opt-in shared memory."""
    fifo = 16 * QROWS * 20 if ksel <= 64 else 0
    rest = ((dim // 64) * QROWS * 128 + QROWS * (TILE_N + 4) * 4 + ksel * QROWS * 8
            + 2 * 2 * 2 * TILE_N * 4 + fifo + QROWS * 4 + (2 * MAX_STAGES + 5) * 8 + 16 + 1024)
    for s in range(MAX_STAGES, 1, -1):
        if TILE_N * 128 * s + rest <= SMEM_OPTIN:
            return s
    return 0


def tile_sets(kernel: int, nq: int, ksel: int, sm_count: int) -> int:
    """run_tc_block's (csrc/capi.cu) tile-set count: CTAs (or pairs) that walk disjoint sets of corpus tiles."""
    if kernel == N.KERNEL_TC2 and nq > QROWS:
        pairs = sm_count // 2
        n_super = -(-nq // (2 * QROWS))
        while n_super > 1 and -(-ksel // (pairs // n_super)) > 4:
            n_super -= 1
        return pairs // n_super
    return (sm_count & ~1) // (1 if nq <= QROWS else 2)


def _sm_count() -> int:
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


def _data(n, d, nq, seed):
    rng = np.random.default_rng(seed)
    C = rng.standard_normal((n, d)).astype(np.float32)
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    for i in range(nq):   # a few close rows per query, spread over the tiles
        for r in rng.choice(n, 3, replace=False):
            C[r] = Q[i] + 0.3 * rng.standard_normal(d).astype(np.float32)
    return O.round_to_bf16(C), O.round_to_bf16(Q)


def _run_both(C, Q, k):
    n, d = C.shape
    want = O.cosine_topk(Q, C, k, return_f64=True)
    got = {}
    with Index(d, n) as ix:
        ix.add(C, np.arange(n, dtype=np.int64))
        for kern in (N.KERNEL_TC1, N.KERNEL_TC2):
            ix.set_kernel(kern)
            got[kern] = dev_search(ix, Q, k)
            assert ix.stats()["last_kernel"] == kern
            check_exact(got[kern], Q, C, k, want=want)
    for a, b in zip(got[N.KERNEL_TC1], got[N.KERNEL_TC2]):
        assert np.array_equal(a, b), "TC1 and TC2 differ"


# (kernel whose geometry sets the corpus size, dim, nq, k, tiles per CTA or pair); the corpus holds
# tile_sets * tiles + tile_sets // 2 tiles, so half the CTAs take one tile more than the other half
@pytest.mark.parametrize("kernel,d,nq,k,tiles", [
    (N.KERNEL_TC1, 64, 1, 10, 3),       # one k-block per tile: every deferred stage release crosses a tile
    (N.KERNEL_TC2, 64, 256, 32, 4),
    (N.KERNEL_TC2, 576, 256, 32, 9),    # 9 k-blocks: not a multiple of the ring depth
    (N.KERNEL_TC2, 768, 256, 32, 12),   # cfg2's shape
])
def test_tile_counts_and_k_blocks(kernel, d, nq, k, tiles):
    ts = tile_sets(kernel, nq, k + KSLACK, _sm_count())
    n = (ts * tiles + ts // 2) * TILE_N
    C, Q = _data(n, d, nq, seed=d + nq + tiles)
    _run_both(C, Q, k)


@pytest.mark.parametrize("kernel,nq", [(N.KERNEL_TC1, 64), (N.KERNEL_TC2, 256)])
def test_two_stage_ring_at_dim_1024(kernel, nq):
    d = 1024
    k = next(k for k in range(32, 128) if tc_stages(d, k + KSLACK) == 2)
    assert tc_stages(d, k - 1 + KSLACK) == 3
    ts = tile_sets(kernel, nq, k + KSLACK, _sm_count())
    n = (ts * 10 + ts // 2) * TILE_N
    C, Q = _data(n, d, nq, seed=nq + k)
    _run_both(C, Q, k)


def test_epi_groups_option_is_rejected():
    """The kernel has one epilogue group: "epi_groups" is not an option."""
    with Index(64, 64) as ix:
        assert ix._lib.aur_set_option(ix._h, b"epi_groups", 2) == N.AUR_ERR_INVALID

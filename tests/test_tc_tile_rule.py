"""The similarity kernel's tile-width rule, mirrored from the host (tc_auto_tile in csrc/capi.cu, make_layout in
csrc/simtopk_tc.cu): a launch takes 128-row corpus tiles when the 128-row shared-memory layout leaves at least four
16 KB ring stages, and 64-row tiles otherwise.  tests/test_gpu_tc_wide_tile.py checks the library against this mirror
through aur_stats.last_tile_n."""

from __future__ import annotations

import pytest

SMEM_OPTIN = 227 * 1024          # sm_90 opt-in shared memory per block
QROWS, MAX_STAGES, FIFO_RECS, FIFO_MAX_KSEL = 64, 12, 16, 64   # kTcQRows, kTcMaxStages, kTcFifoRecs, kTcFifoMaxKsel
NARROW, WIDE, WIDE_MIN_STAGES = 64, 128, 4                      # kTcTileN, kTcTileWide, kTcWideMinStages


def smem_bytes(dim: int, ksel: int, stages: int, tile: int, mask: bool) -> int:
    """tc_smem_bytes: make_layout's total plus the 1 KB alignment slack."""
    wide = tile == WIDE
    fifo = ((FIFO_RECS // 2 if wide else FIFO_RECS) if ksel <= FIFO_MAX_KSEL else 0) * QROWS * 20
    rows_buf = 2 * 2 * tile * 4                                  # inverse norms (and tenant masks): [2 warps][2][tile]
    return (tile * 128 * stages + (dim // 64) * QROWS * 128 + QROWS * (tile + 4) * 4
            + ksel * QROWS * 8 + rows_buf + (rows_buf if mask or not wide else 0) + fifo
            + QROWS * 4 + (2 * MAX_STAGES + 5) * 8 + 16 + 1024)


def stages(dim: int, ksel: int, tile: int, mask: bool = False) -> int:
    """tc_pick_stages: the deepest ring that fits, 0 when not even two stages do."""
    for s in range(MAX_STAGES, 1, -1):
        if smem_bytes(dim, ksel, s, tile, mask) <= SMEM_OPTIN:
            return s
    return 0


def auto_tile(dim: int, ksel: int, mask: bool = False) -> int:
    """tc_auto_tile for a search (the bring-up score dump always takes 64-row tiles)."""
    return WIDE if stages(dim, ksel, WIDE, mask) >= WIDE_MIN_STAGES else NARROW


def largest_wide_k(dim: int, mask: bool = False) -> int:
    """The largest k (ksel = k + 8) for which the search takes 128-row tiles."""
    return max(k for k in range(1, 129) if auto_tile(dim, k + 8, mask) == WIDE)


@pytest.mark.parametrize("dim,k,mask,tile,ring", [
    (768, 32, False, WIDE, 4),      # the benchmark's shape: four 16 KB stages
    (768, 33, False, WIDE, 4),      # the largest k at dim 768
    (768, 34, False, NARROW, 8),    # three stages would starve: the 64-row kernel with its eight 8 KB stages
    (768, 32, True, NARROW, 8),     # tenant-scope masks cost the fourth stage
    (768, 56, False, NARROW, 7),
    (768, 128, False, NARROW, 5),
    (1024, 32, False, NARROW, 4),   # the query block alone takes 128 KB
    (1024, 56, False, NARROW, 3),
    (1024, 128, False, NARROW, 0),  # no tensor-core path at all (tc_shape_ok)
    (576, 32, False, WIDE, 5),
    (64, 32, True, WIDE, 9),
])
def test_tile_width_and_ring_depth(dim, k, mask, tile, ring):
    assert auto_tile(dim, k + 8, mask) == tile
    assert stages(dim, k + 8, tile, mask) == ring


def test_wide_layout_is_never_picked_where_it_does_not_fit():
    for dim in range(64, 1025, 64):
        for k in range(1, 129):
            for mask in (False, True):
                if auto_tile(dim, k + 8, mask) == WIDE:
                    assert smem_bytes(dim, k + 8, WIDE_MIN_STAGES, WIDE, mask) <= SMEM_OPTIN
    assert largest_wide_k(768) == 33

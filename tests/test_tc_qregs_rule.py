"""Where the similarity kernel keeps its query operand, mirrored from the host (run_tc_block in csrc/capi.cu,
make_layout in csrc/simtopk_tc.cu).  The tile width is decided first and from the layout with the whole query block in
shared memory (tests/test_tc_tile_rule.py).  A launch that took 128-row tiles then holds its first QREGS query k-blocks
in the MMA warpgroup's registers when dim / 64 has that many, and the deepest ring is sized without their 8 KB tiles:
every two k-blocks in registers are one more 16 KB stage.  tests/test_gpu_tc_qregs.py checks the library's answers."""

from __future__ import annotations

import pytest

from tests.test_tc_tile_rule import MAX_STAGES, NARROW, SMEM_OPTIN, WIDE, auto_tile, smem_bytes, stages

QREGS = 6                 # kTcQRegs (csrc/internal.h): the one register depth the library is built with
QTILE = 64 * 128          # kQTileBytes: one 64-dim k-block of the 64-query block


def pick_qregs(dim: int, tile: int, opt: int = -1) -> int:
    """run_tc_block: the register depth of a launch whose width is already chosen (opt = the tc_qregs option)."""
    return QREGS if tile == WIDE and opt != 0 and dim // 64 >= QREGS else 0


def smem_bytes_q(dim: int, ksel: int, n_stages: int, tile: int, mask: bool, qregs: int) -> int:
    """tc_smem_bytes with a register depth: the k-blocks in registers have no tile in shared memory."""
    return smem_bytes(dim, ksel, n_stages, tile, mask) - qregs * QTILE


def stages_q(dim: int, ksel: int, tile: int, mask: bool, qregs: int, cap: int = 0) -> int:
    """tc_pick_stages with a register depth, then the tc_stages cap (0 = none), which only makes the ring shallower."""
    for s in range(MAX_STAGES, 1, -1):
        if smem_bytes_q(dim, ksel, s, tile, mask, qregs) <= SMEM_OPTIN:
            return min(s, cap) if cap >= 2 else s
    return 0


@pytest.mark.parametrize("depth,ring", [(0, 4), (2, 5), (4, 6), (6, 7), (8, 8)])
def test_two_kblocks_in_registers_are_one_ring_stage(depth, ring):
    """The benchmark's shape (dim 768, top-32): the footprint stays the same to the byte."""
    assert stages_q(768, 40, WIDE, False, depth) == ring
    assert smem_bytes_q(768, 40, ring, WIDE, False, depth) == smem_bytes(768, 40, 4, WIDE, False)


@pytest.mark.parametrize("dim,k,mask,tile,qregs,ring", [
    (768, 32, False, WIDE, QREGS, 7),
    (768, 33, False, WIDE, QREGS, 7),
    (768, 34, False, NARROW, 0, 8),             # the width rule has not moved: 64-row tiles, nothing in registers
    (768, 32, True, NARROW, 0, 8),
    (1024, 32, False, NARROW, 0, 4),
    (576, 32, False, WIDE, QREGS, 8),
    (64 * QREGS, 32, False, WIDE, QREGS, 10),   # no query tile left in shared memory
    (64 * (QREGS + 1), 32, False, WIDE, QREGS, 9),
    (64 * (QREGS - 1), 32, False, WIDE, 0, 7),  # fewer k-blocks than the depth: all of them in shared memory
    (64, 32, True, WIDE, 0, 9),
])
def test_register_depth_and_ring(dim, k, mask, tile, qregs, ring):
    assert auto_tile(dim, k + 8, mask) == tile
    assert pick_qregs(dim, tile) == qregs
    assert stages_q(dim, k + 8, tile, mask, qregs) == ring
    assert pick_qregs(dim, tile, opt=0) == 0
    assert stages_q(dim, k + 8, tile, mask, 0) == stages(dim, k + 8, tile, mask)


def test_every_pick_fits_and_the_cap_only_shortens():
    for dim in range(64, 1025, 64):
        for k in range(1, 129):
            for mask in (False, True):
                # auto width, and 128-row tiles forced wherever at least two of their stages fit
                for tile in {auto_tile(dim, k + 8, mask), WIDE}:
                    if stages(dim, k + 8, tile, mask) < 2:
                        continue
                    qregs = pick_qregs(dim, tile)
                    assert qregs in (0, QREGS) and qregs <= dim // 64
                    ring = stages_q(dim, k + 8, tile, mask, qregs)
                    assert stages(dim, k + 8, tile, mask) <= ring <= MAX_STAGES
                    assert smem_bytes_q(dim, k + 8, ring, tile, mask, qregs) <= SMEM_OPTIN
                    for cap in (2, 3, MAX_STAGES):
                        assert stages_q(dim, k + 8, tile, mask, qregs, cap) == min(ring, cap)

"""CPU: the work partition of the stream-K matrix-DFT kernel (csrc/mdft_tc.cu, wgmma_gemm_kernel<true>), restated in Python.

The kernel cuts tiles x chunks into gridDim.x contiguous ranges; a CTA walks its range as segments (tile, chunk range).
Invariants the device code relies on:
  * every chunk of every tile belongs to exactly one segment;
  * a segment that starts inside a tile is the FIRST segment of its CTA (so its partial is published before any wait) and
    a CTA has at most one such segment (one partial slot per CTA);
  * the head segment of a split tile is the LAST segment of its CTA and the pieces it gathers are exactly the first
    segments of CTAs g+1, g+2, ... up to the one that reaches the tile's end."""
import pytest


def segments(g, G, ntiles, upt):
    U = ntiles * upt
    u0, u1 = U * g // G, U * (g + 1) // G
    out, u = [], u0
    while u < u1:
        tile = u // upt
        ub = u - tile * upt
        ue = min(upt, ub + (u1 - u))
        out.append((tile, ub, ue))
        u += ue - ub
    return out


def gathered_by_owner(g, G, ntiles, upt, tile):
    U = ntiles * upt
    tile_u1 = (tile + 1) * upt
    got = []
    for gp in range(g + 1, G):
        got.append(gp)
        if U * (gp + 1) // G >= tile_u1:
            break
    return got


# H100 grids (G = 132 SMs, 128 x 128 tiles, 2 K-blocks of 32 per unit): (64, 32) the first stage of a 1024^2 -> 512^2 MDFT,
# (64, 16) of its adjoint, (32, 128) the second stage of C3 (4096^2 -> 512^2) and (128, 32) the first stage of a 1024^2 <->
# 1024^2 coronagraph leg, the last two under PB_MDFT_STREAMK=2.  The rest are other grid sizes and edge cases.
GRIDS = [(64, 32, 132), (64, 16, 132), (32, 128, 132), (128, 32, 132), (33, 4, 132),
         (128, 128, 148), (64, 32, 148), (16, 128, 148), (5, 7, 3), (128, 128, 160), (8, 128, 148)]
# the other grids the tensor-core cases of tests/test_gpu_mdft_vs_fp64.py reach on 132 SMs, by default or under
# PB_MDFT_STREAMK=2 (tests/test_host_mdft_routes.py lists them): rectangular shapes, one K-block pair per unit (nx = 256),
# a 16384-long contraction over 4 tiles, and the 2048 tiles of the C3 adjoint
GRIDS += [(4, 256, 132), (20, 32, 132), (32, 20, 132), (32, 32, 132), (48, 64, 132), (80, 32, 132), (128, 8, 132),
          (128, 16, 132), (128, 24, 132), (192, 64, 132), (256, 8, 132), (256, 16, 132), (256, 128, 132),
          (512, 16, 132), (2048, 16, 132)]


@pytest.mark.parametrize('ntiles,upt,G', GRIDS)
def test_partition_invariants(ntiles, upt, G):
    cover = {}
    first_piece_owner = {}
    for g in range(G):
        segs = segments(g, G, ntiles, upt)
        mid_starts = [i for i, (t, ub, ue) in enumerate(segs) if ub > 0]
        assert mid_starts in ([], [0]), 'only the first segment of a CTA may start inside a tile'
        for i, (t, ub, ue) in enumerate(segs):
            assert 0 <= ub < ue <= upt
            for c in range(ub, ue):
                assert (t, c) not in cover
                cover[(t, c)] = g
            if ub == 0 and ue < upt:
                assert i == len(segs) - 1, 'the head of a split tile is the last segment of its CTA'
                first_piece_owner[t] = g
    assert len(cover) == ntiles * upt
    for t, g in first_piece_owner.items():
        pieces = gathered_by_owner(g, G, ntiles, upt, t)
        want = sorted({cover[(t, c)] for c in range(upt)} - {g})
        assert pieces == want
        for gp in pieces:   # each gathered CTA's partial is its first segment and lies in this tile
            s0 = segments(gp, G, ntiles, upt)[0]
            assert s0[0] == t and s0[1] > 0

"""CPU: which kernels a matrix-DFT apply launches, restated from the host code of csrc/mdft_tc.cu (mdft_tc_shape_ok,
pick_splits, use_streamk) and csrc/cgemm.cu (pb_mdft_apply), and of prysm_b200/fttools.py (MDFT: the tensor-core plans
and the association order of the CUDA-core path).

tests/test_gpu_mdft_vs_fp64.py predicts each case's launches from `mdft_routes` and requires the device to launch
exactly those.  The stream-K grids the cases reach are in the parameter list of tests/test_streamk_partition.py, so
their partition invariants are checked too."""
import pytest

from test_streamk_partition import GRIDS

BM = BN = 128          # wgmma_gemm_kernel output tile
BK = 32                # fp32 elements per K-block
SMS = {'H100 SXM': 132, 'H100 PCIe': 114}

# route kinds of pb_route_launch_count (include/prysm_b200.h)
ROUTE_MDFT_TC, ROUTE_MDFT_REDUCE, ROUTE_CGEMM = 5, 6, 7
OP_N, OP_T, OP_H, OP_C = 0, 1, 2, 3


def route_code(kind, L=0, flags=0):
    return kind << 28 | L << 8 | flags


def tc_shape_ok(my, ny, mx, nx):
    """mdft_tc_shape_ok"""
    return my % 128 == 0 and mx % 128 == 0 and ny % 128 == 0 and nx % 16 == 0 and ny >= 128 and nx >= 16


def pick_splits(ny):
    """split-K pieces of stage 2 (K = 2 ny): the largest of 8, 4, 2 that divides the K-blocks and leaves 4 or more each"""
    kblocks = 2 * ny // BK
    s = 8
    while s > 1 and (kblocks % s != 0 or kblocks // s < 4):
        s >>= 1
    return s


def use_streamk(tiles, kblocks, chunk, sms, streamk=1):
    """use_streamk: a grid that leaves a good part of the SMs idle (=2: any legal grid), in whole drain chunks"""
    return bool(streamk) and kblocks % chunk == 0 and tiles % sms != 0 and \
        (streamk >= 2 or (5 * tiles < 4 * sms and 4 * tiles >= sms)) and tiles * (kblocks // chunk) >= 4 * sms


def tc_stages(my, ny, mx, nx, sms, streamk=1, chunk=2):
    """the forms of the two GEMMs of pb_mdft_tc_apply: ('plain', 1), ('streamk', 1) or ('splitk', s), and the grid of
    each as (tiles, K-blocks); None when the shape is not covered"""
    if not tc_shape_ok(my, ny, mx, nx):
        return None
    t1, k1 = (ny // BM) * (2 * mx // BN), 2 * nx // BK          # M = ny, N = 2 mx, K = 2 nx
    t2, k2 = (mx // BM) * (2 * my // BN), 2 * ny // BK          # M = mx, N = 2 my, K = 2 ny
    s1 = ('streamk', 1) if use_streamk(t1, k1, chunk, sms, streamk) else ('plain', 1)
    s2 = ('streamk', 1) if use_streamk(t2, k2, chunk, sms, streamk) else ('splitk', pick_splits(ny))
    return (s1, (t1, k1)), (s2, (t2, k2))


def tc_launches(stages):
    """route code -> launches of one pb_mdft_tc_apply with these stage forms"""
    (s1, _), (s2, _) = stages
    out = {route_code(ROUTE_MDFT_TC, 1, int(s1[0] == 'streamk')): 1}
    if s2[0] == 'streamk':
        out[route_code(ROUTE_MDFT_TC, 1, 1 | 2)] = 1
    else:
        out[route_code(ROUTE_MDFT_TC, s2[1], 2 | 4)] = 1
        out[route_code(ROUTE_MDFT_REDUCE, s2[1])] = 1
    return out


def left_first(my, ny, mx, nx, adjoint):
    """MDFT._forward_left_first / _adjoint_left_first: the cheaper association"""
    if adjoint:
        return ny * mx * (my + nx) <= my * nx * (mx + ny)
    return my * nx * (ny + mx) <= ny * mx * (nx + my)


def cgemm_pairs(adjoint, lf):
    """the (opA, opB) of the two cgemm_simt calls of one pb_mdft_apply branch, in launch order"""
    if not adjoint:
        return [(OP_N, OP_N), (OP_N, OP_T)] if lf else [(OP_N, OP_T), (OP_N, OP_N)]
    return [(OP_H, OP_N), (OP_N, OP_C)] if lf else [(OP_N, OP_C), (OP_H, OP_N)]


def cgemm_code(dtype, opA, opB):
    """dtype 0: complex64, 1: complex128"""
    return route_code(ROUTE_CGEMM, 0, dtype | opA << 1 | opB << 3)


def mdft_routes(my, ny, mx, nx, sms, adjoint=False, streamk=1, chunk=2, dtype=0):
    """What fttools.MDFT(x, y, fx, fy) with len(fy), len(y), len(fx), len(x) = my, ny, mx, nx launches for one apply:
    ('tc', stages, launches) or ('cgemm', left_first, launches).  The adjoint runs the same tensor-core GEMM pair on the
    swapped shape (ny, my, nx, mx) through the bases Ey^H, Ex^H, when that shape is covered."""
    shape = (ny, my, nx, mx) if adjoint else (my, ny, mx, nx)
    st = tc_stages(*shape, sms, streamk, chunk) if dtype == 0 else None
    if st is not None:
        return 'tc', st, tc_launches(st)
    lf = left_first(my, ny, mx, nx, adjoint)
    launches = {}
    for a, b in cgemm_pairs(adjoint, lf):
        launches[cgemm_code(dtype, a, b)] = launches.get(cgemm_code(dtype, a, b), 0) + 1
    return 'cgemm', lf, launches


def streamk_grids(my, ny, mx, nx, sms, adjoint=False, streamk=1, chunk=2):
    """(tiles, units per tile, SMs) of every stream-K launch of one tensor-core apply"""
    r = mdft_routes(my, ny, mx, nx, sms, adjoint, streamk, chunk)
    if r[0] != 'tc':
        return []
    return [(t, k // chunk, sms) for (form, _), (t, k) in r[1] if form == 'streamk']


def split_tiles(ntiles, upt, G):
    """tiles of a stream-K launch whose K range the partition cuts across two or more CTAs"""
    U = ntiles * upt
    cta = [0] * U
    for g in range(G):
        for u in range(U * g // G, U * (g + 1) // G):
            cta[u] = g
    return {t for t in range(ntiles) if cta[t * upt] != cta[(t + 1) * upt - 1]}


def form_name(stage):
    form, s = stage
    return f'split-K {s}' if form == 'splitk' else form


# (my, ny, mx, nx): the shapes tests/test_gpu_mdft_vs_fp64.py runs on the tensor cores
TC_SHAPES = [(128, 256, 128, 256), (256, 128, 384, 16), (384, 384, 128, 48), (512, 1024, 512, 1024),
             (256, 1024, 640, 1024), (512, 2048, 768, 2048), (512, 4096, 512, 4096), (1024, 1024, 1024, 1024),
             (256, 8192, 128, 256)]

# forms on 132 SMs, default switches: shape -> (forward stage 1, stage 2, adjoint stage 1, stage 2 or 'cgemm')
TABLE_132 = {
    (128, 256, 128, 256): ('plain', 'split-K 4', 'plain', 'split-K 2'),
    (256, 128, 384, 16): ('plain', 'split-K 2', 'cgemm'),
    (384, 384, 128, 48): ('plain', 'split-K 4', 'cgemm'),
    (512, 1024, 512, 1024): ('streamk', 'split-K 8', 'streamk', 'split-K 8'),
    (256, 1024, 640, 1024): ('streamk', 'split-K 8', 'plain', 'split-K 4'),
    (512, 2048, 768, 2048): ('plain', 'streamk', 'plain', 'split-K 8'),
    (512, 4096, 512, 4096): ('plain', 'split-K 8', 'plain', 'split-K 8'),
    (1024, 1024, 1024, 1024): ('plain', 'split-K 8', 'plain', 'split-K 8'),
    (256, 8192, 128, 256): ('plain', 'split-K 8', 'plain', 'split-K 4'),
}
# 114 SMs: stream-K takes grids of 29 to 91 tiles (132 SMs: 33 to 105), so the 32-tile grids qualify as well -- the
# second stage of 1024^2 -> 512^2 and of C3, and the first stage of the (640, 1024) adjoint
TABLE_114 = {
    (128, 256, 128, 256): ('plain', 'split-K 4', 'plain', 'split-K 2'),
    (256, 128, 384, 16): ('plain', 'split-K 2', 'cgemm'),
    (384, 384, 128, 48): ('plain', 'split-K 4', 'cgemm'),
    (512, 1024, 512, 1024): ('streamk', 'streamk', 'streamk', 'split-K 8'),
    (256, 1024, 640, 1024): ('streamk', 'split-K 8', 'streamk', 'split-K 4'),
    (512, 2048, 768, 2048): ('plain', 'streamk', 'plain', 'split-K 8'),
    (512, 4096, 512, 4096): ('plain', 'streamk', 'plain', 'split-K 8'),
    (1024, 1024, 1024, 1024): ('plain', 'split-K 8', 'plain', 'split-K 8'),
    (256, 8192, 128, 256): ('plain', 'split-K 8', 'plain', 'split-K 4'),
}


def summary(shape, sms, streamk=1, chunk=2):
    out = []
    for adjoint in (False, True):
        r = mdft_routes(*shape, sms, adjoint, streamk, chunk)
        out += [form_name(s) for s, _ in r[1]] if r[0] == 'tc' else ['cgemm']
    return tuple(out)


@pytest.mark.parametrize('sms,table', [(132, TABLE_132), (114, TABLE_114)])
def test_route_table(sms, table):
    assert sorted(table) == sorted(TC_SHAPES)
    got = {s: summary(s, sms) for s in TC_SHAPES}
    assert got == table


def test_switches():
    """PB_MDFT_STREAMK=0 never takes stream-K; =2 takes it in both stages of C3 and of 1024^2 <-> 1024^2"""
    for shape in TC_SHAPES:
        assert 'streamk' not in summary(shape, 132, streamk=0)
    for shape in ((512, 4096, 512, 4096), (1024, 1024, 1024, 1024)):
        s = summary(shape, 132, streamk=2)
        assert s[:2] == ('streamk', 'streamk'), s
    # a chunk that does not divide the K-blocks rules stream-K out
    assert summary((512, 1024, 512, 1024), 132, chunk=3)[0] == 'plain'


def test_route_details():
    # one K-block (nx = 16) and three (nx = 48): the drain at the segment's last K-block
    st = tc_stages(256, 128, 384, 16, 132)
    assert st[0][1] == (6, 1) and st[1] == (('splitk', 2), (12, 8))
    assert tc_stages(384, 384, 128, 48, 132)[0][1] == (6, 3)
    # the adjoint runs the swapped shape; a 16-wide output leaves it on the CUDA-core GEMM, right-first
    kind, lf, launches = mdft_routes(256, 128, 384, 16, 132, adjoint=True)
    assert kind == 'cgemm' and lf is False
    assert launches == {cgemm_code(0, OP_N, OP_C): 1, cgemm_code(0, OP_H, OP_N): 1}
    # complex128 never runs on the tensor cores
    assert mdft_routes(512, 4096, 512, 4096, 132, dtype=1)[0] == 'cgemm'
    # split-K pieces: K-blocks of 2 ny / 32, at least 4 per piece
    assert [pick_splits(n) for n in (128, 256, 384, 512, 640, 4096)] == [2, 4, 4, 8, 8, 8]
    # launches of the split-K form: the partial-plane GEMM and the reduce kernel, with the piece count as L
    assert tc_launches(tc_stages(512, 4096, 512, 4096, 132)) == {
        route_code(ROUTE_MDFT_TC, 1, 0): 1, route_code(ROUTE_MDFT_TC, 8, 6): 1, route_code(ROUTE_MDFT_REDUCE, 8): 1}
    assert tc_launches(tc_stages(512, 2048, 768, 2048, 132)) == {
        route_code(ROUTE_MDFT_TC, 1, 0): 1, route_code(ROUTE_MDFT_TC, 1, 3): 1}


def reached_grids(sms=132):
    """stream-K grids of the tensor-core cases, by default and under PB_MDFT_STREAMK=2"""
    return {g for streamk in (1, 2) for shape in TC_SHAPES for adjoint in (False, True)
            for g in streamk_grids(*shape, sms, adjoint, streamk)}


def test_reached_streamk_grids_are_partition_checked():
    missing = sorted(reached_grids(132) - set(GRIDS))
    assert not missing, f'add these (tiles, units per tile, SMs) to test_streamk_partition.GRIDS: {missing}'


def test_split_tiles():
    # 64 tiles x 32 units over 132 CTAs: 2048 / 132 = 15.5 units per CTA, so every tile is cut
    assert split_tiles(64, 32, 132) == set(range(64))
    # one tile per CTA: none is cut
    assert split_tiles(8, 4, 8) == set()
    assert split_tiles(3, 2, 2) == {1}

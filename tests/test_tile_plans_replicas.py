"""The tensor-core planner's decisions for the replica step (Darknet(..., replicas=R)) without a GPU.

The replica step (the reference's four-replica nn.DataParallel step) runs every convolution of both branches over the
whole batch, as the one-replica step does, but with R support sets (R * n_cls support images) and a per-replica head:
replica r's B / R query images go through their own W (.) rw_r, so the head's forward and input-gradient GEMMs have
M = (B / R) G^2 rows and its weight gradient sums over K = (B / R) G^2 pixels, once per replica.  This file lists those
GEMMs for R = 4 at 416 and 608 (B = 64, the reference's training batch) and for B = 4 (one image per replica), and
pins the flavours the planner picks, the head's last M tile and its split-K count.  tests/test_gpu_zzz_step_replicas.py
takes the flavour sets a checked replica step must reach from here.
"""
import pytest

from test_tile_plans_eval import TC_BM, last_m_tile
from test_tile_plans_scales import FLAVOURS, _lib, branch_gemms, flavours, planned_flavours, query_gemms, wgrad_splits

HEAD = ('head', 'head-dgrad', 'head-wgrad')
# (side, B, n_cls, R) of the checked replica steps
SHAPES = ((416, 64, 20, 4), (608, 64, 20, 4), (416, 4, 3, 4), (416, 64, 20, 2))


def replica_gemms(side, B, n_cls, R):
    """The tensor-core GEMMs of one R-replica training step: the query branch at B with its head triple once per replica
    at B / R images, then the reweighting net over R * n_cls support images.  Tuples as in test_tile_plans_scales."""
    from fewshot_detection_b200 import netcfg
    q = query_gemms(side, B, n_cls)
    body = [g for g in q if g[0] not in HEAD]
    head = [(g[0], B // R) + g[2:] for g in q if g[0] in HEAD]
    sup = branch_gemms(netcfg.reweighting_net_blocks(), R * n_cls, n_cls)
    return body + head * R + sup


def one_replica_gemms(side, B, n_cls):
    from fewshot_detection_b200 import netcfg
    return query_gemms(side, B, n_cls) + branch_gemms(netcfg.reweighting_net_blocks(), n_cls, n_cls)


def test_replica_gemm_lists():
    """Every layer but the head as in the one-replica step (the support branch at R * n_cls images); the head's three
    GEMMs R times at B / R images: M = 16 G^2 = 2704 rows at 416 and 5776 at 608, 169 with one image per replica."""
    for side, B, n_cls, R in SHAPES:
        g = replica_gemms(side, B, n_cls, R)
        one = one_replica_gemms(side, B, n_cls)
        G = side // 32
        assert [x for x in g if x[0] not in HEAD and x[1] == B] == [x for x in one if x[0] not in HEAD and x[1] == B]
        heads = [x for x in g if x[0] in HEAD]
        assert len(heads) == 3 * R and all(x[1] == B // R and x[2] == x[3] == G for x in heads)
        assert heads[:3] == [x[:1] + (B // R,) + x[2:] for x in one if x[0] in HEAD]
        assert len(g) == len(one) + 3 * (R - 1)
    M = lambda side, B, R: B // R * (side // 32) ** 2
    assert (M(416, 64, 4), M(608, 64, 4), M(416, 4, 4), M(416, 64, 2)) == (2704, 5776, 169, 5408)


# per shape: (last M tile of the head's forward / input-gradient GEMMs, split-K count of its weight gradient)
HEAD_PLAN = {(416, 64, 20, 4): (16, 3), (608, 64, 20, 4): (16, 3), (416, 4, 3, 4): (41, 1), (416, 64, 20, 2): (32, 3)}


@pytest.mark.parametrize('shape', SHAPES, ids=['r4-416', 'r4-608', 'r4-b4', 'r2-416'])
def test_replica_head_plans(shape):
    """The per-replica head: im2col (short K: a 1x1 GEMM over 1024 channels) forward and input gradient, ending on a
    partial M tile (16 rows at B = 64 and R = 4 for both sides, 41 for one image, 32 for R = 2); its weight gradient is
    one-tap and split three ways over K = (B / R) G^2 pixels (the one-replica head over 64 G^2 pixels splits four
    ways), unsplit for one image per replica."""
    L = _lib()
    side, B, n_cls, R = shape
    heads = [g for g in replica_gemms(*shape) if g[0] in HEAD][:3]
    fwd, dgrad, wgrad = heads
    tile, splits = HEAD_PLAN[shape]
    for g in (fwd, dgrad):
        assert flavours(L, g) == {'im2col-short'}, g
        assert last_m_tile(g) == tile, (g, last_m_tile(g))
        assert L.fsdet_conv_tc_stat_rows(*g[1:]) == -(-g[1] * g[2] * g[3] // TC_BM)
    assert flavours(L, wgrad) == {'wgrad-taps1', 'wgrad-splitk' if splits > 1 else 'wgrad-nosplit'}, wgrad
    assert wgrad_splits(L, wgrad) == splits, (wgrad, wgrad_splits(L, wgrad))


# the flavours each checked replica step reaches (StepChecker's names): all seven at every shape, the one-image replicas
# included (their body runs at B = 4 and the support branch at 12 images)
REPLICA_FLAVOURS = {shape: set(FLAVOURS) for shape in SHAPES}


@pytest.mark.parametrize('shape', SHAPES, ids=['r4-416', 'r4-608', 'r4-b4', 'r2-416'])
def test_replica_flavour_sets(shape):
    """The flavour set of the whole replica step, and the one-replica step's at the same B for comparison: the body of
    the network plans as before, so at B = 64 both sets are all seven flavours."""
    L = _lib()
    got = planned_flavours(L, replica_gemms(*shape))
    assert got == REPLICA_FLAVOURS[shape], (shape, sorted(got))
    side, B, n_cls, R = shape
    if B == 64:
        assert got == planned_flavours(L, one_replica_gemms(side, B, n_cls))

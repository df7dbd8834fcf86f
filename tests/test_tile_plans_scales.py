"""The tensor-core planner's decisions for the query branch at every multi-scale input side (CPU only, no GPU).

Multi-scale training (dataset.multiscale_width) feeds query batches of side 320, 352, ..., 608; the support branch stays
at 416.  Which kernel flavour a convolution takes - halo-tile, short-K or long-K im2col, split or unsplit weight gradient,
one- or two-tap weight tiles - is decided by pure C functions of the library from the layer shape.  This file walks the
network's layer list at each side, lists every tensor-core GEMM of a training step, and pins what the planner decides
for the query branch at B = 64, so that a planner change that moves a side onto another flavour fails without a GPU.
tests/test_gpu_zz_step_scales.py uses the same walk to predict which flavours a real step must reach.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIDES = tuple(range(320, 609, 32))
SMALLK_MAX = 2304      # conv_tc.cu tc_plan: K = k*k*Cin above this (Cin % 64 == 0) runs the long-K (folded) flavour
FWD_MODE, WGRAD_MODE = 3, 0     # engine.TC_TERMS defaults: fp32-grade forward / input gradient / head, fp16 weight gradient
FLAVOURS = ('halo', 'im2col-short', 'im2col-long', 'wgrad-splitk', 'wgrad-nosplit', 'wgrad-taps1', 'wgrad-taps2')


def _lib():
    if not os.path.exists(os.path.join(ROOT, 'fewshot_detection_b200', 'libfsdet.so')):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    from fewshot_detection_b200 import _lib
    return _lib.lib


def _up(v, m):
    return (v + m - 1) // m * m


def conv_layers(blocks):
    """[(Cin, Cout, k, H, W, dynamic)] of every convolution of a Darknet block list, in order (route, reorg and
    max-pool blocks change the shapes; 2x2 max-pools floor odd sides)."""
    head = blocks[0]
    C, H, W = int(head.get('channels', 3)), int(head['height']), int(head['width'])
    outs, convs = [], []
    for b in blocks[1:]:
        t = b['type']
        if t == 'convolutional':
            convs.append((C, int(b['filters']), int(b['size']), H, W, b.get('dynamic') == '1'))
            C = int(b['filters'])
        elif t == 'maxpool' and b['stride'] == '2':
            H, W = H // 2, W // 2
        elif t == 'route':
            src = [len(outs) + int(l) if int(l) < 0 else int(l) for l in b['layers'].split(',')]
            C, H, W = sum(outs[i][0] for i in src), outs[src[0]][1], outs[src[0]][2]
        elif t == 'reorg':
            C, H, W = 4 * C, H // 2, W // 2
        outs.append((C, H, W))
    return convs


def branch_gemms(blocks, B, n_cls):
    """The tensor-core GEMMs of one training step of a branch, as the engine issues them: every convolution but the
    first (an exact-fp32 SIMT kernel) runs forward, input gradient and weight gradient; the dynamic convolution and the
    1x1 head after it run as one head GEMM of N = round_up(n_cls * 30, 64) outputs.  Tuples (kind, B, H, W, Cin, Cout,
    k, mode) with the channel counts the kernels are called with."""
    convs = conv_layers(blocks)
    out = []
    i = 1
    while i < len(convs):
        cin, cout, k, H, W, dyn = convs[i]
        if dyn:
            npad = _up(n_cls * convs[i + 1][1], 64)
            out += [('head', B, H, W, cin, npad, 1, FWD_MODE), ('head-dgrad', B, H, W, npad, cin, 1, FWD_MODE),
                    ('head-wgrad', B, H, W, _up(cin, 64), npad, 1, WGRAD_MODE)]
            i += 2
            continue
        out += [('fwd', B, H, W, _up(cin, 32), cout, k, FWD_MODE), ('dgrad', B, H, W, cout, _up(cin, 32), k, FWD_MODE),
                ('wgrad', B, H, W, _up(cin, 64), _up(cout, 64), k, WGRAD_MODE)]
        i += 1
    return out


def query_gemms(side, B, n_cls=15):
    from fewshot_detection_b200 import netcfg
    return branch_gemms(netcfg.darknet_dynamic_blocks(side, side), B, n_cls)


def support_gemms(n_cls):
    from fewshot_detection_b200 import netcfg
    return branch_gemms(netcfg.reweighting_net_blocks(), n_cls, n_cls)


def wgrad_splits(lib, g):
    _, B, H, W, Cin, Cout, k, mode = g
    ws = lib.fsdet_conv_tc_wgrad_workspace_floats(B, H, W, Cin, Cout, k, mode)
    return max(1, ws // (Cout * k * k * Cin))


def flavours(lib, g):
    """The flavour names test_gpu_zz_step_gemms.StepChecker records for this GEMM."""
    kind, B, H, W, Cin, Cout, k, mode = g
    if kind.endswith('wgrad'):
        return {'wgrad-taps%d' % (1 if Cin >= 128 else 2), 'wgrad-splitk' if wgrad_splits(lib, g) > 1 else 'wgrad-nosplit'}
    if lib.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, mode) == 1:
        return {'halo'}
    return {'im2col-long' if Cin % 64 == 0 and k * k * Cin > SMALLK_MAX else 'im2col-short'}


def planned_flavours(lib, gemms):
    s = set()
    for g in gemms:
        s |= flavours(lib, g)
    return s


def first_layer_tail(side):
    """(width of the last column tile, its remainder mod 3) of conv_first_fwd_kernel: tiles of FT_W = 104 columns, row
    walk unrolled by three (conv_simt.cu)."""
    wn = side - 104 * ((side - 1) // 104)
    return wn, wn % 3


# split-K factor of each query-branch weight gradient at B = 64, in layer order (the head's last).  wg_splits caps the
# count by the tile count, not by the pixels, so it is the same at every side; what changes with the side is the slice
# of pixels per split (a multiple of 64) and with it the length of the last slice, which can be short or empty.
SPLITS = (26, 26, 129, 26, 22, 65, 22, 7, 33, 7, 33, 7, 2, 4, 2, 4, 2, 1, 1, 33, 1, 4)


def last_slice(M, splits):
    """pixels of the last split of conv_tc.cu's weight gradient (<= 0: that split has no pixels)"""
    pps = -(-(-(-M // splits)) // 64) * 64
    return M - (splits - 1) * pps


def test_layer_walk_of_the_detector():
    """The walk reproduces the detector's shapes: 24 convolutions, the passthrough route of 1280 channels at side / 32."""
    from fewshot_detection_b200 import netcfg
    convs = conv_layers(netcfg.darknet_dynamic_blocks(608, 608))
    assert len(convs) == 24
    assert convs[0][:5] == (3, 32, 3, 608, 608)
    assert convs[1][:5] == (32, 64, 3, 304, 304)
    assert convs[20][:5] == (512, 64, 1, 38, 38)          # route -9: the last 512-channel layer at side / 16
    assert convs[21][:5] == (1280, 1024, 3, 19, 19)       # reorg (4 x 64) + the 1024-channel trunk
    assert convs[22][5] and convs[23][:3] == (1024, 30, 1)
    sup = conv_layers(netcfg.reweighting_net_blocks())
    assert [c[3] for c in sup] == [416, 208, 104, 52, 26, 13, 6] and sup[0][0] == 4


@pytest.mark.parametrize('side', SIDES)
def test_query_branch_plans_at_every_side(side):
    """At B = 64: the halo-tile kernel takes exactly the 3x3 layers at side / 2 and side / 4 (both directions, every side
    tiles by 8 columns and wastes at most 8 of 16 rows); BatchNorm partial rows are one per SM for the halo kernel and
    one per 128-pixel tile otherwise; every weight gradient's split-K fills whole rounds of the 132 SMs; the step
    reaches all seven flavours; and the first layer's last column tile is partial at every side but 416."""
    L = _lib()
    gemms = query_gemms(side, 64)
    assert len(gemms) == 3 * 22
    splits_seen, tails = [], []
    for g in gemms:
        kind, B, H, W, Cin, Cout, k, mode = g
        if kind.endswith('wgrad'):
            taps = 1 if Cin >= 128 else 2
            tiles = -(-Cin // (128 // taps)) * -(-k * k // taps) * -(-Cout // 128)
            splits = wgrad_splits(L, g)
            ctas = tiles * splits
            rounds = -(-ctas // 132)
            assert ctas > 0.8 * rounds * 132 or splits == 1, (side, g, tiles, splits)
            splits_seen.append(splits)
            tails.append(last_slice(B * H * W, splits))
            continue
        want = 1 if (k == 3 and H in (side // 2, side // 4)) else 0
        assert L.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, mode) == want, (side, g)
        assert L.fsdet_conv_tc_uses_halo(B, H, W, Cin, Cout, k, mode | 64) == 0
        rows = L.fsdet_conv_tc_stat_rows(B, H, W, Cin, Cout, k, mode)
        assert rows == (132 if want else -(-B * H * W // 128)), (side, g, rows)
    assert tuple(splits_seen) == SPLITS, (side, splits_seen)
    print('side %d: pixels in the last weight-gradient split per layer' % side, tails)
    assert planned_flavours(L, gemms) == set(FLAVOURS), (side, sorted(planned_flavours(L, gemms)))
    wn, rem = first_layer_tail(side)
    assert (wn < 104) == (side != 416) and rem == {320: 2, 352: 1, 384: 0, 416: 2, 448: 2, 480: 1, 512: 0, 544: 0,
                                                   576: 2, 608: 1}[side]

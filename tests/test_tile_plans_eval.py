"""The tensor-core planner's decisions for the evaluation pass at the batch sizes evaluation runs (CPU only, no GPU).

Evaluation (tools/valid_ensemble_b200.py) runs 64 query and 64 support images per forward, then a shorter last batch:
24 of the 4,952 VOC2007 test images, 8 of the 5,000 COCO minival images, 8 of the 200 10-shot VOC support images, 32 of
the 800 10-shot COCO support images; a one-image list or a small shard runs B = 1.  The evaluation forward issues one
GEMM per convolution (no input or weight gradient), so the planner sees other shapes than in a training step: the
halo-tile kernel needs enough 8x16 tiles to fill two rounds of the SMs, and every im2col layer ends on another partial
128-row M tile.  This file pins, for B in EVAL_BATCHES, which layers take the halo kernel, the short- or long-K flavour
of the others and the length of each im2col layer's last M tile.  tests/test_gpu_zz_eval_pass.py takes its flavour
predictions from here.
"""
import pytest

from test_tile_plans_scales import FWD_MODE, _lib, _up, conv_layers, flavours, planned_flavours

EVAL_BATCHES = (1, 2, 3, 8, 24, 32, 64)
TC_BM = 128          # conv_tc_kernels.cuh: rows of one M tile of the im2col kernel


def eval_branch_gemms(blocks, B, n_cls):
    """The tensor-core GEMMs of one evaluation forward of a branch: every convolution but the first (an exact-fp32
    SIMT kernel) as `fwd`, and the dynamic convolution with the 1x1 head after it as one `head` GEMM of
    N = round_up(n_cls * 30, 64).  Tuples (kind, B, H, W, Cin, Cout, k, mode) as in test_tile_plans_scales."""
    convs = conv_layers(blocks)
    out = []
    i = 1
    while i < len(convs):
        cin, cout, k, H, W, dyn = convs[i]
        if dyn:
            out.append(('head', B, H, W, cin, _up(n_cls * convs[i + 1][1], 64), 1, FWD_MODE))
            i += 2
            continue
        out.append(('fwd', B, H, W, _up(cin, 32), cout, k, FWD_MODE))
        i += 1
    return out


def query_eval_gemms(B, n_cls, side=416):
    from fewshot_detection_b200 import netcfg
    return eval_branch_gemms(netcfg.darknet_dynamic_blocks(side, side), B, n_cls)


def support_eval_gemms(B):
    from fewshot_detection_b200 import netcfg
    return eval_branch_gemms(netcfg.reweighting_net_blocks(), B, 0)


def flavour(lib, g):
    (f,) = flavours(lib, g)
    return f


def last_m_tile(g):
    """rows of the last 128-row M tile of an im2col GEMM"""
    _, B, H, W = g[:4]
    return (B * H * W - 1) % TC_BM + 1


# short (S) / long (L) K of the layers that never take the halo kernel, in layer order: K = 9 Cin above 2304 is long
QUERY_K = 'S' * 9 + 'LSLSLLL' + 'SLS'    # 104 (1x1), 52, 26 and 13 pixel layers, the passthrough 1x1, conv22, the head
SUPPORT_K = 'SSLL'                       # the 52, 26, 13 and 6 pixel layers


def test_eval_gemm_lists():
    """22 GEMMs per query forward (21 convolutions and the head), 6 per support forward; heads of the VOC (20 classes:
    N = 600 -> 640) and COCO (80 classes at 416: N = 2400 -> 2432) evaluations."""
    q, s = query_eval_gemms(64, 20), support_eval_gemms(64)
    assert len(q) == 22 and len(s) == 6
    assert q[-1] == ('head', 64, 13, 13, 1024, 640, 1, FWD_MODE)
    assert query_eval_gemms(8, 80)[-1] == ('head', 8, 13, 13, 1024, 2432, 1, FWD_MODE)
    assert [g[2] for g in s] == [208, 104, 52, 26, 13, 6]
    assert all(g[0] == 'fwd' for g in q[:-1] + s)


@pytest.mark.parametrize('B', EVAL_BATCHES)
def test_eval_plans(B):
    """Which layers take the halo kernel: the 208x208 3x3 layer of each branch (338 tiles per image) at every B, the
    104x104 64->128 layers (91 tiles per image) from B = 3 on (264 tiles fill two rounds of the 132 SMs), nothing else.
    The remaining layers keep their short- or long-K flavour at every B, and the BatchNorm statistics rows of a
    convolution that writes them are one per M tile (what the last tile's length counts)."""
    L = _lib()
    for gemms, k_flavours, n_cls in ((query_eval_gemms(B, 20), QUERY_K, 20), (support_eval_gemms(B), SUPPORT_K, 0)):
        halo = [(g[2], g[4], g[5]) for g in gemms if flavour(L, g) == 'halo']
        want = [(208, 32, 64)] + [(104, 64, 128)] * (2 if n_cls else 1) * (B >= 3)
        assert halo == want, (B, n_cls, halo)
        rest = ''.join({'im2col-short': 'S', 'im2col-long': 'L'}[flavour(L, g)] for g in gemms if flavour(L, g) != 'halo')
        assert rest == ('SS' if B < 3 and n_cls else ('S' if B < 3 else '')) + k_flavours, (B, n_cls, rest)
        for g in gemms:
            kind, B_, H, W, Cin, Cout, k, mode = g
            if flavour(L, g) != 'halo':
                assert L.fsdet_conv_tc_stat_rows(B_, H, W, Cin, Cout, k, mode) == -(-B_ * H * W // TC_BM), g
    # the 80-class head plans like the 20-class one
    assert flavour(L, query_eval_gemms(B, 80)[-1]) == 'im2col-short'


# last M-tile length of the im2col layers per side, at each evaluation batch size (a full tile is 128)
LAST_TILE = {       # side: {B: rows}
    104: {1: 64, 2: 128, 3: 64, 8: 128, 24: 128, 32: 128, 64: 128},
    52: {1: 16, 2: 32, 3: 48, 8: 128, 24: 128, 32: 128, 64: 128},
    26: {1: 36, 2: 72, 3: 108, 8: 32, 24: 96, 32: 128, 64: 128},
    13: {1: 41, 2: 82, 3: 123, 8: 72, 24: 88, 32: 32, 64: 64},
    6: {1: 36, 2: 72, 3: 108, 8: 32, 24: 96, 32: 128, 64: 128},
}


@pytest.mark.parametrize('B', EVAL_BATCHES)
def test_eval_last_m_tiles(B):
    """The last M tile of every im2col layer: at B = 64 the 13x13 layers end on 64 rows and the 26x26 ones on a full
    tile; the evaluation tails end elsewhere (13x13: 41, 72 and 88 rows at B = 1, 8 and 24; 26x26: 36, 32 and 96), and
    so does the reweighting net's 6x6 layer (32 rows at B = 8).  At 104x104 only the 1x1 layer runs im2col from B = 3 on."""
    L = _lib()
    for gemms in (query_eval_gemms(B, 20), support_eval_gemms(B), query_eval_gemms(B, 80)):
        for g in gemms:
            if flavour(L, g) == 'halo':
                continue
            assert last_m_tile(g) == LAST_TILE[g[2]][B], (B, g, last_m_tile(g))


def test_eval_flavour_sets():
    """The flavour sets the GPU test expects to reach: halo and both im2col flavours at every evaluation batch size."""
    L = _lib()
    for B in EVAL_BATCHES:
        assert planned_flavours(L, query_eval_gemms(B, 20)) == {'halo', 'im2col-short', 'im2col-long'}, B
        assert planned_flavours(L, support_eval_gemms(B)) == {'halo', 'im2col-short', 'im2col-long'}, B

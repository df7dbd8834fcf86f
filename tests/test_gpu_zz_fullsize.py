"""Size-independent properties of the conv stack at the BASELINE configs[1] size (64 query images, 20 classes,
416x416), where the CPU oracle would take minutes: permuting the query images permutes the (image, class) row blocks
of the head output and nothing else (training-mode BatchNorm statistics, the tensor-wide operand scales of the
tensor-core path and the class reweighting are all permutation invariant up to summation order).
(File name sorts last on purpose: newest GPU tests run last.)"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def relt(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def test_full_size_forward_is_permutation_equivariant_over_images():
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init, synth_masks
    bs, cs = 64, 20
    m = Darknet(netcfg.darknet_dynamic_blocks(), netcfg.reweighting_net_blocks())
    seeded_init(m, 5)
    m = m.cuda().train()
    g = torch.Generator().manual_seed(6)
    x = torch.rand(bs, 3, 416, 416, generator=g).cuda()
    metax = torch.rand(cs, 3, 416, 416, generator=g).cuda()
    mask = torch.from_numpy(synth_masks(cs, 416, 7)).cuda()
    perm = torch.randperm(bs, generator=g).cuda()
    with torch.no_grad():
        out = m(x, metax, mask)
        out_p = m(x[perm].contiguous(), metax, mask)
    assert tuple(out.shape) == (bs * cs, 30, 13, 13)
    assert torch.isfinite(out).all()
    want = out.view(bs, cs, 30, 13, 13)[perm].reshape(bs * cs, 30, 13, 13)
    assert relt(out_p, want) < 1e-3                      # the north star's float bar; measured differences are ~1e-6
    # and the permutation is visible at all (the rows really moved)
    assert relt(out_p, out) > 1e-2
    # class rows of one image differ only through the reweighting vectors: swapping two support classes swaps rows
    sw = list(range(cs))
    sw[0], sw[1] = sw[1], sw[0]
    with torch.no_grad():
        out_s = m(x, metax[sw].contiguous(), mask[sw].contiguous())
    want_s = out.view(bs, cs, 30, 13, 13)[:, sw].reshape(bs * cs, 30, 13, 13)
    assert relt(out_s, want_s) < 1e-3

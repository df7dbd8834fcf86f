"""The replica step on the GPU (Darknet(..., replicas=R)): the reference's nn.DataParallel step of R replicas inside
one process.

- test_segmented_passes_full_size   the segmented BatchNorm passes at the step's shapes (B = 64, R = 4, 416 and 608)
                                    against float64 per segment: statistics, backward sums and dz
- test_replica_step_vs_oracle       mini model, R = 2 and 4: output, loss, running statistics and gradients against an
                                    oracle step that runs R separate forward calls on the chunks with their support
                                    rows, concatenates the outputs, applies one RegionLossV2 and one backward, and
                                    keeps the running statistics of the first call
- test_graph_replay_equals_eager    full size, R = 4: GraphedTrainStep's gradients and running statistics bit-equal to
                                    an eager step of a twin model loaded with the same state, neg = 1 and neg = 0"""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-3


def relt(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def bit_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _bn_stats(m):
    return {n: b for n, b in m.named_buffers() if n.endswith(('running_mean', 'running_var'))}


def _batch(bs, cs, R, side, meta_side, seed):
    from seeding import synth_targets, synth_masks
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(bs, 3, side, side, generator=g)
    metax = torch.rand(R * cs, 3, meta_side, meta_side, generator=g)
    mask = torch.from_numpy(synth_masks(R * cs, meta_side, seed + 1))
    tgt = torch.from_numpy(synth_targets(bs, cs, seed + 2))
    return x.cuda(), metax.cuda(), mask.cuda(), tgt


# ------------------------------------------------------------------------------------------------- segmented passes
@pytest.mark.parametrize('side', [416, 608])
def test_segmented_passes_full_size(side):
    from fewshot_detection_b200 import _lib as L
    st = lambda: torch.cuda.current_stream().cuda_stream
    B, R = 64, 4
    for div, C in ((1, 32), (4, 128), (32, 1024)):
        H = side // div
        seg_pix = B // R * H * H
        g = torch.Generator(device='cuda').manual_seed(H + C)
        # per-segment scales and offsets with |mean| / std below 10, the range where one-pass fp32 statistics hold the bars
        z = (torch.randn(R, seg_pix, C, device='cuda', generator=g) * (0.5 + 2.5 * torch.rand(R, 1, C, device='cuda', generator=g)) +
             torch.randn(R, 1, C, device='cuda', generator=g)).reshape(-1, C).contiguous()
        rows = L.lib.fsdet_bn_seg_colstats_rows(seg_pix, R)
        part = torch.empty(R * (rows + L.lib.fsdet_bn_stat_scratch_rows()), 4 * C, device='cuda')
        gamma = torch.rand(C, device='cuda', generator=g) + 0.5
        beta = torch.randn(C, device='cuda', generator=g)
        rm, rv = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
        vec = torch.empty(5, R, C, device='cuda')
        amax = torch.empty(1, device='cuda')
        L.call('fsdet_bn_seg_colstats', z.data_ptr(), C, seg_pix, R, C, part.data_ptr(), st())
        L.call('fsdet_bn_seg_finalize', part.data_ptr(), rows, R, seg_pix, gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(),
               rv.data_ptr(), 0.1, 1e-5, *[vec[i].data_ptr() for i in range(4)], 0.1, amax.data_ptr(), vec[4].data_ptr(), C, st())
        # float64 references one segment at a time (a 608 x 608 layer is 2.8 M pixels x 32 channels per segment)
        zs = z.view(R, seg_pix, C)
        mu = torch.stack([zs[k].double().mean(0) for k in range(R)])
        var = torch.stack([zs[k].double().var(0, unbiased=False) for k in range(R)])
        std = (var + 1e-5).sqrt()
        em, ei = ((vec[0].double() - mu).abs() / std).max().item(), ((vec[1].double() - 1 / std).abs() * std).max().item()
        print('%d x %d, C %d: mean %.2e std, invstd %.2e relative' % (H, H, C, em, ei))
        assert em <= 1e-5 and ei <= 1e-5, (side, H, C, em, ei)
        assert relt(rv, 0.9 + 0.1 * var[0] * seg_pix / (seg_pix - 1)) < 1e-6 and relt(rm, 0.1 * mu[0]) < 1e-5
        # backward through the unpooled activation (the general kernel) with a gradient dominated by its mean
        dy = (torch.randn(B * H * H, C, device='cuda', generator=g) * 0.1 + 1.0).contiguous()
        brow = L.lib.fsdet_bn_seg_bwd_rows(B, H, H, R)
        bpart = torch.empty(R * (brow + 1), 3 * C, dtype=torch.float64, device='cuda')
        sc, sh, mean, istd, xabs = (vec[i] for i in (2, 3, 0, 1, 4))
        L.call('fsdet_bn_act_bwd_reduce_seg', z.data_ptr(), C, dy.data_ptr(), C, None, 0, sc.data_ptr(), sh.data_ptr(),
               mean.data_ptr(), istd.data_ptr(), 0.1, bpart.data_ptr(), B, H, H, C, R, seg_pix, st())
        coef = torch.empty(R, 2, C, dtype=torch.float64, device='cuda')
        dg, db, bound = torch.empty(C, device='cuda'), torch.empty(C, device='cuda'), torch.empty(1, device='cuda')
        L.call('fsdet_bn_bwd_finalize_seg', bpart.data_ptr(), brow, R, seg_pix, gamma.data_ptr(), istd.data_ptr(),
               xabs.data_ptr(), dg.data_ptr(), db.data_ptr(), coef.data_ptr(), bound.data_ptr(), C, st())
        dz = torch.empty_like(z)
        L.call('fsdet_bn_act_bwd_apply_seg', z.data_ptr(), C, dy.data_ptr(), C, None, 0, sc.data_ptr(), sh.data_ptr(),
               mean.data_ptr(), istd.data_ptr(), coef.data_ptr(), 0.1, dz.data_ptr(), C, None, None, C, None, B, H, H, C, R,
               seg_pix, st())
        dys, dzs = dy.view(R, seg_pix, C), dz.view(R, seg_pix, C)
        s1_all = s2_all = 0
        for k in range(R):
            y = torch.addcmul(sh[k], zs[k], sc[k])
            du = dys[k].double() * torch.where(y > 0, 1.0, float(np.float32(0.1))).double()
            del y
            xh = (zs[k].double() - mean[k].double()) * istd[k].double()
            s1, s2 = du.sum(0), (du * xh).sum(0)
            assert ((coef[k, 0] * seg_pix - s1).abs() <= 1e-6 * du.abs().sum(0)).all(), (side, H, C, k)
            assert ((coef[k, 1] * seg_pix - s2).abs() <= 1e-6 * (du * xh).abs().sum(0)).all(), (side, H, C, k)
            s1_all, s2_all = s1_all + s1, s2_all + s2
            c1, c2 = coef[k, 0], coef[k, 1]
            sg = sc[k].double()
            err = (dzs[k].double() - sg * (du - c1 - xh * c2)).abs()
            assert (err <= 1e-6 * sg.abs() * (du.abs() + c1.abs() + (xh * c2).abs()) + 1e-30).all(), (side, H, C, k)
            del du, xh, err
        assert relt(db, s1_all) < 1e-6 and relt(dg, s2_all) < 1e-6
        assert bound.item() >= dz.abs().max().item()
        del z, zs, dy, dys, dz, dzs, part, bpart
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------- mini model
def _mini(R, seed):
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init
    m = Darknet(netcfg.mini_dynamic_blocks(128, 4), netcfg.mini_reweighting_blocks(64, 4, 128), replicas=R)
    seeded_init(m, seed)
    m = m.cuda().train()
    L = m.models[len(m.models) - 1]
    L.seen = 20000
    L.verbose = False
    return m, L


@pytest.mark.parametrize('R', [2, 4])
def test_replica_step_vs_oracle(R):
    bs, cs = 8, int(_mini(1, 0)[1].num_classes)
    grads = {}
    for seed in (41, 42, 43):
        x, metax, mask, tgt = _batch(bs, cs, R, 128, 64, seed)
        m, L = _mini(R, 7)
        random.seed(seed)
        out = m(x, metax, mask)
        loss = L(out, tgt)
        loss.backward()
        # the oracle: R separate calls of the one-replica model, one loss over the concatenated outputs
        om, oL = _mini(1, 7)
        nb, outs, first = bs // R, [], None
        for r in range(R):
            outs.append(om(x[r * nb:(r + 1) * nb], metax[r * cs:(r + 1) * cs], mask[r * cs:(r + 1) * cs]))
            if r == 0:
                first = {n: b.detach().clone() for n, b in _bn_stats(om).items()}
        random.seed(seed)
        oloss = oL(torch.cat(outs, 0), tgt)
        oloss.backward()
        assert out.shape == (bs * cs,) + tuple(outs[0].shape[1:])
        assert relt(out.detach(), torch.cat(outs, 0).detach()) < TOL, seed
        assert abs(loss.item() - oloss.item()) < TOL * abs(oloss.item()), seed
        for n, b in _bn_stats(m).items():
            assert relt(b, first[n]) < TOL, (seed, n)
        for (n, p), op in zip(m.named_parameters(), om.parameters()):
            grads.setdefault(n, []).append(relt(p.grad, op.grad))
    worst = {n: float(np.median(v)) for n, v in grads.items()}
    print('R=%d: worst median gradient error %.3g (%s)' % (R, max(worst.values()), max(worst, key=worst.get)))
    assert max(worst.values()) < TOL, worst


# --------------------------------------------------------------------------------------------------- graph replay
@pytest.mark.parametrize('neg', [1, 0])
def test_graph_replay_equals_eager(neg, monkeypatch):
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.distributed import GradAllReducer
    from fewshot_detection_b200.graph import GraphedTrainStep
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.trainer import lr_factor, sgd_hyper_parameters
    from seeding import seeded_init
    bs, cs, R = 64, 20, 4
    monkeypatch.setattr(cfg, 'neg_ratio', neg)

    def model():
        m = Darknet(netcfg.darknet_dynamic_blocks(416, 416), netcfg.reweighting_net_blocks(), replicas=R)
        seeded_init(m, 3001)
        m = m.cuda().train()
        L = m.models[len(m.models) - 1]
        L.seen, L.verbose = 20000, False
        return m, L
    m, L = model()
    params = list(m.parameters())
    opt = FusedSGD(params, **sgd_hyper_parameters(1e-3, 0.9, 5e-4, bs, lr_factor(neg, cs)))
    gs = GraphedTrainStep(m, L, opt, GradAllReducer(m))
    twin, tL = model()
    tparams, tbufs = list(twin.parameters()), dict(twin.named_buffers())
    for k in range(3):                          # eager first step, then capture, then replay
        before = ([p.detach().clone() for p in params], {n: b.detach().clone() for n, b in _bn_stats(m).items()})
        x, metax, mask, tgt = _batch(bs, cs, R, 416, 416, 5100 + k)
        random.seed(5200 + k)
        gs(x, metax, mask, tgt)
        grads = [p.grad.detach().clone() for p in params]
        bn = {n: b.detach().clone() for n, b in _bn_stats(m).items()}
        with torch.no_grad():
            for tp, p0 in zip(tparams, before[0]):
                tp.copy_(p0)
            for n, b0 in before[1].items():
                tbufs[n].copy_(b0)
        for tp in tparams:
            tp.grad = None
        random.seed(5200 + k)
        tL(twin(x, metax, mask), tgt).backward()
        dg = [n for (n, _), g, tp in zip(twin.named_parameters(), grads, tparams) if not bit_equal(g, tp.grad)]
        db = [n for n, b in _bn_stats(twin).items() if not bit_equal(b, bn[n])]
        assert not dg and not db, (k, dg[:3], len(dg), db[:3], len(db))
    assert gs.captures >= 1

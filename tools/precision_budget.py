"""Precision budget of the tensor-core GEMM classes (VERDICT r1 item 3): what does each operand-term mode of the
forward / input-gradient / weight-gradient GEMMs cost in accuracy on the REAL layer shapes, and what does it buy?

    python tools/precision_budget.py [B] [n_cls] [out.json]       (on an H100; default B = 16, n_cls = 20)

One seeded meta-training step (full darknet_dynamic + reweighting_net at 416x416) is evaluated
  * with torch's own float64 kernels on the device (the oracle module in float64) = ground truth,
  * with torch's own float32 kernels (cuDNN / cuBLAS, TF32 off) = what "a float32 implementation" scores,
  * with this build under several term policies (engine.TC_TERMS): 3 = hi*hi + lo*hi + hi*lo, 1 / 2 = one operand
    rounded to fp16, 0 = fp16 x fp16.
For every policy: relative L2 error of the head output, of the loss, and of every parameter gradient against the
float64 truth AND against the all-3 run (same arithmetic except the GEMM under test: isolates the GEMM's own error
from the arg-max-flip lottery), plus the step time of a CUDA-graph replay at B = 64.
The oracle is imported here as the checker only (tools/, not the product).
"""
import contextlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

from fewshot_detection_b200 import netcfg, engine  # noqa: E402
from fewshot_detection_b200.darknet_meta import Darknet  # noqa: E402
from fewshot_detection_b200.optim import FusedSGD  # noqa: E402
from fewshot_detection_b200.distributed import GradAllReducer  # noqa: E402
from fewshot_detection_b200.graph import GraphedTrainStep  # noqa: E402
from seeding import seeded_init, synth_targets, synth_masks  # noqa: E402


def relt(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def batch(B, ncls, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, 416, 416, generator=g)
    metax = torch.rand(ncls, 3, 416, 416, generator=g)
    mask = torch.from_numpy(synth_masks(ncls, 416, seed + 1))
    tgt = torch.from_numpy(synth_targets(B, ncls, seed + 2, max_gt=5))
    return x, metax, mask, tgt


def oracle_run(dtype, x, metax, mask, tgt, seed):
    from oracle import darknet as ODK, region_loss as ORL
    om = ODK.MetaDarknet(netcfg.darknet_dynamic_blocks(), netcfg.reweighting_net_blocks())
    seeded_init(om, seed)
    om = om.to(dtype).cuda().train()
    oo = om(x.to(dtype).cuda(), metax.to(dtype).cuda(), mask.to(dtype).cuda())
    o32 = oo.detach().float().cpu().requires_grad_(True)
    lo = ORL.region_loss_v2(o32, tgt, om.anchors, 5, 1, seen=20000)
    lo.backward()
    oo.backward(o32.grad.to(dtype).cuda())
    out = (oo.detach().double().cpu(), lo.item(), {n: p.grad.detach().double().cpu() for n, p in om.named_parameters()})
    del om, oo
    torch.cuda.empty_cache()
    return out


def our_run(policy, x, metax, mask, tgt, seed):
    engine.TC_TERMS.update(policy)
    with contextlib.redirect_stdout(sys.stderr):
        m = Darknet(netcfg.darknet_dynamic_blocks(), netcfg.reweighting_net_blocks())
    seeded_init(m, seed)
    m = m.cuda().train()
    L = m.loss
    L.verbose = False
    L.seen = 20000
    out = m(x.cuda(), metax.cuda(), mask.cuda())
    loss = L(out, tgt)
    loss.backward()
    torch.cuda.synchronize()
    res = (out.detach().double().cpu(), loss.item(),
           {n: p.grad.detach().contiguous().double().cpu() for n, p in m.named_parameters()})
    del m, out, loss
    torch.cuda.empty_cache()
    return res


def timed_policy(policy, B, ncls, steps=6):
    engine.TC_TERMS.update(policy)
    with contextlib.redirect_stdout(sys.stderr):
        m = Darknet(netcfg.darknet_dynamic_blocks(), netcfg.reweighting_net_blocks())
    seeded_init(m, 0)
    m = m.cuda().train()
    L = m.loss
    L.verbose = False
    L.seen = 20000
    opt = FusedSGD(m.parameters(), lr=1e-6, momentum=0.9, weight_decay=0.48)
    red = GradAllReducer(m)
    gs = GraphedTrainStep(m, L, opt, red)
    b = [t.cuda() for t in batch(B, ncls, 5)]
    for _ in range(3):
        gs(*b)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        gs(*b)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del gs, m, opt, red
    torch.cuda.empty_cache()
    return ms


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    ncls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    outp = sys.argv[3] if len(sys.argv) > 3 else os.path.join(ROOT, 'gpurun_out', 'precision_budget.json')
    seed = 7
    x, metax, mask, tgt = batch(B, ncls, 100)
    o64, l64, g64 = oracle_run(torch.float64, x, metax, mask, tgt, seed)
    o32, l32, g32 = oracle_run(torch.float32, x, metax, mask, tgt, seed)
    names = list(g64.keys())
    conv_names = [n for n in names if g64[n].dim() == 4]

    def summarize(tag, o, l, g, base=None):
        e_out, e_loss = relt(o, o64), abs(l - l64) / abs(l64)
        eg = {n: relt(g[n], g64[n]) for n in names}
        row = {'policy': tag, 'out_vs_f64': e_out, 'loss_vs_f64': e_loss,
               'grad_vs_f64_max': max(eg.values()), 'grad_vs_f64_median': float(np.median(list(eg.values()))),
               'grad_vs_f64_worst_tensor': max(eg, key=eg.get)}
        if base is not None:
            ob, lb, gb = base
            eb = {n: relt(g[n], gb[n]) for n in names}
            row.update(out_vs_all3=relt(o, ob), grad_vs_all3_max=max(eb.values()),
                       grad_vs_all3_median=float(np.median(list(eb.values()))),
                       grad_vs_all3_worst_tensor=max(eb, key=eb.get),
                       convgrad_vs_all3={n: eb[n] for n in conv_names})
        return row

    rows = [summarize('torch float32 (cuDNN, TF32 off)', o32, l32, g32)]
    base = our_run(dict(fwd=3, dgrad=3, wgrad=3, head=3), x, metax, mask, tgt, seed)
    rows.append(summarize('fwd=3 dgrad=3 wgrad=3 (round-1 build)', *base, base=base))
    policies = [
        dict(fwd=3, dgrad=3, wgrad=0, head=3), dict(fwd=3, dgrad=3, wgrad=1, head=3), dict(fwd=3, dgrad=3, wgrad=2, head=3),
        dict(fwd=1, dgrad=3, wgrad=3, head=3), dict(fwd=2, dgrad=3, wgrad=3, head=3), dict(fwd=0, dgrad=3, wgrad=3, head=3),
        dict(fwd=3, dgrad=1, wgrad=3, head=3), dict(fwd=3, dgrad=2, wgrad=3, head=3), dict(fwd=3, dgrad=0, wgrad=3, head=3),
        dict(fwd=1, dgrad=1, wgrad=0, head=3), dict(fwd=2, dgrad=2, wgrad=0, head=3), dict(fwd=0, dgrad=0, wgrad=0, head=0),
        dict(fwd=3, dgrad=3, wgrad=0, head=0),
    ]
    for pol in policies:
        tag = ' '.join('%s=%d' % kv for kv in pol.items())
        rows.append(summarize(tag, *our_run(pol, x, metax, mask, tgt, seed), base=base))
    # step time per policy (CUDA-graph replay, B = 64)
    timing = {}
    for pol in [dict(fwd=3, dgrad=3, wgrad=3, head=3), dict(fwd=3, dgrad=3, wgrad=0, head=3), dict(fwd=1, dgrad=1, wgrad=0, head=3),
                dict(fwd=2, dgrad=2, wgrad=0, head=3), dict(fwd=0, dgrad=0, wgrad=0, head=0)]:
        tag = ' '.join('%s=%d' % kv for kv in pol.items())
        try:
            timing[tag] = timed_policy(pol, 64, ncls)
        except Exception as e:  # keep the accuracy table even if a timing run fails
            timing[tag] = repr(e)
    res = {'B': B, 'n_cls': ncls, 'rows': rows, 'ms_per_step_B64_graph': timing}
    os.makedirs(os.path.dirname(outp), exist_ok=True)
    json.dump(res, open(outp, 'w'), indent=1)
    for r in rows:
        print('%-44s out %.2e loss %.2e | grad vs f64: max %.2e med %.2e (%s) | vs all-3: out %s grad max %s med %s (%s)' % (
            r['policy'], r['out_vs_f64'], r['loss_vs_f64'], r['grad_vs_f64_max'], r['grad_vs_f64_median'],
            r['grad_vs_f64_worst_tensor'], '%.2e' % r['out_vs_all3'] if 'out_vs_all3' in r else '-',
            '%.2e' % r['grad_vs_all3_max'] if 'out_vs_all3' in r else '-',
            '%.2e' % r['grad_vs_all3_median'] if 'out_vs_all3' in r else '-', r.get('grad_vs_all3_worst_tensor', '-')))
    print(json.dumps(timing))


if __name__ == '__main__':
    main()

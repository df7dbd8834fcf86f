"""Worker of tests/test_gpu_replicas_multi.py (one process per rank, launched with torch.distributed.run, world 2):
the replica step of W = 2 ranks x 2 replicas against W = 1 x 4 replicas, neg = 0 (no random row draws).

Every rank takes its images and, through lists.rank_support_rows, its replicas' support rows of the global batch,
runs Darknet(replicas=2) with the bucketed GradAllReducer and its own RegionLossV2, and compares with a local
Darknet(replicas=4) step over the whole batch: the sum of the ranks' losses, the all-reduced gradients and (rank 0)
the running statistics of replica 0.  NCCL when every rank has a GPU of its own, gloo with both ranks on one GPU
otherwise.  Prints 'REPLICA_MULTI_OK rank r' on success."""
import contextlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

TOL = 1e-3


def relt(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    own_gpu = torch.cuda.device_count() >= world
    dev = torch.device('cuda', local if own_gpu else 0)
    torch.cuda.set_device(dev)
    if own_gpu:
        dist.init_process_group('nccl', device_id=dev)
    else:
        dist.init_process_group('gloo')
    from fewshot_detection_b200 import netcfg, lists as LS
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.distributed import GradAllReducer
    from seeding import seeded_init, synth_targets, synth_masks
    cfg.neg_ratio = 0
    det, ler = netcfg.mini_dynamic_blocks(128, 4), netcfg.mini_reweighting_blocks(64, 4, 128)
    R, bs = 4, 8
    per = R // world

    def model(replicas):
        with contextlib.redirect_stdout(sys.stderr):
            m = Darknet([dict(b) for b in det], [dict(b) for b in ler], replicas=replicas)
        seeded_init(m, 3)
        m = m.to(dev).train()
        L = m.models[len(m.models) - 1]
        L.verbose, L.seen = False, 20000
        return m, L

    cs = int(model(1)[1].num_classes)
    errs = {}
    for seed in (11, 12, 13):
        g = torch.Generator().manual_seed(seed)
        x = torch.rand(bs, 3, 128, 128, generator=g).to(dev)
        metax = torch.rand(R * cs, 3, 64, 64, generator=g).to(dev)
        mask = torch.from_numpy(synth_masks(R * cs, 64, seed + 1)).to(dev)
        tgt = torch.from_numpy(synth_targets(bs, cs, seed + 2, max_gt=3))
        tgt[0] = tgt[bs // 2] = 0            # every rank's shard has labelled rows and empty ones for neg = 0 to drop
        # this rank: images of its replicas, support rows of its replicas (as the driver takes them from the index)
        rows = torch.tensor(LS.rank_support_rows(list(range(R * cs)), cs, R, world, rank), device=dev)
        assert rows.tolist() == list(range(rank * per * cs, (rank + 1) * per * cs))
        q = slice(rank * bs // world, (rank + 1) * bs // world)
        m, L = model(per)
        red = GradAllReducer(m)
        assert red.world == world
        red.begin_step()
        loss = L(m(x[q], metax[rows], mask[rows]), tgt[q])
        loss.backward()
        red.finish()
        total = loss.detach().reshape(1).clone()
        dist.all_reduce(total)
        # one process, four replicas, one loss over the whole batch
        om, oL = model(R)
        oloss = oL(om(x, metax, mask), tgt)
        oloss.backward()
        torch.cuda.synchronize()
        assert abs(total.item() - oloss.item()) <= TOL * abs(oloss.item()), (seed, total.item(), oloss.item())
        if rank == 0:
            for (n, b), ob in zip(m.named_buffers(), om.buffers()):
                if n.endswith(('running_mean', 'running_var')):
                    assert relt(b, ob) < TOL, (seed, n, relt(b, ob))
        for (n, p), op in zip(m.named_parameters(), om.parameters()):
            errs.setdefault(n, []).append(relt(p.grad, op.grad))
        del m, om, red
    worst = {n: float(np.median(v)) for n, v in errs.items()}
    assert max(worst.values()) < TOL, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    dist.barrier()
    print('REPLICA_MULTI_OK rank %d (%s) worst median gradient error %.2e' % (rank, 'nccl' if own_gpu else 'gloo, one GPU',
                                                                            max(worst.values())), flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()

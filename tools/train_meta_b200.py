#!/usr/bin/env python
"""Command-line front end with the reference driver's arguments (train_meta.py:1-6):

    python tools/train_meta_b200.py datacfg darknetcfg learnetcfg weightfile            # one GPU
    torchrun --nproc-per-node 8 tools/train_meta_b200.py datacfg darknetcfg learnetcfg weightfile

The `.data` file drives everything as in the reference: `train` (image list or class dict), `meta` (support dict),
`novel` / `novelid` (base / novel split), `neg`, `tuning` (+ `max_epoch`, `repeat`, `dynamic`) - the image list comes
from lists.build_dataset, the support index from lists.support_index, the step from trainer.MetaTrainer (CUDA-graph
replay, one graph per multi-scale input size).  Under torchrun every rank builds the same lists with the same seeds,
takes its slice of each global batch, and rank 0's parameters are broadcast once before the first step.
A trained weight file is scored by tools/valid_ensemble_b200.py (valid_ensemble.py + scripts/voc_eval.py).  Opt-in,
every checkpoint is scored the same way while training runs, sharded over the ranks (valid.score_batches):

    --eval-devkit DIR [--eval-year Y]      VOC AP on the `valid` list: one line with mean, base and novel AP
    --eval-coco-annotations JSON           COCO box AP on the `valid` list: one line with AP, AP50, AP75
    --eval-base-rw PATH                    with either: the base classes detected with the rows of a stored vectors
                                           file (the evaluation command's --base-rw)

with the support set, batch sizes and thresholds of the evaluation command.  Opt-in as well, resuming exactly
(fewshot_detection_b200/resume.py):

    --save-state                           every checkpoint also writes backup/%06d.state beside %06d.weights: momentum,
                                           schedule position, both `seen` counters, every rank's random streams (only the
                                           newest state file the run wrote is kept)
    --resume PATH.state                    continue from that state; `weightfile` must be its paired weight file.  Every
                                           check (file, version, weight checksum, world, replicas, batch, cfg, .data,
                                           training list) is made before any CUDA work

Opt-in, the reference's own step on any number of GPUs (its configs train 4 nn.DataParallel replicas, `gpus=1,2,3,4`):

    --replicas R                           R replicas per global step, R / world on each rank: BatchNorm statistics per
                                           replica (batch / R query images, n_cls support images), R support sets per
                                           step from the support index built for R GPUs, replica r's images reweighted
                                           by replica r's vectors.  R must be a multiple of the world size and divide
                                           the global batch.  Without it each rank is one replica.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def read_list(path):
    with open(path, 'r') as f:
        return [l.rstrip() for l in f.readlines() if l.strip()]


def broadcast_parameters(model, src=0):
    """Identical replicas: the gradient all-reduce keeps replicas in sync only if they START in sync.  A weight file
    may initialise just the trunk (darknet19_448.conv.23 stops after 23 layers, darknet_meta.py:367-368), every other
    tensor is per-process random - so rank `src`'s parameters and BN buffers are broadcast once."""
    import torch.distributed as dist
    with torch.no_grad():
        for t in list(model.parameters()) + list(model.buffers()):
            dist.broadcast(t.data, src)
        chk = torch.stack([p.detach().double().sum() for p in model.parameters()]).sum().reshape(1)
        ref = chk.clone()
        dist.broadcast(ref, src)
        if not torch.equal(chk, ref):
            raise RuntimeError('replicas differ after the parameter broadcast')


def checkpoint_evaluator(data_options, devkit, year, coco_annotations, world, rank, batch_size=64, support_batch=64,
                         base_rw=None):
    """evaluate(model, epoch) for MetaTrainer: the evaluation command's pass over `valid`, this rank's shard of it;
    returns the line rank 0 logs.  base_rw: stored vectors (valid.load_reweighting_vectors) whose rows replace those
    of the base classes, cfg._real_base_ids, as the evaluation command's --base-rw does."""
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.dataset import DetectionBatcher, MetaBatcher
    from fewshot_detection_b200.shard import rank0_first, shard_range
    from fewshot_detection_b200 import lists as LS, valid as VA, voc_eval as VE, coco_eval as CE
    classes, novel = list(cfg.classes), list(cfg.novel_classes)
    metalines, inds = LS.support_index(data_options['meta'], classes, 0, ensemble=True)
    lines = read_list(data_options['valid'])
    imgids = [os.path.basename(l).split('.')[0] for l in lines]
    if coco_annotations is not None:
        proto = CE.DeviceCocoEval(classes, imgids, CE.load_coco_annotations(coco_annotations, imgids, classes))
        result_kwargs = dict(novel_classes=novel)
    else:
        voc = os.path.join(devkit, 'VOC' + year)
        names = read_list(os.path.join(voc, 'ImageSets', 'Main', 'test.txt'))
        load = lambda: VE.load_annotations(os.path.join(voc, 'Annotations', '{}.xml'), names,
                                           os.path.join(devkit, 'annotations_cache'))
        recs = rank0_first(load) if world > 1 else load()  # rank 0 writes the cache, the others read it
        proto = VE.DeviceVocEval(classes, names, recs)
        result_kwargs = dict(use_07_metric=int(year) < 2010, novel_classes=novel)
    s0, s1 = shard_range(len(inds), support_batch, world, rank)
    q0, q1 = shard_range(len(lines), batch_size, world, rank)
    if base_rw is not None:
        result_kwargs.update(base_rw=base_rw, base_rows=list(cfg._real_base_ids))

    def evaluate(model, epoch):
        mb = MetaBatcher(metalines, inds, classes=classes, train=False, ensemble=True, with_ids=True)
        meta = (mb.batch(range(s, min(s + support_batch, s1))) for s in range(s0, s1, support_batch))
        db = DetectionBatcher(lines, shape=(model.width, model.height), shuffle=False, train=False, batch_size=batch_size)

        def images():
            for s in range(q0, q1, batch_size):
                idx = range(s, min(s + batch_size, q1))
                yield db.batch(idx)[0], [imgids[i] for i in idx], [db._entry(i).size() for i in idx]
        r = VA.score_batches(model, meta, images(), proto.empty_like(), sharded=world > 1, **result_kwargs)
        if coco_annotations is not None:
            return 'COCO AP %.4f AP50 %.4f AP75 %.4f' % tuple(r['all'][:3])
        fmt = lambda v: 'n/a' if v is None else '%.4f' % v
        return 'mAP %s base %s novel %s' % (fmt(r['mean']), fmt(r['mean_base']), fmt(r['mean_novel']))
    return evaluate


def main():
    import argparse
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument('args', nargs='*')
    ap.add_argument('--eval-devkit', default=None)
    ap.add_argument('--eval-year', default='2007')
    ap.add_argument('--eval-coco-annotations', default=None)
    ap.add_argument('--eval-base-rw', default=None)
    ap.add_argument('--save-state', action='store_true')
    ap.add_argument('--resume', default=None)
    ap.add_argument('--replicas', type=int, default=None)
    opts = ap.parse_args()
    scored = opts.eval_devkit is not None or opts.eval_coco_annotations is not None
    if len(opts.args) != 4 or (opts.eval_devkit is not None and opts.eval_coco_annotations is not None) or \
            (opts.eval_base_rw is not None and not scored):
        if opts.eval_base_rw is not None and not scored:
            print('--eval-base-rw needs --eval-devkit or --eval-coco-annotations')
        print('Usage:')
        print('python tools/train_meta_b200.py datacfg darknetcfg learnetcfg weightfile '
              '[--eval-devkit DIR [--eval-year Y] | --eval-coco-annotations JSON] [--eval-base-rw PATH] '
              '[--save-state] [--resume PATH.state] [--replicas R]')
        return 1
    if opts.eval_base_rw is not None and not os.path.isfile(opts.eval_base_rw):
        print('--eval-base-rw: no such file: %s' % opts.eval_base_rw)
        return 1
    argv = [sys.argv[0]] + opts.args
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.utils import read_data_cfg, logging
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.distributed import GradAllReducer
    from fewshot_detection_b200.dataset import DetectionBatcher, MetaBatcher
    from fewshot_detection_b200 import trainer as T, lists as LS, resume as R
    import torch.distributed as dist

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if opts.replicas is not None and (opts.replicas < 1 or opts.replicas % world):
        print('--replicas %d: the replicas must be a positive multiple of the world size %d' % (opts.replicas, world))
        return 1
    resume_state = None
    if opts.resume is not None:           # every check on the state file is made before any CUDA work
        try:
            resume_state = R.read_state(opts.resume)
            R.check_weights(resume_state, opts.resume, argv[4])
        except R.StateFileError as e:
            print('--resume: %s' % e)
            return 1

    data_options = read_data_cfg(argv[1])
    darknetcfg, learnetcfg = parse_cfg(argv[2]), parse_cfg(argv[3])
    net_options, meta_options = darknetcfg[0], learnetcfg[0]
    cfg.config_data(data_options)
    cfg.config_meta(meta_options)
    cfg.config_net(net_options)
    batch_size = int(net_options['batch'])                      # GLOBAL batch, as in the reference
    per_rank = batch_size // world
    replicas = world if opts.replicas is None else opts.replicas
    if batch_size % replicas:
        print('--replicas %d: the global batch %d does not split into %d replicas' % (replicas, batch_size, replicas))
        return 1
    steps = [float(s) for s in net_options['steps'].split(',')]
    scales = [float(s) for s in net_options['scales'].split(',')]
    base_rw = None
    if opts.eval_base_rw is not None:             # checked against the model before training starts
        from fewshot_detection_b200 import valid as VA
        base_rw = VA.load_reweighting_vectors(opts.eval_base_rw, VA.reweighting_vector_shapes(learnetcfg, len(cfg.classes)))
    fingerprint = lambda trainlist=None: R.fingerprint(darknetcfg, learnetcfg, data_options, world, batch_size, per_rank,
                                                       trainlist, replicas)
    if resume_state is not None:
        try:
            R.check_fingerprint(resume_state, opts.resume, fingerprint())
        except R.StateFileError as e:
            print('--resume: %s' % e)
            return 1

    if resume_state is not None:
        seed = int(resume_state['seed'])     # the stored seed rebuilds the training list; the streams are restored below
    else:
        seed = int(os.environ.get('FSDET_SEED', str(int.from_bytes(os.urandom(4), 'little')) if world == 1 else '0'))
    import random
    random.seed(seed)                 # every rank must build the same lists and draw the same sizes
    np.random.seed(seed % (2 ** 32))
    torch.manual_seed(seed)           # train_meta.py:79; unseeded, torch's CPU generator starts from a per-process seed
    trainlist = LS.build_dataset(data_options)
    nsamples = len(trainlist)
    if resume_state is not None:
        try:
            R.check_fingerprint(resume_state, opts.resume, fingerprint(trainlist))
        except R.StateFileError as e:
            print('--resume: %s' % e)
            return 1

    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))

    model = Darknet(darknetcfg, learnetcfg, replicas=replicas // world)
    if opts.replicas is not None and rank == 0:
        logging('%d replicas per step, %d per rank on %d rank(s): %d query images and %d support images per replica'
                % (replicas, replicas // world, world, batch_size // replicas, len(cfg.base_classes)))
    if os.path.exists(argv[4]):
        model.load_weights(argv[4])
    else:
        logging('weight file %s not found: training from the random initialisation' % argv[4])
    model = model.cuda()
    if world > 1:
        broadcast_parameters(model)
    classes = cfg.base_classes
    factor = T.lr_factor(cfg.neg_ratio, len(classes))
    hp = T.sgd_hyper_parameters(float(net_options['learning_rate']), float(net_options['momentum']), float(net_options['decay']),
                                batch_size, factor)
    optimizer = FusedSGD(model.parameters(), **hp)
    reducer = GradAllReducer(model) if world > 1 else None

    processed, init_epoch, max_epochs = T.epoch_plan(model.seen, nsamples, batch_size, int(net_options['max_batches']),
                                                     cfg.tuning, cfg.get('max_epoch'), cfg.repeat)
    backupdir = cfg.get('backup') or data_options.get('backup', 'backup')     # cfg.py:133-145 names it after the run's switches
    if rank == 0 and not os.path.exists(backupdir):
        os.makedirs(backupdir)

    def make_train_batcher(seen):
        # every rank walks the same shuffled list and takes its own slice of each global batch
        lines = trainlist if world == 1 else \
            [trainlist[i] for b in range(0, nsamples - batch_size + 1, batch_size) for i in range(b + rank * per_rank, b + (rank + 1) * per_rank)]
        return DetectionBatcher(lines, shape=(model.width, model.height), shuffle=False, train=True, seen=seen,
                                batch_size=per_rank, seen_step=world)

    def make_meta_batcher():
        if opts.replicas is None:
            cfg.num_gpus = 1          # one process per GPU: each rank draws its own n_cls support images per step
            metalines, inds = LS.support_index(data_options['meta'], classes, LS.support_batches_per_epoch(train=True),
                                               shuffle=cfg.randmeta)
            return MetaBatcher(metalines, inds, classes=classes, train=True)
        cfg.num_gpus = replicas       # the reference's index for `replicas` GPUs; every rank takes its replicas' rows
        metalines, inds = LS.support_index(data_options['meta'], classes, LS.support_batches_per_epoch(train=True),
                                           shuffle=cfg.randmeta)
        inds = LS.rank_support_rows(inds, len(classes), replicas, world, rank)
        return MetaBatcher(metalines, inds, classes=classes, train=True, replicas=replicas // world)

    evaluate = None
    if opts.eval_devkit is not None or opts.eval_coco_annotations is not None:
        state = random.getstate(), np.random.get_state()          # the training lists' draws stay as without it
        evaluate = checkpoint_evaluator(data_options, opts.eval_devkit, opts.eval_year, opts.eval_coco_annotations,
                                        world, rank, base_rw=base_rw)
        random.setstate(state[0])
        np.random.set_state(state[1])
    tr = T.MetaTrainer(model, optimizer, float(net_options['learning_rate']) / factor, batch_size, steps, scales,
                       make_train_batcher, make_meta_batcher, backupdir=backupdir if rank == 0 else None,
                       save_interval=cfg.save_interval, reducer=reducer, world=world, processed_batches=processed,
                       log=logging if rank == 0 else (lambda *_: None), evaluate=evaluate,
                       save_state=R.state_saver(fingerprint(trainlist), seed, world, rank, logging) if opts.save_state else None)
    model.loss.verbose = rank == 0
    if resume_state is not None:
        R.restore(tr, resume_state, rank)    # last: it sets this rank's random generators
        if rank == 0:
            logging('resumed from %s at epoch %d, processed %d batches' % (opts.resume, tr.epoch, tr.processed_batches))
    tr.fit(init_epoch, max_epochs)
    if world > 1:
        if tr.graphed is not None:
            tr.graphed.entries.clear()      # graphs that captured NCCL work go before their communicator
        import gc
        gc.collect()
        torch.cuda.synchronize()
        dist.destroy_process_group()
    return 0


if __name__ == '__main__':
    sys.exit(main())

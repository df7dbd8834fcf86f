#!/usr/bin/env python
"""Evaluation command: the reference README's two evaluation steps (valid_ensemble.py, then scripts/voc_eval.py) in
one run, with the detections scored on the GPU where decode and NMS leave them.

    python tools/valid_ensemble_b200.py datacfg darknetcfg learnetcfg weightfile [--devkit DIR] [--write-results]
                                        [--coco-annotations instances_val2014.json] [--write-coco-results PATH]
                                        [--base-rw PATH] [--save-rw PATH] [--tta-sides 416,544,608] [--tta-flip]

The `.data` file is read as tools/train_meta_b200.py reads it: `valid` (image list), `meta` (support dictionary), the
class list and the `novel` / `novelid` split.  The support images of every class are run through the reweighting net
and averaged per class (valid_ensemble.py:86-100); every image of `valid` is detected with those vectors
(conf_thresh 0.005, NMS 0.45).  Image ids are file basenames and sizes come from the image headers, as in the
reference.

--devkit DIR       DIR/VOC<year>/Annotations/<id>.xml and DIR/VOC<year>/ImageSets/Main/test.txt (annotations cached
                   in DIR/annotations_cache as scripts/voc_eval.py does): prints the AP per class and the mean, base
                   and novel mean AP (VOC07 11-point metric for years before 2010, as the reference).
--write-results    writes the reference's result files results/<backup>/ene<ckpt>/comp4_det_test_<class>.txt.
--coco-annotations JSON
                   scores the detections with the COCO box metric (coco_eval.DeviceCocoEval) against an
                   instances_*.json whose images[].file_name stems are the image ids: prints pycocotools' twelve summary
                   lines for all, base and novel classes, and the AP@[.5:.95] of each class.
--write-coco-results PATH
                   writes the standard COCO results json of the same detections (with --coco-annotations).
--base-rw PATH     the reference's `use_baserw` mode (valid_ensemble.py:108-119): after the ensemble, the rows of the
                   base classes (the classes that are not novel) are replaced by those of the stored vectors in PATH,
                   so that after k-shot fine-tuning the base classes are detected with vectors averaged over a large
                   support set while the novel classes keep their k-shot ones.  The reference reads
                   data/rws/voc_novel0_.pkl; here the path is always given.  The file is checked against the model
                   before the model is built.  Result files go to results/<backup>/ene_<ckpt>.
--save-rw PATH     writes the ensembled vectors before any substitution, in the reference's format (a pickled list
                   of one float32 [n_cls, C, 1, 1] numpy array per dynamic layer, rows in class-list order): the file
                   --base-rw reads, e.g. from a run whose `meta` is the full support dictionary.  Alone, only the
                   support pass runs.

--tta-sides S1,S2,...
                   test-time augmentation (TTA): every query batch is detected at each side (multiples of 32, no
                   repeats); the candidates of all passes are merged per image and class and suppressed by one NMS on
                   the device (valid.detect_tta).  Result files go to results/<backup>/ene<ckpt>_tta (ene_<ckpt>_tta
                   with --base-rw), so they never overwrite single-pass results.  No AP gain is claimed for it.
--tta-flip         TTA: adds the mirrored image of each side (alone: at the network's side), its boxes mirrored back.

Ranking differs from the reference's file-based evaluation only for detections whose printed confidences tie: they
keep result-file order here (voc_eval.DeviceVocEval).

Under `torchrun --nproc-per-node N` every process takes the GPU of its LOCAL_RANK and a contiguous block of whole
support and query batches (shard.shard_range); the support vectors and the detection pools are gathered in rank order,
so the printed numbers and the written files are those of one process, bit for bit.  Only rank 0 prints and writes.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def read_list(path):
    with open(path, 'r') as f:
        return [l.rstrip() for l in f.readlines() if l.strip()]


def result_prefix(weightfile, base_rw=False, tta=False):
    """valid_ensemble.py:15-22: results/<directory of the weight file>/ene<weight file stem>, ene_<stem> with stored
    base-class vectors; `_tta` appended under a test-time augmentation plan."""
    ckpt = os.path.basename(weightfile).split('.')[0]
    backup = os.path.basename(os.path.dirname(os.path.abspath(weightfile)))
    return os.path.join('results', backup, ('ene_' if base_rw else 'ene') + ckpt + ('_tta' if tta else ''))


def load_base_rw(path, datacfg, learnetcfg):
    """The stored vectors of --base-rw, checked against the class list and reweighting net of the cfgs."""
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.utils import read_data_cfg
    from fewshot_detection_b200 import valid as VA
    cfg.config_data(read_data_cfg(datacfg))
    return VA.load_reweighting_vectors(path, VA.reweighting_vector_shapes(parse_cfg(learnetcfg), len(cfg.classes)))


def tta_plan_of(ap, args):
    """The test-time augmentation plan of --tta-sides / --tta-flip (None without them); bad sides end the command."""
    if args.tta_sides is None and not args.tta_flip:
        return None
    from fewshot_detection_b200.cfg import parse_cfg
    from fewshot_detection_b200 import valid as VA
    try:
        if args.tta_sides is not None:
            sides = VA.parse_tta_sides(args.tta_sides)
        else:
            if not os.path.isfile(args.darknetcfg):
                ap.error('no such file: %s' % args.darknetcfg)
            sides = [int(parse_cfg(args.darknetcfg)[0]['width'])]
        return VA.tta_plan(sides, args.tta_flip)
    except ValueError as e:
        ap.error('--tta-sides: %s' % e)


def parse_args(argv=None):
    """The checked arguments and the --base-rw vectors (None without it), before any GPU work."""
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('datacfg')
    ap.add_argument('darknetcfg')
    ap.add_argument('learnetcfg')
    ap.add_argument('weightfile')
    ap.add_argument('--devkit', default=None, help='VOCdevkit directory: score the detections against its annotations')
    ap.add_argument('--year', default='2007')
    ap.add_argument('--write-results', action='store_true', help='write the per-class result files')
    ap.add_argument('--coco-annotations', default=None, help='instances_*.json: score with the COCO box metric')
    ap.add_argument('--write-coco-results', default=None, help='COCO results json to write (with --coco-annotations)')
    ap.add_argument('--batch-size', type=int, default=64, help='query images per forward')
    ap.add_argument('--support-batch', type=int, default=64, help='support images per reweighting-net forward')
    ap.add_argument('--base-rw', default=None, help='stored vectors file: detect the base classes with its rows')
    ap.add_argument('--save-rw', default=None, help='write the ensembled vectors to this file')
    ap.add_argument('--tta-sides', default=None, help='test-time augmentation: comma-separated sides, multiples of 32')
    ap.add_argument('--tta-flip', action='store_true', help='test-time augmentation: add the mirrored pass of each side')
    args = ap.parse_args(argv)
    if args.devkit is None and not args.write_results and args.coco_annotations is None and args.save_rw is None:
        ap.error('nothing to do: give --devkit, --coco-annotations, --write-results and/or --save-rw')
    if args.coco_annotations is not None and args.devkit is not None:
        ap.error('--devkit and --coco-annotations score the same detections twice: give one')
    if args.write_coco_results is not None and args.coco_annotations is None:
        ap.error('--write-coco-results needs --coco-annotations (the COCO image and category ids)')
    if args.coco_annotations is not None and args.write_results:
        ap.error('--write-results writes the VOC result files; with --coco-annotations use --write-coco-results')
    args.tta = tta_plan_of(ap, args)
    base_rw = None
    if args.base_rw is not None:                      # a bad file fails here, before the support pass
        if not os.path.isfile(args.base_rw):
            ap.error('--base-rw: no such file: %s' % args.base_rw)
        try:
            base_rw = load_base_rw(args.base_rw, args.datacfg, args.learnetcfg)
        except (OSError, ValueError) as e:
            ap.error('--base-rw: %s' % e)
    if args.save_rw is not None:
        os.makedirs(os.path.dirname(os.path.abspath(args.save_rw)), exist_ok=True)
    return args, base_rw


def main(argv=None):
    args, base_rw = parse_args(argv)
    import torch

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if world > 1:
        import torch.distributed as dist
        local = int(os.environ['LOCAL_RANK'])
        torch.cuda.set_device(local)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
        try:
            return run(args, world, dist.get_rank(), base_rw)
        finally:
            torch.cuda.synchronize()
            dist.destroy_process_group()
    torch.cuda.set_device(0)
    return run(args, 1, 0, base_rw)


def run(args, world, rank, base_rw=None):
    """The evaluation on this process's shard (the whole set when world == 1); `base_rw` are the stored vectors of
    --base-rw (load_base_rw)."""
    import torch
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.utils import read_data_cfg, logging
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.dataset import DetectionBatcher, MetaBatcher
    from fewshot_detection_b200.shard import rank0_first, shard_range
    from fewshot_detection_b200 import coco_eval as CE, lists as LS, valid as VA, voc_eval as VE
    sharded, lead = world > 1, rank == 0
    data_options = read_data_cfg(args.datacfg)
    darknetcfg, learnetcfg = parse_cfg(args.darknetcfg), parse_cfg(args.learnetcfg)
    cfg.config_data(data_options)
    cfg.config_meta(learnetcfg[0])
    cfg.config_net(darknetcfg[0])
    classes = list(cfg.classes)
    novel = list(cfg.novel_classes)

    m = Darknet(darknetcfg, learnetcfg)
    m.load_weights(args.weightfile)
    m = m.cuda().eval()

    metalines, inds = LS.support_index(data_options['meta'], classes, 0, ensemble=True)
    mb = MetaBatcher(metalines, inds, classes=classes, train=False, ensemble=True, with_ids=True)
    s0, s1 = shard_range(len(inds), args.support_batch, world, rank)
    meta_batches = (mb.batch(range(s, min(s + args.support_batch, s1))) for s in range(s0, s1, args.support_batch))

    lines = read_list(data_options['valid'])
    db = DetectionBatcher(lines, shape=(m.width, m.height), shuffle=False, train=False, batch_size=args.batch_size)
    imgids = [os.path.basename(l).split('.')[0] for l in lines]

    q0, q1 = shard_range(len(lines), args.batch_size, world, rank)

    def image_batches():
        for s in range(q0, q1, args.batch_size):
            idx = range(s, min(s + args.batch_size, q1))
            data = db.batch(idx)[0] if args.tta is None else VA.tta_inputs(db, idx, args.tta)
            yield data, [imgids[i] for i in idx], [db._entry(i).size() for i in idx]

    def detect(data):
        if args.tta is None:
            return VA.detect(m, data, dw, n_cls)
        return VA.detect_tta(m, data, dw, n_cls, args.tta)

    out = None                                        # result files: VOC per class, or the COCO results json
    if args.write_results and not lead:
        out = True                                    # this rank's lines go to rank 0
    elif args.write_results:
        prefix = result_prefix(args.weightfile, base_rw is not None, args.tta is not None)
        if not os.path.exists(prefix):
            os.makedirs(prefix)
        logging('saving to: %s' % prefix)
        out = [open(os.path.join(prefix, 'comp4_det_test_%s.txt' % c), 'w') for c in classes]
    rw = dict(base_rw=base_rw, base_rows=list(cfg._real_base_ids) if base_rw is not None else None, save_rw=args.save_rw)
    try:
        if args.devkit is None and args.coco_annotations is None:
            n_cls = len(classes)
            dw = VA.evaluation_dynamic_weights(m, meta_batches, n_cls, sharded, **rw)
            if not args.write_results:                # --save-rw alone: the support pass only
                return 0
            if not sharded:
                for data, ids, sizes in image_batches():
                    VA.write_detections(out, detect(data), ids, sizes, n_cls)
                return 0
            mine = dict((i, []) for i in range(n_cls))
            for data, ids, sizes in image_batches():
                for i, l in VA.detection_lines(detect(data), ids, sizes, n_cls).items():
                    mine[i].extend(l)
            parts = VA.gather_to(mine, None, 0)
            if lead:
                for part in parts:
                    for i in range(n_cls):
                        out[i].writelines(part[i])
            return 0
        if args.coco_annotations is not None:
            ev = CE.DeviceCocoEval(classes, imgids, CE.load_coco_annotations(args.coco_annotations, imgids, classes))
            if args.write_coco_results:
                out = open(args.write_coco_results, 'w') if lead else True
            result_kwargs = dict(novel_classes=novel)
        else:
            voc = os.path.join(args.devkit, 'VOC' + args.year)
            imagenames = read_list(os.path.join(voc, 'ImageSets', 'Main', 'test.txt'))
            load = lambda: VE.load_annotations(os.path.join(voc, 'Annotations', '{}.xml'), imagenames,
                                               os.path.join(args.devkit, 'annotations_cache'))
            recs = rank0_first(load) if sharded else load()    # rank 0 writes the cache, the others read it
            ev = VE.DeviceVocEval(classes, imagenames, recs)
            result_kwargs = dict(use_07_metric=int(args.year) < 2010, novel_classes=novel)
        r = VA.score_batches(m, meta_batches, image_batches(), ev, out, sharded, tta=args.tta, **rw, **result_kwargs)
    finally:
        for f in out if isinstance(out, list) else [out]:
            if f is not None and f is not True:
                f.close()
    if not lead:
        return 0
    if args.coco_annotations is not None:
        print_coco(r, classes, novel)
        return 0
    print_voc(r, classes, novel, result_kwargs['use_07_metric'])
    return 0


def print_voc(r, classes, novel, use_07_metric):
    """scripts/voc_eval.py's lines: the AP of each class, then the mean, base and novel mean AP."""
    print('VOC07 metric? ' + ('Yes' if use_07_metric else 'No'))
    for c in classes:
        print('AP for {} = {:.4f}{}'.format(c, r['ap'][c], ' (novel)' if c in novel else ''))
    print('Mean AP = {:.4f}'.format(r['mean']))
    if r['mean_base'] is not None and novel:
        print('Mean Base AP = {:.4f}'.format(r['mean_base']))
    if r['mean_novel'] is not None:
        print('Mean Novel AP = {:.4f}'.format(r['mean_novel']))


def print_coco(r, classes, novel):
    """The summary lines as pycocotools prints them, for all, base and novel classes, then the AP of each class."""
    from fewshot_detection_b200 import coco_eval as CE
    for title, key in (('all classes', 'all'), ('base classes', 'base'), ('novel classes', 'novel')):
        if r[key] is None:
            continue
        print('COCO box metric, %s:' % title)
        for line in CE.format_stats(r[key]):
            print(line)
    for c in classes:
        print('AP for {} = {:.4f}{}'.format(c, r['ap'][c], ' (novel)' if c in novel else ''))


if __name__ == '__main__':
    sys.exit(main())

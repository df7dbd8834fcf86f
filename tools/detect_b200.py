#!/usr/bin/env python
"""Detection command: the boxes of the meta detector in any images, one text file (and optionally one drawn image) per
image.

    python tools/detect_b200.py darknetcfg learnetcfg weightfile IMAGES... \\
           (--rw vectors.pkl --names classes.names | --data datacfg) \\
           [--conf 0.5] [--nms 0.4] [--max-det 100] [--batch-size 64] [--out DIR] [--draw]
           [--tta-sides 416,544,608] [--tta-flip]

IMAGES are image files, directories (their .jpg / .jpeg / .png files, sorted) or .txt lists of image paths.

The reweighting vectors come from one of:
--rw PATH --names FILE  a vectors file (valid.save_reweighting_vectors, or the evaluation command's --save-rw) and the
                        class names of its rows, one per line.  The file is checked against the reweighting net of
                        the cfgs and against the number of names before the model is built.
--data DATACFG          ensembled over the `.data` file's `meta` support dictionary, as the evaluation command does;
                        the classes are the `.data` file's.

Every image is decoded on the host and resized on the device to the network's input size (the evaluation's plain
resize); a batch is detected, decoded, suppressed (conf 0.5 and NMS 0.4 by default, the reference's do_detect) and
reduced on the device to the max_det best boxes of each image over all classes, replayed as one CUDA graph per batch
size.  Outputs in --out (default `detections`):
  <stem>.txt   one line per box, best first: `class prob x1 y1 x2 y2` (pixels of the original image, floats printed so
               that they read back exactly; the class name may contain spaces, the last five fields never do)
  <stem>.jpg   with --draw: the original image with one rectangle and label per box, one colour per class.

Test-time augmentation (TTA): --tta-sides S1,S2,... runs every batch at each side (multiples of 32, no repeats) and
--tta-flip adds the mirrored image of each side (alone: at the network's side); the candidates of all passes are merged
per image and class, the mirrored boxes mirrored back, and suppressed by one NMS on the device (valid.detect_tta).
The outputs then go to `<out>_tta`, so they never overwrite single-pass results.  A TTA plan runs eagerly (no CUDA
graph).  Whether it improves the boxes of a given model is for the user to measure.
One GPU (cuda:0).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

IMAGE_EXTS = ('.jpg', '.jpeg', '.png')


def list_images(items):
    """Image paths of the IMAGES arguments, in order: files as given, directories' image files sorted, .txt lists."""
    out = []
    for item in items:
        if os.path.isdir(item):
            out.extend(os.path.join(item, f) for f in sorted(os.listdir(item)) if f.lower().endswith(IMAGE_EXTS))
        elif item.lower().endswith('.txt'):
            with open(item, 'r') as f:
                out.extend(l.strip() for l in f if l.strip())
        else:
            out.append(item)
    return out


def parse_args(argv=None):
    """The checked arguments, the class names, the --rw vectors (None with --data) and the image paths, before any
    CUDA work."""
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('darknetcfg')
    ap.add_argument('learnetcfg')
    ap.add_argument('weightfile')
    ap.add_argument('images', nargs='+', metavar='IMAGES')
    ap.add_argument('--rw', default=None, help='reweighting vectors file (with --names)')
    ap.add_argument('--names', default=None, help='class names of the vectors file, one per line')
    ap.add_argument('--data', default=None, help='.data file: ensemble the vectors over its support dictionary')
    ap.add_argument('--conf', type=float, default=0.5, help='confidence threshold (det_conf * cls_conf)')
    ap.add_argument('--nms', type=float, default=0.4, help='NMS IoU threshold')
    ap.add_argument('--max-det', type=int, default=100, help='boxes kept per image, over all classes')
    ap.add_argument('--batch-size', type=int, default=64, help='images per forward')
    ap.add_argument('--support-batch', type=int, default=64, help='support images per reweighting-net forward (--data)')
    ap.add_argument('--out', default='detections', help='output directory')
    ap.add_argument('--draw', action='store_true', help='also write each image with its boxes drawn')
    ap.add_argument('--eager', action='store_true', help='launch every kernel instead of replaying a CUDA graph')
    ap.add_argument('--tta-sides', default=None, help='test-time augmentation: comma-separated sides, multiples of 32')
    ap.add_argument('--tta-flip', action='store_true', help='test-time augmentation: add the mirrored pass of each side')
    args = ap.parse_args(argv)
    if (args.rw is None) == (args.data is None):
        ap.error('give the vectors either as --rw PATH --names FILE or as --data DATACFG')
    if args.rw is not None and args.names is None:
        ap.error('--rw needs --names: the class of each row of the vectors')
    if args.data is not None and args.names is not None:
        ap.error('--names goes with --rw; with --data the classes are the .data file\'s')
    if args.max_det < 1 or args.batch_size < 1:
        ap.error('--max-det and --batch-size must be positive')
    for path in (args.darknetcfg, args.learnetcfg, args.weightfile, args.rw, args.names, args.data):
        if path is not None and not os.path.isfile(path):
            ap.error('no such file: %s' % path)
    from fewshot_detection_b200.cfg import parse_cfg
    from fewshot_detection_b200.utils import load_class_names
    from fewshot_detection_b200 import valid as VA
    args.tta = tta_plan_of(ap, args, args.darknetcfg)
    names, rws = None, None
    if args.rw is not None:
        names = load_class_names(args.names)
        if not names:
            ap.error('--names: no class names in %s' % args.names)
        try:
            rws = VA.load_reweighting_vectors(args.rw, VA.reweighting_vector_shapes(parse_cfg(args.learnetcfg), len(names)))
        except (OSError, ValueError) as e:
            ap.error('--rw: %s (%d names in %s)' % (e, len(names), args.names))
    images = list_images(args.images)
    if not images:
        ap.error('no images in %s' % ' '.join(args.images))
    missing = [p for p in images if not os.path.isfile(p)]
    if missing:
        ap.error('no such image: %s' % missing[0])
    return args, names, rws, images


def tta_plan_of(ap, args, darknetcfg):
    """The test-time augmentation plan of --tta-sides / --tta-flip (None without them); bad sides end the command."""
    if args.tta_sides is None and not args.tta_flip:
        return None
    from fewshot_detection_b200.cfg import parse_cfg
    from fewshot_detection_b200 import valid as VA
    try:
        sides = (VA.parse_tta_sides(args.tta_sides) if args.tta_sides is not None
                 else [int(parse_cfg(darknetcfg)[0]['width'])])
        return VA.tta_plan(sides, args.tta_flip)
    except ValueError as e:
        ap.error('--tta-sides: %s' % e)


def output_dir(args):
    """--out, or `<out>_tta` under a test-time augmentation plan."""
    return args.out + '_tta' if args.tta is not None else args.out


def class_colour(c, n_cls):
    """One colour per class, hues spread around the wheel."""
    import colorsys
    r, g, b = colorsys.hsv_to_rgb((c * 0.618033988749895) % 1.0, 0.9, 1.0)
    return int(r * 255), int(g * 255), int(b * 255)


def draw_boxes(arr, rows, names):
    """A PIL image of arr (uint8 [h, w, 3]) with a rectangle and a `name prob` label per (name, prob, x1, y1, x2, y2)."""
    from PIL import Image, ImageDraw
    img = Image.fromarray(arr)
    draw = ImageDraw.Draw(img)
    for name, prob, x1, y1, x2, y2 in rows:
        colour = class_colour(names.index(name), len(names))
        draw.rectangle([x1, y1, x2, y2], outline=colour, width=2)
        draw.text((x1 + 2, y1 + 1), '%s %.2f' % (name, prob), fill=colour)
    return img


def format_line(row):
    name, prob, x1, y1, x2, y2 = row
    return '%s %r %r %r %r %r\n' % (name, prob, x1, y1, x2, y2)


def main(argv=None):
    args, names, rws, images = parse_args(argv)
    import torch
    torch.cuda.set_device(0)
    return run(args, names, rws, images)


def run(args, names, rws, images):
    import numpy as np
    import torch
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.dataset import DetectionBatcher
    from fewshot_detection_b200.graph import GraphedDetect
    from fewshot_detection_b200.image import decode_many
    from fewshot_detection_b200.utils import logging, read_data_cfg
    from fewshot_detection_b200 import valid as VA
    darknetcfg, learnetcfg = parse_cfg(args.darknetcfg), parse_cfg(args.learnetcfg)
    data_options = None
    if args.data is not None:
        data_options = read_data_cfg(args.data)
        cfg.config_data(data_options)
        names = list(cfg.classes)
    cfg.config_meta(learnetcfg[0])
    cfg.config_net(darknetcfg[0])
    n_cls = len(names)

    m = Darknet(darknetcfg, learnetcfg)
    m.load_weights(args.weightfile)
    m = m.cuda().eval()
    if rws is not None:
        dw = [torch.from_numpy(a).cuda() for a in rws]
    else:
        from fewshot_detection_b200.dataset import MetaBatcher
        from fewshot_detection_b200 import lists as LS
        metalines, inds = LS.support_index(data_options['meta'], names, 0, ensemble=True)
        mb = MetaBatcher(metalines, inds, classes=names, train=False, ensemble=True, with_ids=True)
        meta_batches = (mb.batch(range(s, min(s + args.support_batch, len(inds))))
                        for s in range(0, len(inds), args.support_batch))
        dw = VA.evaluation_dynamic_weights(m, meta_batches, n_cls)
    graphed = None if args.eager or args.tta is not None else GraphedDetect(m, dw, min(args.batch_size, len(images)), m.width, n_cls, args.conf,
                                                    args.nms, args.max_det)
    out_dir = output_dir(args)
    os.makedirs(out_dir, exist_ok=True)
    n_boxes = 0
    no_labels = np.zeros((0, 5), dtype=np.float64)
    for s in range(0, len(images), args.batch_size):
        paths = images[s:s + args.batch_size]
        arrays = decode_many(paths)
        batcher = DetectionBatcher([(a, no_labels) for a in arrays], shape=(m.width, m.height), shuffle=False,
                                   train=False, batch_size=len(paths))
        data = batcher.batch(range(len(paths)))[0] if args.tta is None else None
        sizes = [(int(a.shape[1]), int(a.shape[0])) for a in arrays]
        if args.tta is not None:
            inputs = VA.tta_inputs(batcher, range(len(paths)), args.tta)
            result = VA.detect_tta(m, inputs, dw, n_cls, args.tta, args.conf, args.nms).select(n_cls, sizes, args.max_det)
        elif graphed is not None:
            result = graphed(data, sizes)
        else:
            result = VA.detect_images(m, data, dw, n_cls, sizes, args.conf, args.nms, args.max_det)
        for path, arr, rows in zip(paths, arrays, result.lists(names)):
            stem = os.path.splitext(os.path.basename(path))[0]
            with open(os.path.join(out_dir, stem + '.txt'), 'w') as f:
                f.writelines(format_line(r) for r in rows)
            if args.draw:
                draw_boxes(arr, rows, names).save(os.path.join(out_dir, stem + '.jpg'), quality=95)
            n_boxes += len(rows)
    logging('%d images, %d boxes, written to %s' % (len(images), n_boxes, out_dir))
    return 0


if __name__ == '__main__':
    sys.exit(main())

"""Few-shot list construction: which images a training run iterates over, and which support images feed the
reweighting net (dataset.py:17-169 and MetaDataset.__init__, dataset.py:286-360 of the reference).

Pure host bookkeeping over text files - image-list files (one path per line), "dict" files (`<class> <list-file>`
per line) and Darknet label files (`cls cx cy w h` rows) - that decides the few-shot protocol:

  base training   every image of `train` that shows at least one BASE-class object (novel classes stay unseen);
  fine-tuning     the k-shot dict `meta`, repeated `cfg.repeat` times, or - `dynamic = 1` - the novel k-shot images
                  topped up with randomly drawn base-class images until every class has `shot * repeat` boxes;
  support index   per class `nbatch` random picks from its list, interleaved class by class (one support image per
                  class per step), or every image once for the ensembling pass.

The random draws (`random.sample`, `random.shuffle`, `numpy.random.choice`) are made in the reference's order, so a
seeded run builds the reference's lists (tests/test_lists.py compares with lists minted by the reference itself).
"""
import os
import random

import numpy as np

from .cfg import cfg
from .dataset import get_labpath


def topath(p):
    """The reference rewrites one site-specific path prefix (dataset.py:17-18); identity everywhere else."""
    return p.replace('scratch', 'tmp_scratch/basilisk')


def is_dict(filename):
    """A "dict" file has two fields on its first line: `<class> <list-file>` (utils.py:488-494)."""
    with open(filename, 'r') as f:
        return len(f.readline().strip().split()) == 2


def label_classes(imgpath):
    """Class ids of the boxes in the image's label file as a list (one entry per box); [] for an empty file."""
    labpath = get_labpath(imgpath.rstrip())
    if not os.path.getsize(labpath):
        return []
    rows = np.reshape(np.loadtxt(labpath), (-1, 5))
    return rows[:, 0].astype(int).tolist()


def shows_base_class(imgpath):
    """listDataset.is_valid (dataset.py:273-283): the image has at least one box of a base class."""
    return not set(label_classes(imgpath)).isdisjoint(cfg.base_ids)


def _read_pairs(dictfile):
    """`<class> <list-file>` lines; class names of two words (COCO: 'traffic light') come as four fields."""
    pairs = []
    with open(dictfile, 'r') as f:
        for line in f.readlines():
            p = line.rstrip().split()
            if len(p) == 4:
                p = [p[0] + ' ' + p[1], p[2] + ' ' + p[3]]
            elif len(p) != 2:
                raise NotImplementedError('{} not recognized'.format(p))
            pairs.append(p)
    return pairs


def load_lines(root, checkvalid=True):
    """dataset.py:20-40.  A dict file contributes the lists of its base classes (all classes when checkvalid is
    False), merged, de-duplicated and sorted; a plain list file its lines.  With checkvalid only images showing a
    base-class object survive."""
    if is_dict(root):
        with open(root, 'r') as f:
            rows = [line.rstrip().split() for line in f.readlines()]
        wanted = cfg.base_classes if checkvalid else cfg.classes
        lines = []
        for row in rows:
            if row[0] in wanted:
                with open(topath(row[-1]), 'r') as g:
                    lines.extend(g.readlines())
        lines = sorted(set(lines))
    else:
        with open(root, 'r') as f:
            lines = f.readlines()
    if checkvalid:
        lines = [topath(l) for l in lines if shows_base_class(topath(l))]
    return lines


def load_metadict(metapath, repeat=1):
    """dataset.py:73-109: the NOVEL classes' k-shot images of a dict file and the number of boxes per class they
    already contain (both times `repeat`).  Returns (image list, {class: box count})."""
    metadict = {name: load_lines(listfile) for name, listfile in _read_pairs(metapath)}
    for name in metadict:
        if name not in cfg.novel_classes:
            metadict[name] = []
    metalist = set(sum(metadict.values(), []))
    counts = {name: 0 for name in metadict}
    for imgpath in metalist:
        ids = label_classes(imgpath.strip())
        for ci in set(ids):
            counts[cfg.classes[ci]] += ids.count(ci)
    for name in counts:
        counts[name] *= repeat
    return list(metalist) * repeat, counts


def build_fewset(imglist, metalist, metacnt, shot, replace=True):
    """dataset.py:112-164: top the few-shot list up with randomly drawn images (at most 3 boxes, no novel objects,
    never exceeding `shot` boxes of any class) until every class has `shot` boxes; shuffled."""
    if isinstance(imglist, str):
        with open(imglist) as f:
            names = f.readlines()
    elif isinstance(imglist, list):
        names = imglist.copy()
    else:
        raise NotImplementedError('imglist type not recognized')
    novel = set(cfg.novel_ids)
    while min(metacnt.values()) < shot:
        imgpath = random.sample(names, 1)[0]
        if not os.path.getsize(get_labpath(imgpath.strip())):
            names.remove(imgpath)                  # nothing annotated
            continue
        ids = label_classes(imgpath.strip())
        if len(ids) > 3:
            continue                               # crowded image: skipped but left in the pool
        if not set(ids).isdisjoint(novel):
            names.remove(imgpath)
            continue
        if any(metacnt[cfg.classes[ci]] + ids.count(ci) > shot for ci in set(ids)):
            names.remove(imgpath)
            continue
        for ci in set(ids):
            metacnt[cfg.classes[ci]] += ids.count(ci)
        metalist.append(imgpath)
        if not replace:
            names.remove(imgpath)
    random.shuffle(metalist)
    return metalist


def build_dataset(dataopt):
    """dataset.py:57-70: the image list a training run iterates over."""
    if not cfg.tuning:
        return load_lines(dataopt['train'])
    if cfg.repeat == 1:
        return load_lines(dataopt['meta'])
    if 'dynamic' not in dataopt or int(dataopt['dynamic']) == 0:
        return load_lines(dataopt['meta']) * cfg.repeat
    metalist, metacnt = load_metadict(dataopt['meta'], cfg.repeat)
    return build_fewset(dataopt['train'], metalist, metacnt, cfg.shot * cfg.repeat)


def support_index(metafile, classes, nbatch, ensemble=False, shuffle=False):
    """MetaDataset.__init__ (dataset.py:316-345): per-class support pools `metalines[c]` and the sample order `inds`
    = (clsid, position) pairs: training draws `nbatch` positions per class with numpy.random.choice (class order) and
    interleaves them class by class, the ensembling pass lists every image of every class."""
    files = {name: topath(path) for name, path in _read_pairs(metafile)}
    metalines, per_class = [], []
    for i, name in enumerate(classes):
        with open(files[name], 'r') as f:
            lines = [topath(l) for l in f.readlines()]
        metalines.append(lines)
        if ensemble:
            per_class.append(list(zip([i] * len(lines), list(range(len(lines))))))
        else:
            picks = np.random.choice(range(len(lines)), nbatch).tolist()
            per_class.append(list(zip([i] * nbatch, picks)))
    inds = sum(per_class, []) if ensemble else sum(list(zip(*per_class)), ())
    if shuffle:                                    # cfg.randmeta
        inds = list(inds)
        random.shuffle(inds)
        inds = tuple(inds)
    return metalines, inds


def rank_support_rows(inds, n_cls, replicas, world, rank):
    """The support index of `replicas` replicas per global step (built with cfg.num_gpus = replicas, consumed
    replicas * n_cls entries at a time and scattered in order, replica r taking entries [r * n_cls, (r + 1) * n_cls) of
    each step) as rank `rank` of `world` sees it: the entries of its replicas replicas / world * rank ... in order."""
    per = replicas // world * n_cls
    step = replicas * n_cls
    return [inds[s + rank * per + j] for s in range(0, len(inds) - step + 1, step) for j in range(per)]


def support_batches_per_epoch(train=True):
    """dataset.py:296-309: `nbatch` of MetaDataset - how many support batches one epoch's index holds."""
    if train:
        factor = 4 if cfg.get('data', 'voc') == 'coco' else 1
    else:
        factor = 10
    return factor * 500 * 64 * cfg.num_gpus // cfg.batch_size

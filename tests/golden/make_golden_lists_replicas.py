#!/usr/bin/env python
"""Mint tests/golden/lists_replicas.json: the support index the REFERENCE's own dataset.py (MetaDataset.__init__, run
unmodified) builds for its shipped 4-GPU configurations (cfg.num_gpus = 4), on the directory stored in lists.json -
build container only:

    python tests/golden/make_golden_lists_replicas.py

Stored: the seed, the index length, the per-class pool sizes, MetaDataset.batch_size and the first 2400 entries.
tests/test_replicas_cpu.py rebuilds the directory from lists.json and compares fewshot_detection_b200.lists."""
import io
import json
import os
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.dont_write_bytecode = True
sys.path.insert(0, os.path.join(HERE, '_shims'))
sys.path.insert(0, '/root/reference')
if not hasattr(np, 'int'):
    np.int = int                      # numpy >= 1.24 removed the alias the reference uses
with redirect_stdout(io.StringIO()):
    import dataset as RD              # the reference's dataset.py
from cfg import cfg as RC


def main():
    d = json.load(open(os.path.join(HERE, 'lists.json')))
    root = tempfile.mkdtemp()
    os.makedirs(os.path.join(root, 'JPEGImages'))
    for rel, text in d['files'].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'w') as f:
            f.write(text.replace('<ROOT>', root))
    classes, novel = d['classes'], d['novel']
    RC.data, RC.classes, RC.tuning, RC.repeat, RC.shot = 'voc', classes, False, 1, 2
    RC.novel_classes = novel
    RC.base_classes = [c for c in classes if c not in novel]
    RC.base_ids = [classes.index(c) for c in RC.base_classes]
    RC.novel_ids = [classes.index(c) for c in novel]
    RC.num_gpus, RC.batch_size, RC.randmeta = 4, 64, False
    RC.meta_width = RC.meta_height = RC.mask_width = RC.mask_height = 64
    with redirect_stdout(io.StringIO()):
        np.random.seed(3)
        md = RD.MetaDataset(os.path.join(root, 'lists/dict_full.txt'), train=True)
    out = {'seed': 3, 'num_gpus': 4, 'n': len(md.inds), 'meta_cnts': md.meta_cnts, 'batch_size': md.batch_size,
           'inds': [list(map(int, t)) for t in md.inds[:2400]]}
    with open(os.path.join(HERE, 'lists_replicas.json'), 'w') as f:
        json.dump(out, f)
    print('wrote lists_replicas.json: n %d, batch_size %d' % (out['n'], out['batch_size']))


if __name__ == '__main__':
    main()

"""The replica step's host side without a GPU: the support index for 4 replicas against what the reference's own
dataset.py built with num_gpus = 4 (tests/golden/lists_replicas.json, minted by make_golden_lists_replicas.py), the
rows each rank takes from it, and the refusals of `tools/train_meta_b200.py --replicas` and of a state file written
under another replica count, all made before any CUDA work."""
import importlib.util
import json
import os
import random
import sys

import numpy as np
import pytest
import torch

from fewshot_detection_b200 import resume as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture()
def saved_cfg():
    from fewshot_detection_b200.cfg import cfg
    saved = dict(cfg)
    yield cfg
    cfg.clear()
    cfg.update(saved)


def test_support_index_for_four_replicas_matches_the_reference(tmp_path, saved_cfg):
    from fewshot_detection_b200 import lists as LS
    cfg = saved_cfg
    d = json.load(open(os.path.join(G, 'lists.json')))
    w = json.load(open(os.path.join(G, 'lists_replicas.json')))
    root = str(tmp_path)
    for rel, text in d['files'].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'w') as f:
            f.write(text.replace('<ROOT>', root))
    classes, novel = d['classes'], d['novel']
    cfg.data, cfg.classes, cfg.tuning, cfg.repeat, cfg.shot = 'voc', classes, False, 1, 2
    cfg.novel_classes = novel
    cfg.base_classes = [c for c in classes if c not in novel]
    cfg.num_gpus, cfg.batch_size, cfg.randmeta = w['num_gpus'], 64, False
    n_cls = len(cfg.base_classes)
    np.random.seed(w['seed'])
    metalines, inds = LS.support_index(os.path.join(root, 'lists/dict_full.txt'), cfg.base_classes,
                                       LS.support_batches_per_epoch(train=True))
    assert len(inds) == w['n'] and [len(m) for m in metalines] == w['meta_cnts']
    assert [list(map(int, t)) for t in inds[:len(w['inds'])]] == w['inds']
    assert n_cls * 4 == w['batch_size']            # one global step = 4 support sets
    # replica r of a step: one support image per class, in class order
    for r in range(4):
        assert [c for c, _ in inds[r * n_cls:(r + 1) * n_cls]] == list(range(n_cls))
    # every rank takes the rows of its own replicas, in order; together the ranks cover each step once
    one = LS.rank_support_rows(inds, n_cls, 4, 1, 0)
    assert one == list(inds)
    for world in (2, 4):
        parts = [LS.rank_support_rows(inds, n_cls, 4, world, k) for k in range(world)]
        per = 4 // world * n_cls
        for s in range(3):
            got = sum([p[s * per:(s + 1) * per] for p in parts], [])
            assert got == list(inds[s * 4 * n_cls:(s + 1) * 4 * n_cls])


def test_meta_batcher_takes_one_support_set_per_replica(saved_cfg):
    from fewshot_detection_b200.dataset import MetaBatcher
    saved_cfg.metain_type = 2
    saved_cfg.meta_width = saved_cfg.meta_height = saved_cfg.mask_width = saved_cfg.mask_height = 64
    classes = ['a', 'b', 'c']
    assert MetaBatcher([[]] * 3, [], classes=classes).batch_size == 3
    assert MetaBatcher([[]] * 3, [], classes=classes, replicas=4).batch_size == 12


class _CudaReached(Exception):
    pass


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_driver_refuses_replica_layouts_and_state_files_before_any_cuda_work(tmp_path, monkeypatch, capsys, saved_cfg):
    from fewshot_detection_b200.cfg import parse_cfg
    from fewshot_detection_b200 import netcfg, lists as LS
    from fewshot_detection_b200.utils import read_data_cfg
    cfg = saved_cfg
    monkeypatch.setattr(torch.cuda, 'set_device', lambda *a: (_ for _ in ()).throw(_CudaReached()))
    monkeypatch.delenv('WORLD_SIZE', raising=False)
    root = str(tmp_path)
    with open(os.path.join(root, 'novels.txt'), 'w') as f:
        f.write('bird,bus,cow,motorbike,sofa\n')
    os.makedirs(os.path.join(root, 'JPEGImages'))
    os.makedirs(os.path.join(root, 'labels'))
    for i in range(17):
        with open(os.path.join(root, 'labels', '%06d.txt' % i), 'w') as f:
            f.write('0 0.5 0.5 0.2 0.2\n')
    train = os.path.join(root, 'train.txt')
    with open(train, 'w') as f:
        f.write(''.join(os.path.join(root, 'JPEGImages', '%06d.jpg\n' % i) for i in range(16)))
    data = os.path.join(root, 'meta.data')
    with open(data, 'w') as f:
        f.write('metayolo=1\nmetain_type=2\ndata=voc\nneg = 1\nrand = 0\nnovel = %s\nnovelid = 0\nmeta = unused.txt\n'
                'train = %s\nbackup = %s\n' % (os.path.join(root, 'novels.txt'), train, os.path.join(root, 'backup')))
    det = netcfg.mini_dynamic_blocks(128, 16)
    det[0]['batch'] = '8'
    netcfg.write_cfg(det, os.path.join(root, 'det.cfg'))
    netcfg.write_cfg(netcfg.mini_reweighting_blocks(64, 16, 512), os.path.join(root, 'ler.cfg'))
    weights = os.path.join(root, '000002.weights')
    with open(weights, 'wb') as f:
        f.write(b'\0' * 64)
    args = ['train_meta_b200.py', data, os.path.join(root, 'det.cfg'), os.path.join(root, 'ler.cfg'), weights]
    cli = _tool('train_meta_b200')

    def run(extra, world=1):
        monkeypatch.setenv('WORLD_SIZE', str(world))
        monkeypatch.setattr(sys, 'argv', args + list(extra))
        try:
            rc = cli.main()
        except _CudaReached:
            rc = 'cuda'
        return rc, capsys.readouterr().out

    assert run(['--replicas', '4'])[0] == 'cuda'                   # 8 images, 4 replicas of 2
    assert run(['--replicas', '4'], world=2)[0] == 'cuda'
    rc, out = run(['--replicas', '3'], world=2)
    assert rc == 1 and '--replicas 3' in out and 'world size 2' in out
    rc, out = run(['--replicas', '0'])
    assert rc == 1 and 'positive multiple' in out
    rc, out = run(['--replicas', '16'])
    assert rc == 1 and 'global batch 8 does not split into 16 replicas' in out

    # a state file records the replicas; one written under another count is refused with both values
    opts = read_data_cfg(data)
    dk, lk = parse_cfg(args[2]), parse_cfg(args[3])
    cfg.config_data(opts)
    cfg.config_meta(lk[0])
    cfg.config_net(dk[0])
    random.seed(3)
    np.random.seed(3)
    trainlist = LS.build_dataset(opts)
    for stored, extra, want in ((4, [], 'replicas per step 4, this run has 1'),
                                (1, ['--replicas', '4'], 'replicas per step 1, this run has 4'),
                                (2, ['--replicas', '4'], 'replicas per step 2, this run has 4')):
        fp = R.fingerprint(dk, lk, opts, 1, 8, 8, trainlist, replicas=stored)
        path = os.path.join(root, 'r%d.state' % stored)
        R.write_state(path, dict(format=R.FORMAT, weights=R.file_digest(weights), fingerprint=fp, seed=3, trainer={}, ranks=[]))
        rc, out = run(extra + ['--resume', path])
        assert rc == 1 and want in out, out
    fp = R.fingerprint(dk, lk, opts, 1, 8, 8, trainlist, replicas=4)
    R.write_state(os.path.join(root, 'ok.state'), dict(format=R.FORMAT, weights=R.file_digest(weights), fingerprint=fp, seed=3,
                                                       trainer={}, ranks=[]))
    assert run(['--replicas', '4', '--resume', os.path.join(root, 'ok.state')])[0] == 'cuda'
    # a state file from before replicas were recorded stands for one replica per rank
    old = R.fingerprint(dk, lk, opts, 1, 8, 8, trainlist)
    del old['replicas']
    R.write_state(os.path.join(root, 'old.state'), dict(format=R.FORMAT, weights=R.file_digest(weights), fingerprint=old, seed=3,
                                                        trainer={}, ranks=[]))
    assert run(['--resume', os.path.join(root, 'old.state')])[0] == 'cuda'
    rc, out = run(['--replicas', '4', '--resume', os.path.join(root, 'old.state')])
    assert rc == 1 and 'replicas per step 1, this run has 4' in out


def test_darknet_refuses_batches_that_do_not_split_into_replicas():
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    with pytest.raises(ValueError, match='replicas must be >= 1'):
        Darknet(netcfg.mini_dynamic_blocks(128, 4), netcfg.mini_reweighting_blocks(64, 4, 128), replicas=0)
    m = Darknet(netcfg.mini_dynamic_blocks(128, 4), netcfg.mini_reweighting_blocks(64, 4, 128), replicas=4).train()
    for bs, rows in ((6, 16), (8, 6)):           # checked before anything runs on a device
        with pytest.raises(ValueError, match=r'4 replicas .* got x \(%d, 3, 128, 128\) and metax \(%d, 3, 64, 64\)' % (bs, rows)):
            m(torch.zeros(bs, 3, 128, 128), torch.zeros(rows, 3, 64, 64), torch.zeros(rows, 1, 64, 64))

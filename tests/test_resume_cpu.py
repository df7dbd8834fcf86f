"""Resuming meta-training from a training-state file (fewshot_detection_b200/resume.py) on the CPU:

  * four epochs in one MetaTrainer equal two epochs, then a new MetaTrainer loaded from the epoch-2 state file, then
    two more - parameters, momentum, the lr of every step, processed_batches, both `seen` counters, the logged lines -
    for the base-training and the fine-tuning (`tuning=1`) schedule;
  * the state file's round trip, and a write interrupted by an exception leaving the previous file intact;
  * every refusal of `tools/train_meta_b200.py --resume`, each made before the first CUDA call;
  * the BackgroundPrep handshake: a worker and a consumer drawing from `random` make the draws of the serial loop,
    whichever side is slower.

The model is a stub (as in test_trainer_cpu.py) whose loss makes one `random()` draw per step like neg_filter; the data
side is the real DetectionBatcher / MetaBatcher with the C-ABI calls routed to the host-emulated kernels."""
import os
import random
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn as nn

from emul_util import build_emul, route_image_calls_to_emulation
from fewshot_detection_b200 import resume as R
from fewshot_detection_b200 import trainer as T

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class StubLoss(nn.Module):
    seen = 0

    def forward(self, output, target):
        return output.sum() * 1e-3 * (1. + random.random())      # one draw per step, as neg_filter makes


class StubModel(nn.Module):
    """The Darknet surface MetaTrainer touches; save_weights writes `seen` and the parameters to a file."""

    def __init__(self, n_cls):
        super().__init__()
        self.w = nn.Parameter(torch.ones(1))
        self.b = nn.Parameter(torch.zeros(3))
        self.n_cls, self.seen = n_cls, 0
        self.loss = StubLoss()

    def forward(self, x, metax, mask):
        g = x.size(-1) // 32
        return (x.mean() * self.w + metax.mean() * self.b.sum()).expand(x.size(0) * self.n_cls, 30, g, g)

    def save_weights(self, path):
        with open(path, 'wb') as f:
            np.array([0, 0, 0, self.seen], np.int32).tofile(f)
            torch.cat([self.w.detach(), self.b.detach()]).numpy().tofile(f)

    def load_weights(self, path):
        with open(path, 'rb') as f:
            self.seen = int(np.fromfile(f, count=4, dtype=np.int32)[3])
            v = torch.from_numpy(np.fromfile(f, dtype=np.float32))
        with torch.no_grad():
            self.w.copy_(v[:1])
            self.b.copy_(v[1:])


@pytest.fixture()
def data_side(monkeypatch):
    emul = build_emul('augment', 'augment.cu')
    route_image_calls_to_emulation(monkeypatch, emul)
    from fewshot_detection_b200.cfg import cfg
    saved = dict(cfg)
    ncls = 3
    cfg.base_classes, cfg.base_ids, cfg.metain_type, cfg.multiscale, cfg.metayolo = cfg.voc_classes[:ncls], list(range(ncls)), 2, 0, True
    cfg.meta_width = cfg.meta_height = cfg.mask_width = cfg.mask_height = 48
    gold = np.load(os.path.join(G, 'dataset.npz'), allow_pickle=False)
    lines = [(gold['src%d' % i], gold['lab%d' % i]) for i in range(8)]
    pool = gold['meta/pool']
    metalines = [[(gold['src%d' % i], gold['meta_lab/%d/%d' % (c, i)]) for i in pool[c] if i >= 0] for c in range(ncls)]
    inds = [tuple(int(v) for v in r) for r in gold['meta/inds']]
    yield ncls, lines, metalines, inds
    cfg.clear()
    cfg.update(saved)


def make_trainer(data, backup, weights=None, save_state=None):
    from fewshot_detection_b200.dataset import DetectionBatcher, MetaBatcher
    ncls, lines, metalines, inds = data
    model = StubModel(ncls)
    if weights is not None:
        model.load_weights(weights)
    opt = torch.optim.SGD(model.parameters(), **T.sgd_hyper_parameters(0.001, 0.9, 0.0005, 4, 15.))
    logs, lrs = [], []
    tr = T.MetaTrainer(model, opt, 0.001 / 15., 4, [-1, 1, 3, 5], [0.1, 10, 0.1, 0.5],
                       lambda seen: DetectionBatcher(list(lines), shape=(64, 64), shuffle=True, train=True, seen=seen,
                                                     batch_size=4, num_workers=1),
                       lambda: MetaBatcher(metalines, [inds[i] for i in np.random.permutation(len(inds))], train=True),
                       backupdir=backup, save_interval=1, log=logs.append, save_state=save_state)
    orig = tr.train_step
    tr.train_step = lambda *a: (lrs.append(opt.param_groups[0]['lr']), orig(*a))[1]
    return tr, logs, lrs


def snapshot(tr):
    opt = tr.optimizer
    return dict(params=[p.detach().clone() for p in tr.model.parameters()],
                momentum=[opt.state[p]['momentum_buffer'].clone() for p in tr.model.parameters()],
                processed=tr.processed_batches, loss_seen=tr.region_loss.seen, model_seen=tr.model.seen,
                draw=(random.random(), float(np.random.rand()), float(torch.rand(1))))


def bit_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def fit_plan(model_seen, tuning):
    """The driver's epoch_plan for this stub data set: 8 images, batch 4, 4 epochs (fine-tuning: max_epoch 4)."""
    return T.epoch_plan(model_seen, 8, 4, 7, tuning, 4, 1)


@pytest.mark.parametrize('tuning', [0, 1])
@pytest.mark.parametrize('bg_prep', ['1', '0'])
def test_resumed_run_equals_uninterrupted(data_side, tmp_path, monkeypatch, tuning, bg_prep):
    monkeypatch.setenv('FSDET_NO_BG_PREP', '0' if bg_prep == '1' else '1')
    fp = dict(world=1)
    a_dir, b_dir = tmp_path / 'a', tmp_path / 'b'
    a_dir.mkdir()
    b_dir.mkdir()

    # uninterrupted: epochs 0..3, a state file per checkpoint (only the newest kept)
    random.seed(9)
    np.random.seed(9)
    torch.manual_seed(9)
    tr, logs_a, lrs_a = make_trainer(data_side, str(a_dir), save_state=R.state_saver(fp, 9, log=lambda *_: None))
    processed, init_epoch, max_epochs = fit_plan(tr.model.seen, tuning)
    assert max_epochs == 4
    tr.processed_batches = processed
    tr.fit(init_epoch, max_epochs)
    want = snapshot(tr)
    assert sorted(os.listdir(a_dir)) == sorted(['%06d.weights' % e for e in range(1, 5)] + ['000004.state'])

    # stopped after epoch 2, then a new trainer continues from the epoch-2 state
    class Killed(Exception):
        pass
    saver = R.state_saver(fp, 9, log=lambda *_: None)

    def save_then_stop(trainer, epoch):
        saver(trainer, epoch)
        if epoch == 2:
            raise Killed()
    random.seed(9)
    np.random.seed(9)
    torch.manual_seed(9)
    tr, logs_b, lrs_b = make_trainer(data_side, str(b_dir), save_state=save_then_stop)
    tr.processed_batches = processed
    with pytest.raises(Killed):
        tr.fit(init_epoch, max_epochs)
    assert sorted(os.listdir(b_dir)) == ['000001.weights', '000002.state', '000002.weights']
    state = R.read_state(str(b_dir / '000002.state'))
    R.check_weights(state, str(b_dir / '000002.state'), str(b_dir / '000002.weights'))
    assert state['trainer']['epoch'] == 2 and state['trainer']['processed_batches'] == processed + 4
    assert state['seed'] == 9 and state['fingerprint'] == fp and len(state['ranks']) == 1

    random.seed(12345)                 # the restored streams make the seed irrelevant
    np.random.seed(12345)
    torch.manual_seed(12345)
    tr2, logs_c, lrs_c = make_trainer(data_side, str(b_dir), weights=str(b_dir / '000002.weights'),
                                      save_state=R.state_saver(fp, 9, log=lambda *_: None))
    processed2, init_epoch2, _ = fit_plan(tr2.model.seen, tuning)
    tr2.processed_batches = processed2
    R.restore(tr2, state)
    tr2.fit(init_epoch2, max_epochs)
    got = snapshot(tr2)

    assert lrs_b + lrs_c == lrs_a and len(lrs_a) == 8
    for k in ('params', 'momentum'):
        assert all(bit_equal(x, y) for x, y in zip(got[k], want[k])), k
    for k in ('processed', 'loss_seen', 'model_seen', 'draw'):
        assert got[k] == want[k], (k, got[k], want[k])
    timing = lambda logs: [l.replace(str(b_dir), str(a_dir)) for l in logs if 'samples/s' not in l]
    assert timing(logs_b) + timing(logs_c) == timing(logs_a)
    for e in (3, 4):
        with open(a_dir / ('%06d.weights' % e), 'rb') as f, open(b_dir / ('%06d.weights' % e), 'rb') as g:
            assert f.read() == g.read()
    # the resumed run deletes only the state file it wrote itself
    assert sorted(os.listdir(b_dir)) == sorted(['%06d.weights' % e for e in range(1, 5)] + ['000002.state', '000004.state'])


def test_state_file_round_trip_and_interrupted_write(tmp_path, monkeypatch):
    m = nn.Linear(3, 2)
    opt = torch.optim.SGD(m.parameters(), lr=0.1, momentum=0.9)
    m(torch.randn(4, 3)).sum().backward()
    opt.step()
    random.seed(1)
    np.random.seed(2)
    state = dict(format=R.FORMAT, weights=dict(name='w', bytes=3, sha256='x'), fingerprint=dict(world=1), seed=7,
                 trainer=dict(epoch=2, optimizer=opt.state_dict()), ranks=[dict(model_seen=5, rng=T.rng_state())])
    p = str(tmp_path / '000002.state')
    R.write_state(p, state)
    got = R.read_state(p)
    assert got['seed'] == 7 and got['trainer']['epoch'] == 2 and got['ranks'][0]['model_seen'] == 5
    for k, s in opt.state_dict()['state'].items():
        assert bit_equal(got['trainer']['optimizer']['state'][k]['momentum_buffer'], s['momentum_buffer'])
    want = (random.random(), float(np.random.rand()), float(torch.rand(1)))
    random.seed(0)
    np.random.seed(0)
    T.set_rng_state(got['ranks'][0]['rng'])
    assert (random.random(), float(np.random.rand()), float(torch.rand(1))) == want
    opt2 = torch.optim.SGD(m.parameters(), lr=0.5, momentum=0.1)
    opt2.load_state_dict(got['trainer']['optimizer'])
    assert opt2.param_groups[0]['lr'] == 0.1 and opt2.param_groups[0]['momentum'] == 0.9
    # the same state written twice gives the same bytes
    R.write_state(str(tmp_path / 'again.state'), state)
    assert open(p, 'rb').read() == open(str(tmp_path / 'again.state'), 'rb').read()

    # a write that fails part-way leaves the previous file as it was and no temporary file
    before = open(p, 'rb').read()

    def killed(fd):
        raise KeyboardInterrupt('killed mid-write')
    monkeypatch.setattr(os, 'fsync', killed)
    with pytest.raises(KeyboardInterrupt):
        R.write_state(p, dict(state, seed=8))
    assert open(p, 'rb').read() == before and sorted(os.listdir(tmp_path)) == ['000002.state', 'again.state']


def tool(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _CudaReached(Exception):
    pass


def test_driver_refuses_a_state_that_does_not_fit_before_any_cuda_work(tmp_path, monkeypatch, capsys):
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200 import netcfg, lists as LS
    from fewshot_detection_b200.utils import read_data_cfg
    saved = dict(cfg)
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
    try:
        opts = read_data_cfg(data)
        dk, lk = parse_cfg(args[2]), parse_cfg(args[3])
        cfg.config_data(opts)
        cfg.config_meta(lk[0])
        cfg.config_net(dk[0])
        random.seed(3)
        np.random.seed(3)
        fp = R.fingerprint(dk, lk, opts, 1, 8, 8, LS.build_dataset(opts))
        good = dict(format=R.FORMAT, weights=R.file_digest(weights), fingerprint=fp, seed=3, trainer={}, ranks=[])
        cli = tool('train_meta_b200')

        def run(state, name='s.state', extra=()):
            path = os.path.join(root, name)
            if state is not None:
                R.write_state(path, state)
            monkeypatch.setattr(sys, 'argv', args + ['--resume', path] + list(extra))
            try:
                rc = cli.main()
            except _CudaReached:
                rc = 'cuda'
            return rc, capsys.readouterr().out

        assert run(good)[0] == 'cuda'                      # every check passes: the run goes on to the device
        rc, out = run(None, 'missing.state')
        assert rc == 1 and 'missing.state' in out and 'no such file' in out
        R.write_state(os.path.join(root, 'full.state'), good)
        blob = open(os.path.join(root, 'full.state'), 'rb').read()
        with open(os.path.join(root, 'cut.state'), 'wb') as f:
            f.write(blob[:len(blob) // 2])
        rc, out = run(None, 'cut.state')
        assert rc == 1 and 'cut.state' in out and 'truncated' in out
        rc, out = run(dict(good, format=99))
        assert rc == 1 and 'format version 99' in out and 'reads 1' in out
        w2 = dict(good, weights=dict(good['weights'], sha256='0' * 64))
        rc, out = run(w2)
        assert rc == 1 and '0' * 64 in out and good['weights']['sha256'] in out and weights in out
        monkeypatch.setenv('WORLD_SIZE', '2')
        rc, out = run(good)
        assert rc == 1 and 'world size 1, this run has 2' in out
        monkeypatch.delenv('WORLD_SIZE')
        rc, out = run(dict(good, fingerprint=dict(fp, batch=16)))
        assert rc == 1 and 'global batch 16, this run has 8' in out
        rc, out = run(dict(good, fingerprint=dict(fp, cfg='c' * 64)))
        assert rc == 1 and 'c' * 64 in out and fp['cfg'] in out
        rc, out = run(dict(good, fingerprint=dict(fp, data=dict(fp['data'], neg='0'))))
        assert rc == 1 and ".data options {'neg': '0'}, this run has {'neg': '1'}" in out
        with open(train, 'a') as f:
            f.write(os.path.join(root, 'JPEGImages', '000016.jpg\n'))
        rc, out = run(good)
        assert rc == 1 and 'training list' in out and "'n': 16" in out and "'n': 17" in out
    finally:
        cfg.clear()
        cfg.update(saved)


def _prep_draws(worker_sleep, consumer_sleep, n=5):
    """Worker thunks and a consumer loop both drawing from `random`, with the consumer signalling after its draws."""
    from fewshot_detection_b200.prefetch import BackgroundPrep
    seq = []

    def thunk(i):
        def t():
            time.sleep(worker_sleep)
            seq.append(('prepare', i, random.random(), random.random()))
            return i
        return t
    random.seed(21)
    prep = BackgroundPrep(thunk(i) for i in range(n))
    for i in prep:
        time.sleep(consumer_sleep)
        seq.append(('step', i, random.random()))
        prep.draws_done()
    return seq


def test_background_prep_draws_in_the_serial_order():
    random.seed(21)
    serial = []
    for i in range(5):
        serial.append(('prepare', i, random.random(), random.random()))
        serial.append(('step', i, random.random()))
    assert _prep_draws(0.0, 0.02) == serial        # a fast worker waits for each step's draws
    assert _prep_draws(0.02, 0.0) == serial        # a slow worker: the consumer waits for each batch

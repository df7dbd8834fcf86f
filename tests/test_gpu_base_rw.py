"""Stored base-class reweighting vectors on the GPU (the reference's `use_baserw`): the evaluation command's --save-rw
and --base-rw, valid.score_batches with the substitution, sharded evaluation and the training driver's checkpoint
scoring, on the synthetic data set of test_gpu_eval_shard_multi (JPEGs, devkit, mini cfgs, a seeded weight file) plus
a COCO annotation file of the same objects and a second weight file whose vectors are "foreign":
  * the model's own vectors stored and substituted change nothing: the same AP lines and result files, only the
    result directory is ene_<ckpt>;
  * foreign vectors: the command equals valid.score_batches with the vectors substituted by hand, which differ from
    the ensembled ones in exactly the base rows, for the VOC and the COCO metric; valid.valid_batches reading the file
    writes the command's result files;
  * two processes (NCCL with 2 GPUs; gloo on one GPU, the ranks sharing it) print the same lines and write the same
    result files and vectors file as one process, with and without --base-rw;
  * the training driver's checkpoint_evaluator logs the command's mean / base / novel AP and leaves training as it
    was without it.

Run as a script under torch.distributed.run, this file is the gloo worker: every rank runs the command's argument
checks and its run() on the shared GPU."""
import contextlib
import importlib.util
import io
import json
import os
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools')
PRINTED = ('VOC07', 'AP for', 'Mean', 'COCO box', ' Average')
SIZES = ['--batch-size', '4', '--support-batch', '8']


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(TOOLS, name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def printed(text):
    return [l for l in text.splitlines() if l.startswith(PRINTED)]


def result_dirs(cwd):
    """{result directory name: {file: bytes}} under cwd/results/<backup>/."""
    out = {}
    top = os.path.join(cwd, 'results')
    for backup in sorted(os.listdir(top)) if os.path.isdir(top) else []:
        for d in sorted(os.listdir(os.path.join(top, backup))):
            p = os.path.join(top, backup, d)
            out[d] = dict((f, open(os.path.join(p, f), 'rb').read()) for f in sorted(os.listdir(p)))
    return out


def torchrun(port, args, cwd):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr',
           '127.0.0.1', '--master-port', str(port)] + args
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=cwd)


def command(args, cwd, port=None):
    """The evaluation command in a fresh directory, in one process (port None) or two under NCCL.  Returns the
    printed result lines and the result directories."""
    os.makedirs(cwd)
    if port is None:
        r = subprocess.run([sys.executable, os.path.join(TOOLS, 'valid_ensemble_b200.py')] + args, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=900, cwd=cwd)
    else:
        r = torchrun(port, [os.path.join(TOOLS, 'valid_ensemble_b200.py')] + args, cwd)
    assert r.returncode == 0, r.stdout[-4000:]
    return printed(r.stdout), result_dirs(cwd)


def write_coco_annotations(root, path):
    """instances json of the data set's label boxes (class k is category k + 1, COCO spellings), the third object of
    an image marked crowd as the devkit marks it difficult."""
    from PIL import Image
    from fewshot_detection_b200 import coco_eval as CE
    from fewshot_detection_b200.cfg import cfg
    images, anns = [], []
    names = sorted(f[:-4] for f in os.listdir(os.path.join(root, 'JPEGImages')))
    for i, name in enumerate(names):
        W, H = Image.open(os.path.join(root, 'JPEGImages', name + '.jpg')).size
        images.append({'id': i + 1, 'file_name': name + '.jpg', 'width': W, 'height': H})
        with open(os.path.join(root, 'labels', name + '.txt')) as f:
            for k, l in enumerate(f):
                c, x, y, w, h = [float(v) for v in l.split()]
                box = [(x - w / 2) * W, (y - h / 2) * H, w * W, h * H]
                anns.append({'id': len(anns) + 1, 'image_id': i + 1, 'category_id': int(c) + 1, 'bbox': box,
                             'area': box[2] * box[3], 'iscrowd': int(k == 2)})
    cats = [{'id': k + 1, 'name': CE.COCO_ALIASES.get(c, c)} for k, c in enumerate(cfg.voc_classes)]
    with open(path, 'w') as f:
        json.dump({'images': images, 'annotations': anns, 'categories': cats}, f)


@pytest.fixture(scope='module')
def ds(tmp_path_factory):
    from test_gpu_eval_shard_multi import write_data_set
    root = str(tmp_path_factory.mktemp('base_rw'))
    data = os.path.join(root, 'data')
    args = write_data_set(data)
    from fewshot_detection_b200.cfg import parse_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from seeding import seeded_init
    m = Darknet(parse_cfg(args[1]), parse_cfg(args[2]))
    seeded_init(m, 4)
    os.makedirs(os.path.join(root, 'foreign'))
    foreign = os.path.join(root, 'foreign', '000004.weights')
    m.save_weights(foreign)
    write_coco_annotations(data, os.path.join(root, 'instances.json'))
    rw = lambda n: os.path.join(root, 'rws', n)
    cfgs = args[:3]
    voc = args[4:7] + SIZES                             # --devkit DIR --write-results, the batch sizes
    d = dict(root=root, data=data, cfgs=cfgs, weights=args[3], foreign=foreign, devkit=args[5], voc=voc, rw=rw,
             coco=os.path.join(root, 'instances.json'))
    d['runs'] = {
        # the plain evaluation, also writing the model's own vectors
        'plain': cfgs + [args[3]] + voc + ['--save-rw', rw('own.pkl')],
        'own': cfgs + [args[3]] + voc + ['--base-rw', rw('own.pkl')],
        # the foreign model's vectors: the support pass only
        'save_foreign': cfgs + [foreign, '--save-rw', rw('foreign.pkl')] + SIZES,
        'foreign': cfgs + [args[3]] + voc + ['--base-rw', rw('foreign.pkl'), '--save-rw', rw('own_again.pkl')],
        'coco_foreign': cfgs + [args[3], '--coco-annotations', d['coco'], '--write-coco-results',
                                os.path.join(root, 'coco_foreign.json'), '--base-rw', rw('foreign.pkl')] + SIZES,
    }
    d['out'] = {}
    for name in ('plain', 'own', 'save_foreign', 'foreign', 'coco_foreign'):
        d['out'][name] = command(d['runs'][name], os.path.join(root, 'one', name))
    return d


@pytest.fixture()
def saved_cfg():
    from fewshot_detection_b200.cfg import cfg
    saved = dict(cfg)
    yield cfg
    cfg.clear()
    cfg.update(saved)


def test_own_vectors_change_nothing(ds):
    lines, dirs = ds['out']['plain']
    lines_own, dirs_own = ds['out']['own']
    assert len(lines) >= 22 and lines[0].startswith('VOC07') and any(l.startswith('Mean Novel') for l in lines)
    assert list(dirs) == ['ene000010'] and list(dirs_own) == ['ene_000010']
    files = dirs['ene000010']
    assert len(files) == 20 and sum(len(v) for v in files.values()) > 0
    assert lines_own == lines
    assert dirs_own['ene_000010'] == files
    with open(ds['rw']('own.pkl'), 'rb') as f:
        own = pickle.load(f)
    assert isinstance(own, list) and len(own) == 1 and own[0].dtype == np.float32 and own[0].shape == (20, 512, 1, 1)
    assert np.isfinite(own[0]).all() and np.abs(own[0]).max() > 0
    with open(ds['rw']('own_again.pkl'), 'rb') as f:            # written by the --base-rw run before substituting
        assert f.read() == open(ds['rw']('own.pkl'), 'rb').read()
    assert not os.path.exists(os.path.join(ds['root'], 'one', 'save_foreign', 'results'))   # support pass only


def api_setup(ds):
    """The command's model, support batches and image batches, built in this process through the API."""
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.utils import read_data_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.dataset import DetectionBatcher, MetaBatcher
    from fewshot_detection_b200 import lists as LS
    data_options = read_data_cfg(ds['cfgs'][0])
    det, ler = parse_cfg(ds['cfgs'][1]), parse_cfg(ds['cfgs'][2])
    cfg.config_data(data_options)
    cfg.config_meta(ler[0])
    cfg.config_net(det[0])
    classes = list(cfg.classes)
    m = Darknet(det, ler)
    m.load_weights(ds['weights'])
    m = m.cuda().eval()
    metalines, inds = LS.support_index(data_options['meta'], classes, 0, ensemble=True)
    mb = MetaBatcher(metalines, inds, classes=classes, train=False, ensemble=True, with_ids=True)
    supports = lambda: (mb.batch(range(s, min(s + 8, len(inds)))) for s in range(0, len(inds), 8))
    with open(data_options['valid']) as f:
        lines = [l.rstrip() for l in f if l.strip()]
    db = DetectionBatcher(lines, shape=(m.width, m.height), shuffle=False, train=False, batch_size=4)
    imgids = [os.path.basename(l).split('.')[0] for l in lines]

    def images():
        for s in range(0, len(lines), 4):
            idx = range(s, min(s + 4, len(lines)))
            yield db.batch(idx)[0], [imgids[i] for i in idx], [db._entry(i).size() for i in idx]
    return m, supports, images, classes, list(cfg.novel_classes), imgids


def api_pass(ds, evaluator_of, out, **result_kwargs):
    """valid.score_batches over the command's batches, detecting with the ensembled vectors whose base rows are
    substituted by hand from the foreign file; those must differ from the ensembled ones in exactly the base rows."""
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200 import valid as VA
    m, supports, images, classes, novel, imgids = api_setup(ds)
    ensembled = VA.ensemble_dynamic_weights(m, supports(), len(classes))[0].clone()
    with open(ds['rw']('own.pkl'), 'rb') as f:                 # --save-rw wrote the ensemble, bit for bit
        own = torch.from_numpy(pickle.load(f)[0]).cuda()
    assert torch.equal(own.view(torch.int32), ensembled.view(torch.int32))
    with open(ds['rw']('foreign.pkl'), 'rb') as f:
        stored = torch.from_numpy(pickle.load(f)[0])
    base = [i for i, c in enumerate(classes) if c not in novel]
    assert len(base) == 15 and base == cfg._real_base_ids
    hand = ensembled.clone()
    hand[base] = stored[base].cuda()
    differs = (hand.view(20, -1).view(torch.int32) != ensembled.view(20, -1).view(torch.int32)).any(1)
    assert differs.nonzero().reshape(-1).tolist() == base
    r = VA.score_batches(m, supports(), images(), evaluator_of(classes, imgids), out=out, base_rw=[hand.cpu().numpy()],
                         base_rows=range(len(classes)), **result_kwargs)
    return r, classes, novel


def test_foreign_vectors_equal_score_batches_substituted_by_hand(ds, saved_cfg):
    from fewshot_detection_b200 import voc_eval as VE
    cli = tool('valid_ensemble_b200')
    voc = os.path.join(ds['devkit'], 'VOC2007')
    with open(os.path.join(voc, 'ImageSets', 'Main', 'test.txt')) as f:
        names = [l.strip() for l in f if l.strip()]
    recs = VE.load_annotations(os.path.join(voc, 'Annotations', '{}.xml'), names,
                               os.path.join(ds['devkit'], 'annotations_cache'))
    fps = [io.StringIO() for _ in range(20)]
    r, classes, novel = api_pass(ds, lambda classes, ids: VE.DeviceVocEval(classes, names, recs), fps,
                                 use_07_metric=True, novel_classes=novel_of(ds))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        cli.print_voc(r, classes, novel, True)
    lines, dirs = ds['out']['foreign']
    assert printed(buf.getvalue()) == lines and len(lines) >= 22
    assert list(dirs) == ['ene_000010']
    files = dirs['ene_000010']
    assert [fps[i].getvalue().encode() for i in range(20)] == [files['comp4_det_test_%s.txt' % c] for c in classes]
    assert files != ds['out']['plain'][1]['ene000010']            # the foreign rows reached the detector


def test_valid_batches_with_the_stored_file(ds, saved_cfg, tmp_path):
    """valid.valid_batches reading the foreign file: the command's result files, and the model's own vectors saved
    before the substitution."""
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200 import valid as VA
    m, supports, images, classes, novel, _ = api_setup(ds)
    stored = VA.load_reweighting_vectors(ds['rw']('foreign.pkl'), VA.reweighting_vector_shapes(parse_cfg(ds['cfgs'][2]), 20))
    saved = str(tmp_path / 'own.pkl')
    dw = VA.valid_batches(m, supports(), images(), classes, str(tmp_path / 'out'), 'comp4_det_test_', base_rw=stored,
                          base_rows=cfg._real_base_ids, save_rw=saved)
    assert open(saved, 'rb').read() == open(ds['rw']('own.pkl'), 'rb').read()
    assert torch.equal(dw[0][cfg._real_base_ids].cpu(), torch.from_numpy(stored[0])[cfg._real_base_ids])
    got = dict((f, open(str(tmp_path / 'out' / f), 'rb').read()) for f in sorted(os.listdir(str(tmp_path / 'out'))))
    assert got == ds['out']['foreign'][1]['ene_000010']


def novel_of(ds):
    from fewshot_detection_b200.cfg import novel_classes_of
    from fewshot_detection_b200.utils import read_data_cfg
    o = read_data_cfg(ds['cfgs'][0])
    return novel_classes_of(o['novel'], o['novelid'])


def test_foreign_vectors_coco_equal_score_batches_substituted_by_hand(ds, saved_cfg):
    from fewshot_detection_b200 import coco_eval as CE
    cli = tool('valid_ensemble_b200')
    fo = io.StringIO()
    r, classes, novel = api_pass(
        ds, lambda classes, ids: CE.DeviceCocoEval(classes, ids, CE.load_coco_annotations(ds['coco'], ids, classes)),
        fo, novel_classes=novel_of(ds))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        cli.print_coco(r, classes, novel)
    lines, dirs = ds['out']['coco_foreign']
    assert printed(buf.getvalue()) == lines and sum(l.startswith('COCO box') for l in lines) == 3
    assert dirs == {}
    assert fo.getvalue() == open(os.path.join(ds['root'], 'coco_foreign.json')).read() and len(fo.getvalue()) > 2


# ---- two processes ----------------------------------------------------------------------------------------------------
SHARDED = ('plain', 'foreign', 'files_only')


def sharded_runs(ds, tag):
    """The runs compared across process counts, each writing its vectors file to a run-specific path."""
    runs = {}
    for name in ('plain', 'foreign'):
        a = list(ds['runs'][name])
        a[a.index('--save-rw') + 1] = ds['rw']('%s_%s.pkl' % (tag, name))
        runs[name] = a
    # result files only: the command's other branch, against the scored run's files
    runs['files_only'] = ds['cfgs'] + [ds['weights'], '--write-results', '--base-rw', ds['rw']('foreign.pkl')] + SIZES
    return runs


def check_sharded(ds, tag, out):
    for name in ('plain', 'foreign'):
        assert out[name][0] == ds['out'][name][0], name
        assert out[name][1] == ds['out'][name][1], name
        with open(ds['rw']('%s_%s.pkl' % (tag, name)), 'rb') as f:
            assert f.read() == open(ds['rw']('own.pkl'), 'rb').read(), name
    assert out['files_only'][0] == []
    assert out['files_only'][1] == ds['out']['foreign'][1]


def test_two_processes_gloo_equal_one_process(ds):
    runs = sharded_runs(ds, 'gloo')
    spec = os.path.join(ds['root'], 'gloo_cases.json')
    with open(spec, 'w') as f:
        json.dump([[name, runs[name]] for name in SHARDED], f)
    outdir = os.path.join(ds['root'], 'gloo')
    os.makedirs(outdir)
    r = torchrun(29653, [os.path.abspath(__file__), spec, outdir], ROOT)
    assert r.returncode == 0 and r.stdout.count('BASE_RW_OK') == 2, r.stdout[-4000:]
    out = {}
    for name in SHARDED:
        cwd = os.path.join(outdir, name)
        out[name] = (printed(open(os.path.join(cwd, 'stdout.txt')).read()), result_dirs(cwd))
    check_sharded(ds, 'gloo', out)


def test_two_gpus_nccl_equal_one_process(ds):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    runs = sharded_runs(ds, 'nccl')
    out = dict((name, command(runs[name], os.path.join(ds['root'], 'nccl', name), port=29657)) for name in SHARDED)
    check_sharded(ds, 'nccl', out)


# ---- the training driver's checkpoint scoring -------------------------------------------------------------------------
def test_checkpoint_evaluator_with_stored_vectors(ds, saved_cfg):
    """checkpoint_evaluator(base_rw=) run by MetaTrainer on the weight file logs the command's mean / base / novel AP.
    Then MetaTrainer.fit over two checkpoint epochs of graphed steps, scoring each checkpoint with stored vectors, ends
    with the losses, parameters, momentum buffers, BatchNorm buffers and random-number states of the same run without
    scoring (the mini model and batches of test_checkpoint_evaluation_leaves_training_unchanged)."""
    from fewshot_detection_b200 import netcfg, trainer as T, valid as VA
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.optim import FusedSGD
    from fewshot_detection_b200.utils import read_data_cfg
    from seeding import seeded_init, synth_targets, synth_masks
    drv = tool('train_meta_b200')
    data_options = read_data_cfg(ds['cfgs'][0])
    det, ler = parse_cfg(ds['cfgs'][1]), parse_cfg(ds['cfgs'][2])
    cfg.config_data(data_options)
    cfg.config_meta(ler[0])
    cfg.config_net(det[0])
    assert cfg.neg_ratio == 1
    scorer = lambda stored: drv.checkpoint_evaluator(data_options, ds['devkit'], '2007', None, 1, 0, batch_size=4,
                                                     support_batch=8, base_rw=stored)
    bs, cs, K = 6, 5, 3

    def trainer(m, evaluate):
        opt = FusedSGD(m.parameters(), lr=1e-3, momentum=0.9, dampening=0, weight_decay=5e-4)
        logs, epochs = [], [0, 0]

        def queries(seen):
            epochs[0] += 1
            return Queries(epochs[0] - 1)

        def supports():
            epochs[1] += 1
            return Supports(epochs[1] - 1)
        tr = T.MetaTrainer(m, opt, 1e-3, bs, [0], [1], queries, supports, save_interval=1, world=1, log=logs.append,
                           use_graph=True, evaluate=evaluate)
        assert tr.graphed is not None
        m.models[len(m.models) - 1].verbose = False
        tr.region_loss.seen = 20000
        return tr, opt, logs

    # the weight file the command scored
    m = Darknet([dict(b) for b in det], [dict(b) for b in ler])
    m.load_weights(ds['weights'])
    m = m.cuda().train()
    stored = VA.load_reweighting_vectors(ds['rw']('foreign.pkl'), VA.reweighting_vector_shapes(ler, len(cfg.classes)))
    tr, _, logs = trainer(m, scorer(stored))
    means = dict(l.split(' = ') for l in ds['out']['foreign'][0] if l.startswith('Mean'))
    want = 'mAP %s base %s novel %s' % (means['Mean AP'], means['Mean Base AP'], means['Mean Novel AP'])
    assert tr.evaluate_checkpoint(10) == want and logs == ['evaluation at epoch 10: ' + want]
    assert m.training
    del tr, m

    def batch(it):
        g = torch.Generator().manual_seed(100 + it)
        x = torch.rand(bs, 3, 128, 128, generator=g).cuda()
        metax = torch.rand(cs, 3, 64, 64, generator=g).cuda()
        return x, metax, torch.from_numpy(synth_masks(cs, 64, 200 + it)).cuda(), torch.from_numpy(synth_targets(bs, cs, 300 + it, max_gt=2))

    class Queries(object):
        def __init__(self, epoch):
            self.epoch = epoch

        def __len__(self):
            return K

        def __iter__(self):
            for i in range(K):
                x, _, _, tgt = batch(self.epoch * K + i)
                yield x, tgt

    class Supports(object):
        batch_size = cs

        def __init__(self, epoch):
            self.epoch = epoch

        def batch(self, r):
            return batch(self.epoch * K + r.start // cs)[1:3]

    stored256 = [np.random.RandomState(5).standard_normal((20, 256, 1, 1)).astype(np.float32)]

    def run(with_eval):
        m = Darknet(netcfg.mini_dynamic_blocks(128, 8), netcfg.mini_reweighting_blocks(64, 8, 256))
        seeded_init(m, 11)
        m = m.cuda().train()
        tr, opt, logs = trainer(m, scorer(stored256) if with_eval else None)
        random.seed(77)
        np.random.seed(78)
        tr.fit(0, 2)                                             # K steps, checkpoint epoch, K steps, checkpoint epoch
        torch.cuda.synchronize()
        evals = [l for l in logs if l.startswith('evaluation at epoch')]
        return evals, ([l.item() for l in tr.losses], [p.detach().clone() for p in m.parameters()],
                       [opt.state[p]['momentum_buffer'].clone() for p in m.parameters()],
                       [b.clone() for b in m.buffers()], random.random(), float(np.random.rand()))

    evals_plain, plain = run(False)
    evals, scored = run(True)
    assert evals_plain == [] and len(evals) == 2 and all(e.split(': ')[1].startswith('mAP ') for e in evals), evals
    assert len(plain[0]) == 2 * K and np.isfinite(plain[0]).all() and plain[0] == scored[0]
    for k in (1, 2, 3):
        assert len(plain[k]) == len(scored[k]) > 0
        assert all(torch.equal(a, b) for a, b in zip(plain[k], scored[k])), k
    assert plain[4:] == scored[4:]


# ---- gloo worker: python -m torch.distributed.run --nproc-per-node=2 tests/test_gpu_base_rw.py CASES.json OUTDIR --------
def worker(spec, outdir):
    import torch.distributed as dist
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local % torch.cuda.device_count())
    dist.init_process_group('gloo')
    cli = tool('valid_ensemble_b200')
    with open(spec) as f:
        cases = json.load(f)
    for name, argv in cases:
        cwd = os.path.join(outdir, name)
        if rank == 0:
            os.makedirs(cwd)
        dist.barrier()
        os.chdir(cwd)                                            # the result files go to ./results
        args, base_rw = cli.parse_args(argv)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            cli.run(args, world, rank, base_rw)
        if rank == 0:
            with open('stdout.txt', 'w') as f:
                f.write(buf.getvalue())
        dist.barrier()
    print('BASE_RW_OK rank %d' % rank, flush=True)
    torch.cuda.synchronize()
    dist.destroy_process_group()


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    worker(sys.argv[1], sys.argv[2])

"""Sharded evaluation over two processes (tests/eval_shard_worker.py, launched with torch.distributed.run):
  * with NCCL, one GPU per rank (needs 2 GPUs);
  * with gloo, the two ranks sharing one GPU: the same collectives' logic on a single-GPU machine;
and the evaluation command tools/valid_ensemble_b200.py on a synthetic data set written to a temp dir (PIL-written
JPEGs, VOC XMLs, the `.data` file with its `valid` list, support dictionary and per-class label files): the same AP
lines and byte-identical result files in one process and, with 2 GPUs, in two."""
import importlib.util
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, 'tests', 'eval_shard_worker.py')
TOOL = os.path.join(ROOT, 'tools', 'valid_ensemble_b200.py')


def torchrun(port, args, cwd=None, timeout=600):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr',
           '127.0.0.1', '--master-port', str(port)] + args
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout, cwd=cwd)


def test_two_gpus_nccl_sharded_equals_one_process():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    r = torchrun(29633, [WORKER, 'nccl'])
    assert r.returncode == 0 and r.stdout.count('SHARD_OK') == 2, r.stdout[-4000:]


def test_two_processes_gloo_score_batches_equals_one_process():
    r = torchrun(29637, [WORKER, 'gloo'])
    assert r.returncode == 0 and r.stdout.count('SHARD_OK') == 2, r.stdout[-4000:]


def write_data_set(root, n_img=30):
    """tools/e2e_train_synth.py's JPEG set (labels, support dictionary, per-class label files) plus a devkit with
    one annotation per image (its label boxes, some difficult), mini network cfgs and a seeded weight file."""
    spec = importlib.util.spec_from_file_location('e2e_train_synth', os.path.join(ROOT, 'tools', 'e2e_train_synth.py'))
    synth = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(synth)
    synth.make_dataset(root, n_img)
    from PIL import Image
    voc = os.path.join(root, 'devkit', 'VOC2007')
    os.makedirs(os.path.join(voc, 'Annotations'))
    os.makedirs(os.path.join(voc, 'ImageSets', 'Main'))
    obj = ('<object><name>%s</name><pose>Unspecified</pose><truncated>0</truncated><difficult>%d</difficult>'
           '<bndbox><xmin>%d</xmin><ymin>%d</ymin><xmax>%d</xmax><ymax>%d</ymax></bndbox></object>')
    names = []
    for i in range(n_img):
        name = '%06d' % i
        W, H = Image.open(os.path.join(root, 'JPEGImages', name + '.jpg')).size
        objs = []
        with open(os.path.join(root, 'labels', name + '.txt')) as f:
            for k, l in enumerate(f):
                c, x, y, w, h = [float(v) for v in l.split()]
                objs.append(obj % (synth.VOC[int(c)], int(k == 2), int((x - w / 2) * W) + 1, int((y - h / 2) * H) + 1,
                                   int((x + w / 2) * W), int((y + h / 2) * H)))
        with open(os.path.join(voc, 'Annotations', name + '.xml'), 'w') as f:
            f.write('<annotation><filename>%s.jpg</filename>%s</annotation>' % (name, ''.join(objs)))
        names.append(name)
    with open(os.path.join(voc, 'ImageSets', 'Main', 'test.txt'), 'w') as f:
        f.write('\n'.join(names) + '\n')
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden'))
    from seeding import seeded_init
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.darknet_meta import Darknet
    det, ler = netcfg.mini_dynamic_blocks(128, 16), netcfg.mini_reweighting_blocks(64, 16, 512)
    netcfg.write_cfg(det, os.path.join(root, 'det.cfg'))
    netcfg.write_cfg(ler, os.path.join(root, 'ler.cfg'))
    m = Darknet([dict(b) for b in det], [dict(b) for b in ler])
    seeded_init(m, 3)
    os.makedirs(os.path.join(root, 'backup'))
    m.save_weights(os.path.join(root, 'backup', '000010.weights'))
    with open(os.path.join(root, 'meta.data'), 'w') as f:
        f.write('metayolo=1\nmetain_type=2\ndata=voc\nneg = 1\nrand = 0\nnovel = %s\nnovelid = 0\nmeta = %s\n'
                'train = %s\nvalid = %s\nbackup = %s\ngpus=0\n' % (
                    os.path.join(root, 'novels.txt'), os.path.join(root, 'lists', 'dict_full.txt'),
                    os.path.join(root, 'lists', 'train.txt'), os.path.join(root, 'lists', 'train.txt'),
                    os.path.join(root, 'backup')))
    return [os.path.join(root, 'meta.data'), os.path.join(root, 'det.cfg'), os.path.join(root, 'ler.cfg'),
            os.path.join(root, 'backup', '000010.weights'), '--devkit', os.path.join(root, 'devkit'), '--write-results',
            '--batch-size', '4', '--support-batch', '8']


def run_tool(args, cwd, two):
    os.makedirs(cwd)
    if two:
        r = torchrun(29641, [TOOL] + args, cwd=cwd)
    else:
        r = subprocess.run([sys.executable, TOOL] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           timeout=600, cwd=cwd)
    assert r.returncode == 0, r.stdout[-4000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith(('AP for', 'Mean', 'VOC07'))]
    out = os.path.join(cwd, 'results', 'backup', 'ene000010')
    files = dict((f, open(os.path.join(out, f), 'rb').read()) for f in sorted(os.listdir(out)))
    return lines, files


def test_evaluation_command_one_and_two_processes(tmp_path):
    """With 2 GPUs the two-process run goes first, on a devkit without annotation cache: rank 0 writes the cache
    while the other rank waits, then reads it."""
    args = write_data_set(str(tmp_path / 'data'))
    two = torch.cuda.device_count() >= 2
    if two:
        lines2, files2 = run_tool(args, str(tmp_path / 'two'), True)
    lines1, files1 = run_tool(args, str(tmp_path / 'one'), False)
    assert len(lines1) >= 22 and len(files1) == 20 and sum(len(v) for v in files1.values()) > 0, lines1
    if not two:
        pytest.skip('the two-process run needs 2 GPUs')
    assert lines2 == lines1
    assert files2 == files1

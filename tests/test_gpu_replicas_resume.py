"""Resuming a replica run from its state file on the GPU, byte for byte: tools/train_meta_b200.py --replicas 4 on the
synthetic VOC set (tests/resume_worker.py, base training, neg = 1, multi-scale sizes drawn), run for four epochs
uninterrupted, then stopped after epoch 2 and continued with --resume.  The resumed run rebuilds the same 4-replica
support index, draws the same rows and writes the same weight files, state files and per-step losses from epoch 3 on.
The state files record the replica count."""
import os
import shutil

import pytest

from test_gpu_resume import WORKER, _backup, _env, _read, _run, _same_files, _worker

pytestmark = pytest.mark.gpu
FLAGS = ['--replicas', '4', '--save-state']


def _train(root, name, stop=0, resume=None, flags=FLAGS):
    out = os.path.join(root, 'out', name)
    backup = _backup(root, 'base')
    if resume is None:
        if os.path.isdir(backup):
            shutil.rmtree(backup)
        args = [os.path.join(root, 'init.weights')]
    else:
        args = [os.path.join(backup, '%06d.weights' % resume), '--resume', os.path.join(backup, '%06d.state' % resume)]
    return _run(_worker(1) + ['run', root, 'base', out, str(stop)] + args + flags, _env(), root), out


def test_resumed_replica_run_equals_uninterrupted(tmp_path):
    import sys
    from fewshot_detection_b200 import resume as R
    root = str(tmp_path)
    _run([sys.executable, WORKER, 'setup', root, 'base'], _env(), root)
    log, out = _train(root, 'full')
    assert '4 replicas per step, 4 per rank on 1 rank(s): 16 query images' in log, log[-3000:]
    full_files, full_steps = _read(out)
    epochs = sorted({int(e) for e, _, _ in full_steps})
    assert len(epochs) == 4 and len(full_steps) >= 8
    assert len({s for _, s, _ in full_steps}) > 1, 'the multi-scale schedule drew only one input size'
    last = os.path.join(out, 'files', '%06d.state' % (epochs[-1] + 1))
    assert R.read_state(last)['fingerprint']['replicas'] == 4

    _, stopped = _train(root, 'stopped', stop=2)
    stopped_files, stopped_steps = _read(stopped)
    assert stopped_steps == [s for s in full_steps if int(s[0]) in epochs[:2]]
    mid = epochs[1] + 1
    _, resumed = _train(root, 'resumed', resume=mid)
    resumed_files, resumed_steps = _read(resumed)
    assert resumed_steps == [s for s in full_steps if int(s[0]) in epochs[2:]]
    later = ['%06d.%s' % (e + 1, k) for e in epochs[2:] for k in ('weights', 'state')]
    bad = _same_files(resumed_files, full_files, later, root)
    assert not bad, ('resumed', bad)

"""Resuming the training driver from a state file on the GPU, byte for byte (tests/resume_worker.py runs
tools/train_meta_b200.py on the synthetic VOC set of tools/e2e_train_synth.py, background preparation on):

  * two uninterrupted 4-epoch runs with the same FSDET_SEED write the same weight files, state files and per-step
    losses (the seeded run is reproducible with the worker thread preparing batches);
  * a run stopped after epoch 2 and continued with --resume writes the same bytes from epoch 3 on;
  * the run with FSDET_NO_BG_PREP=1 (serial preparation) equals the threaded one;
  * the starting weights say seen = 256000, so the multi-scale schedule draws input sizes: more than one occurs;
for the base-training protocol (neg = 1) and for fine-tuning (tuning = 1, neg = 0), and under torchrun with two GPUs.

Also FusedSGD.load_state_dict before and after a CUDA-graph capture of its step."""
import os
import shutil
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
WORKER = os.path.join(HERE, 'resume_worker.py')

pytestmark = pytest.mark.gpu


def _env(**kw):
    env = dict(os.environ, FSDET_SEED='5')
    env.pop('FSDET_NO_BG_PREP', None)
    env.update(kw)
    return env


def _run(cmd, env, cwd):
    r = subprocess.run(cmd, env=env, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-6000:]
    return r.stdout


def _worker(world):
    if world == 1:
        return [sys.executable, WORKER]
    return [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(world), WORKER]


def _train(root, mode, name, world, stop=0, resume=None, **env):
    """One driver run from the starting weights, or with resume = epoch from that epoch's weight and state files;
    returns its output directory.  A run that does not resume starts from an empty backup directory."""
    out = os.path.join(root, 'out', name)
    backup = _backup(root, mode)
    if resume is None:
        if os.path.isdir(backup):
            shutil.rmtree(backup)
        flags = [os.path.join(root, 'init.weights')]
    else:
        flags = [os.path.join(backup, '%06d.weights' % resume), '--resume', os.path.join(backup, '%06d.state' % resume)]
    _run(_worker(world) + ['run', root, mode, out, str(stop)] + flags + ['--save-state'], _env(**env), root)
    return out


def _backup(root, mode):
    return os.path.join(root, 'backup_novel0_neg%d' % (1 if mode == 'base' else 0))


def _read(out):
    files = os.path.join(out, 'files')
    with open(os.path.join(out, 'steps.txt')) as f:
        steps = [l.split() for l in f.read().splitlines()]
    return {n: open(os.path.join(files, n), 'rb').read() for n in sorted(os.listdir(files))}, steps


def _state_diff(a, b, where=''):
    """Paths of the fields in which two decoded states differ."""
    if torch.is_tensor(a) and torch.is_tensor(b):
        return [] if a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b) else [where]
    if isinstance(a, dict) and isinstance(b, dict):
        if set(a) != set(b):
            return [where + ' keys']
        return sum((_state_diff(a[k], b[k], '%s/%s' % (where, k)) for k in a), [])
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)) and len(a) == len(b):
        return sum((_state_diff(x, y, '%s[%d]' % (where, i)) for i, (x, y) in enumerate(zip(a, b))), [])
    return [] if a == b else [where]


def _same_files(got, want, names, tmp):
    """Byte equality of the named files; a message naming what differs (for state files: which fields)."""
    from fewshot_detection_b200 import resume as R
    bad = []
    for n in names:
        if got.get(n) == want.get(n):
            continue
        detail = ''
        if n.endswith('.state') and n in got and n in want:
            states = []
            for k, blob in (('got', got[n]), ('want', want[n])):
                path = os.path.join(tmp, k + '_' + n)
                with open(path, 'wb') as f:
                    f.write(blob)
                states.append(R.read_state(path))
            detail = ' fields %s' % _state_diff(*states)[:8]
        bad.append(n + detail)
    return bad


def _check_resume(tmp_path, mode, world):
    root = str(tmp_path)
    _run([sys.executable, WORKER, 'setup', root, mode], _env(), root)
    full_files, full_steps = _read(_train(root, mode, 'full', world))
    epochs = sorted({int(e) for e, _, _ in full_steps})
    assert len(epochs) == 4 and len(full_steps) >= 8
    assert len({s for _, s, _ in full_steps}) > 1, 'the multi-scale schedule drew only one input size'
    names = ['%06d.weights' % (e + 1) for e in epochs] + ['%06d.state' % (e + 1) for e in epochs]
    assert sorted(full_files) == sorted(names)
    backup = _backup(root, mode)
    assert sorted(f for f in os.listdir(backup) if f.endswith('.state')) == ['%06d.state' % (epochs[-1] + 1)]

    if world == 1:                  # the same seed again, threaded, then serially prepared: the same bytes
        for name, env in (('again', {}), ('serial', dict(FSDET_NO_BG_PREP='1'))):
            files, steps = _read(_train(root, mode, name, world, **env))
            assert steps == full_steps, name
            assert sorted(files) == sorted(full_files), (name, sorted(files))
            bad = _same_files(files, full_files, sorted(files), root)
            assert not bad, (name, bad)

    stopped_files, stopped_steps = _read(_train(root, mode, 'stopped', world, stop=2))
    assert stopped_steps == [s for s in full_steps if int(s[0]) in epochs[:2]]
    mid = epochs[1] + 1
    resumed_files, resumed_steps = _read(_train(root, mode, 'resumed', world, resume=mid))
    assert resumed_steps == [s for s in full_steps if int(s[0]) in epochs[2:]]
    later = ['%06d.%s' % (e + 1, k) for e in epochs[2:] for k in ('weights', 'state')]
    bad = _same_files(resumed_files, full_files, later, root)
    assert not bad, ('resumed', bad)


@pytest.mark.parametrize('mode', ['base', 'tune'])
def test_resumed_driver_run_equals_uninterrupted(tmp_path, mode):
    _check_resume(tmp_path, mode, 1)


@pytest.mark.parametrize('mode', ['base', 'tune'])
def test_resumed_two_gpu_driver_run_equals_uninterrupted(tmp_path, mode):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs, %d present' % torch.cuda.device_count())
    _check_resume(tmp_path, mode, 2)


def test_fused_sgd_load_state_dict_before_and_after_capture():
    """Momentum loaded into a fresh FusedSGD (buffers created) and into one whose step is captured in a CUDA graph
    (buffers overwritten in place, the graph's pointers stay valid): both continue exactly as the optimizer the state
    came from."""
    from fewshot_detection_b200.optim import FusedSGD
    g = torch.Generator().manual_seed(3)
    shapes = [(64, 32, 3, 3), (64,), (1000,)]
    init = [torch.randn(s, generator=g) for s in shapes]
    grads = [[torch.randn(s, generator=g).cuda() for s in shapes] for _ in range(6)]

    def make():
        ps = [t.clone().cuda().requires_grad_() for t in init]
        return ps, FusedSGD(ps, lr=0.01, momentum=0.9, dampening=0, weight_decay=5e-4)

    def step(ps, opt, k):
        for p, gr in zip(ps, grads[k]):
            p.grad = gr.clone()
        opt.step()

    ref_p, ref = make()
    for k in range(3):
        step(ref_p, ref, k)
    sd = ref.state_dict()
    sd['state'] = {i: {'momentum_buffer': s['momentum_buffer'].cpu()} for i, s in sd['state'].items()}
    saved_p = [p.detach().clone() for p in ref_p]
    for k in range(3, 6):
        step(ref_p, ref, k)

    # before a capture: no buffers yet
    ps, opt = make()
    with torch.no_grad():
        for p, s in zip(ps, saved_p):
            p.copy_(s)
    opt.load_state_dict(sd)
    for k in range(3, 6):
        step(ps, opt, k)
    assert all(torch.equal(a, b) for a, b in zip(ps, ref_p))

    # after a capture: the step graph keeps addressing the same buffers
    ps, opt = make()
    for p, gr in zip(ps, grads[0]):
        p.grad = gr.clone()
    opt.step()
    opt.capturable = True
    opt.sync_hyper()
    opt.prepare()
    bufs = [opt.state[p]['momentum_buffer'] for p in ps]
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    with torch.no_grad():
        for p, s in zip(ps, saved_p):
            p.copy_(s)
    opt.load_state_dict(sd)
    assert all(opt.state[p]['momentum_buffer'] is b for p, b in zip(ps, bufs))
    for k in range(3, 6):
        for p, gr in zip(ps, grads[k]):
            p.grad.copy_(gr)
        opt.sync_hyper()
        graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(ps, ref_p))

    stale = {'state': {}, 'param_groups': sd['param_groups']}
    with pytest.raises(ValueError, match='without momentum'):
        opt.load_state_dict(stale)

"""Test-time augmentation on the host (CPU): the plan checks, the commands' refusals of bad sides before any CUDA work,
the `_tta` result prefix, and what ptxas makes of the new kernels (no spills)."""
import os
import re
import subprocess

import pytest

from test_conv_tc_ptxas import _build_flags, _nvcc
from test_detect_command import tool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tta_plan():
    from fewshot_detection_b200 import valid as VA
    assert VA.tta_plan([416, 544, 608], True) == [(416, 0), (416, 1), (544, 0), (544, 1), (608, 0), (608, 1)]
    assert VA.tta_plan([608, 320]) == [(608, 0), (320, 0)]
    assert VA.parse_tta_sides('416, 544,608') == [416, 544, 608]
    for bad in ([], [416, 400], [416, 416], [0], [-32]):
        with pytest.raises(ValueError):
            VA.tta_plan(bad)
    for bad in ('', '416,x', '416,,416', '33'):
        with pytest.raises(ValueError):
            VA.parse_tta_sides(bad)
    assert VA.check_tta_passes([(416, 0), (416, 1)]) == [(416, 0), (416, 1)]
    for bad in ([], [(416, 0), (416, 0)], [(416, 2)], [(100, 0)]):
        with pytest.raises(ValueError):
            VA.check_tta_passes(bad)


def _files(tmp_path):
    paths = []
    for name in ('det.cfg', 'ler.cfg', 'w.weights', 'c.names', 'x.data', 'img.png'):
        p = str(tmp_path / name)
        with open(p, 'w') as f:
            f.write('cat\n' if name == 'c.names' else '')
        paths.append(p)
    return paths


@pytest.mark.parametrize('sides', ['416,400', '416,416', '', '416,abc'])
def test_commands_refuse_bad_sides_before_cuda(tmp_path, monkeypatch, capsys, sides):
    import torch
    det, ler, w, names, data, img = _files(tmp_path)

    def no_cuda(*a, **k):
        raise AssertionError('CUDA work before the arguments were checked')
    monkeypatch.setattr(torch.cuda, 'set_device', no_cuda)
    with pytest.raises(SystemExit):
        tool('detect_b200').main([det, ler, w, img, '--rw', w, '--names', names, '--tta-sides', sides])
    assert '--tta-sides' in capsys.readouterr().err
    with pytest.raises(SystemExit):
        tool('valid_ensemble_b200').main([data, det, ler, w, '--write-results', '--tta-sides', sides])
    assert '--tta-sides' in capsys.readouterr().err


def test_result_files_go_under_the_tta_prefix():
    ve, dt = tool('valid_ensemble_b200'), tool('detect_b200')
    w = os.path.join('backup', 'model_000010.weights')
    assert ve.result_prefix(w) == os.path.join('results', 'backup', 'ene' + 'model_000010')
    assert ve.result_prefix(w, tta=True) == os.path.join('results', 'backup', 'enemodel_000010_tta')
    assert ve.result_prefix(w, True, True) == os.path.join('results', 'backup', 'ene_model_000010_tta')

    class Args(object):
        out, tta = 'detections', None
    assert dt.output_dir(Args) == 'detections'
    Args.tta = [(416, 0), (416, 1)]
    assert dt.output_dir(Args) == 'detections_tta'


NEW_KERNELS = ('tta_merge_kernel', 'nms_merged_', 'MergedRows')


def test_new_kernels_do_not_spill(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not found')
    checked, spills = 0, []
    for name in ('detect.cu', 'voc_eval.cu', 'coco_eval.cu'):
        src = os.path.join(ROOT, 'fewshot_detection_b200', 'csrc', name)
        cmd = [nvcc] + _build_flags() + ['-Xptxas', '-v', '-c', src, '-o', str(tmp_path / (name + '.o'))]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout[-4000:]
        func = None
        for line in r.stdout.splitlines():
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m:
                func = m.group(1)
                continue
            m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
            if m and func and any(k in func for k in NEW_KERNELS):
                checked += 1
                if int(m.group(1)) or int(m.group(2)):
                    spills.append('%s: %s' % (func, line.strip()))
                func = None
    # merge, compact, keys, suppress; the merged selection's keys and write; the VOC and COCO gathers
    assert checked >= 8, checked
    assert not spills, 'register spills:\n' + '\n'.join(spills)

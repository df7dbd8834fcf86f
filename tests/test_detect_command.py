"""The host side of the detection command (CPU): the reference utils names the drop-in module must provide, the image
header sizes, the class names file, and the command's refusals, which all happen before any CUDA work."""
import importlib.util
import os
import pickle
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# the functions of the reference's utils.py that its valid_ensemble.py and valid.py call (`from utils import *`)
VALID_UTILS_NAMES = ['get_image_size', 'get_region_boxes', 'get_region_boxes_v2', 'load_class_names', 'nms',
                     'read_data_cfg']


def test_dropin_utils_exposes_what_the_reference_validation_scripts_use():
    sys.path.insert(0, os.path.join(ROOT, 'dropin'))
    try:
        spec = importlib.util.spec_from_file_location('dropin_utils', os.path.join(ROOT, 'dropin', 'utils.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path.pop(0)
    star = {}
    exec('from fewshot_detection_b200.utils import *', star)
    for name in VALID_UTILS_NAMES:
        assert callable(getattr(mod, name)), name
    assert 'get_image_size' in star and 'load_class_names' in star


@pytest.mark.parametrize('fmt,size', [('PNG', (37, 23)), ('JPEG', (640, 427)), ('JPEG', (1, 1)), ('PNG', (1000, 3))])
def test_get_image_size_reads_the_header(tmp_path, fmt, size):
    from PIL import Image
    from fewshot_detection_b200.utils import get_image_size
    path = str(tmp_path / ('img.' + fmt.lower()))
    arr = np.random.RandomState(size[0]).randint(0, 256, (size[1], size[0], 3)).astype(np.uint8)
    Image.fromarray(arr).save(path, fmt)
    assert get_image_size(path) == size


def test_get_image_size_of_other_files_is_none(tmp_path):
    from fewshot_detection_b200.utils import get_image_size
    short = tmp_path / 'short.jpg'
    short.write_bytes(b'\xff\xd8\xff\xe0')
    text = tmp_path / 'a.txt'
    text.write_text('not an image at all, just some text\n')
    assert get_image_size(str(short)) is None and get_image_size(str(text)) is None


def test_load_class_names(tmp_path):
    from fewshot_detection_b200.utils import load_class_names
    p = tmp_path / 'c.names'
    p.write_text('aeroplane\ntraffic light  \nsofa\n')
    assert load_class_names(str(p)) == ['aeroplane', 'traffic light', 'sofa']


def command_files(root, n_names=3, C=512):
    """Mini cfgs whose reweighting vectors are 512 wide, a names file, a vectors file and an image."""
    from PIL import Image
    from fewshot_detection_b200 import netcfg
    netcfg.write_cfg(netcfg.mini_dynamic_blocks(128, 16), os.path.join(root, 'det.cfg'))
    netcfg.write_cfg(netcfg.mini_reweighting_blocks(64, 16, 512), os.path.join(root, 'ler.cfg'))
    open(os.path.join(root, 'w.weights'), 'wb').close()
    with open(os.path.join(root, 'c.names'), 'w') as f:
        f.write(''.join('class%d\n' % i for i in range(n_names)))
    with open(os.path.join(root, 'rw.pkl'), 'wb') as f:
        pickle.dump([np.ones((3, C, 1, 1), np.float32)], f)
    Image.fromarray(np.zeros((20, 30, 3), np.uint8)).save(os.path.join(root, 'a.jpg'))
    return [os.path.join(root, f) for f in ('det.cfg', 'ler.cfg', 'w.weights', 'a.jpg')]


@pytest.fixture()
def no_cuda(monkeypatch):
    """Any CUDA work in the command fails the test."""
    import torch

    def refuse(*a, **k):
        raise AssertionError('CUDA work before the arguments were checked')
    monkeypatch.setattr(torch.cuda, 'set_device', refuse)
    cli = tool('detect_b200')
    monkeypatch.setattr(cli, 'run', refuse)
    return cli


def refusal(cli, args, capsys):
    with pytest.raises(SystemExit) as e:
        cli.main(args)
    assert e.value.code == 2
    return capsys.readouterr().err


def test_command_refuses_vectors_that_do_not_fit_the_cfgs_or_the_names(tmp_path, no_cuda, capsys):
    cli = no_cuda
    root = str(tmp_path)
    base = command_files(root)
    names, rw = os.path.join(root, 'c.names'), os.path.join(root, 'rw.pkl')
    # the vectors are 512 wide and 3 rows: 4 names do not fit
    with open(os.path.join(root, 'c4.names'), 'w') as f:
        f.write('a\nb\nc\nd\n')
    err = refusal(cli, base + ['--rw', rw, '--names', os.path.join(root, 'c4.names')], capsys)
    assert '(4, 512, 1, 1)' in err and '(3, 512, 1, 1)' in err and '4 names' in err, err
    # 1024-wide vectors do not fit the reweighting net
    with open(os.path.join(root, 'c1024.pkl'), 'wb') as f:
        pickle.dump([np.ones((3, 1024, 1, 1), np.float32)], f)
    err = refusal(cli, base + ['--rw', os.path.join(root, 'c1024.pkl'), '--names', names], capsys)
    assert '(3, 512, 1, 1)' in err and '(3, 1024, 1, 1)' in err, err
    # not a pickle
    with open(os.path.join(root, 'junk.pkl'), 'w') as f:
        f.write('junk')
    assert 'junk.pkl' in refusal(cli, base + ['--rw', os.path.join(root, 'junk.pkl'), '--names', names], capsys)
    # the source of the vectors
    assert '--rw PATH --names FILE' in refusal(cli, base, capsys)
    assert '--rw PATH --names FILE' in refusal(cli, base + ['--rw', rw, '--names', names, '--data', names], capsys)
    assert '--rw needs --names' in refusal(cli, base + ['--rw', rw], capsys)
    assert 'missing.pkl' in refusal(cli, base + ['--rw', os.path.join(root, 'missing.pkl'), '--names', names], capsys)
    assert 'no such image' in refusal(cli, base[:3] + [os.path.join(root, 'none.jpg'), '--rw', rw, '--names', names],
                                      capsys)
    assert '--max-det' in refusal(cli, base + ['--rw', rw, '--names', names, '--max-det', '0'], capsys)
    # and a fitting file passes the checks
    args, got_names, rws, images = cli.parse_args(base + ['--rw', rw, '--names', names])
    assert got_names == ['class0', 'class1', 'class2'] and rws[0].shape == (3, 512, 1, 1) and images == [base[3]]


def test_command_lists_files_directories_and_lists(tmp_path):
    cli = tool('detect_b200')
    d = tmp_path / 'dir'
    d.mkdir()
    for n in ('b.png', 'a.jpg', 'c.JPEG', 'notes.md'):
        (d / n).write_bytes(b'')
    lst = tmp_path / 'list.txt'
    lst.write_text('/x/1.jpg\n\n/x/2.png\n')
    got = cli.list_images([str(tmp_path / 'one.jpg'), str(d), str(lst)])
    assert got == [str(tmp_path / 'one.jpg'), str(d / 'a.jpg'), str(d / 'b.png'), str(d / 'c.JPEG'), '/x/1.jpg', '/x/2.png']


def test_command_lines_read_back_exactly():
    cli = tool('detect_b200')
    row = ('traffic light', 0.1 + 0.2, 1 / 3.0, 2.5e-7, 1e5 / 7, 640.0)
    line = cli.format_line(row)
    fields = line.rstrip('\n').rsplit(' ', 5)
    assert fields[0] == row[0] and [float(v) for v in fields[1:]] == list(row[1:])

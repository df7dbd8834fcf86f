"""The reference's stored reweighting vectors (valid_ensemble.py:102-119, `use_baserw`), CPU only:
  * valid.save_reweighting_vectors / load_reweighting_vectors: the reference's file (a pickled list of one float32
    [n_cls, C, 1, 1] array per dynamic layer), also as Python 2 wrote it, and ValueError for files that do not fit;
  * valid.substitute_base_rows with the rows of the evaluation command (cfg._real_base_ids) for a fine-tuning and a
    base-training `.data` file: the 15 base rows of 20, and no novel row;
  * tools/valid_ensemble_b200.py: the result prefix ene_<ckpt>, and a missing or misfitting --base-rw file refused
    before any GPU work; tools/train_meta_b200.py refuses --eval-base-rw without an evaluation flag."""
import importlib.util
import io
import os
import pickle
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOVELS = 'bird,bus,cow,motorbike,sofa\naeroplane,bottle,cow,horse,sofa\nboat,cat,motorbike,sheep,sofa\n'
BASE0 = [0, 1, 3, 4, 6, 7, 8, 10, 11, 12, 14, 15, 16, 18, 19]          # the base ids of novel split 0


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def vectors(n_cls=20, C=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n_cls, C, 1, 1, generator=g)]


class Py2Pickler(pickle._Pickler):
    """Protocol 2 as Python 2's pickle writes a list of numpy arrays: every string as an 8-bit str (the array bytes
    included, which Python 3 reads only with encoding='latin1') and numpy's reconstructor under numpy.core."""
    dispatch = dict(pickle._Pickler.dispatch)

    def save_bytes(self, obj):
        n = len(obj)
        self.write(pickle.SHORT_BINSTRING + bytes([n]) + obj if n < 256 else pickle.BINSTRING + struct.pack('<i', n) + obj)
        self.memoize(obj)
    dispatch[bytes] = save_bytes

    def save_str(self, obj):
        self.save_bytes(obj.encode('latin1'))
    dispatch[str] = save_str

    def save_global(self, obj, name=None):
        mod, name = obj.__module__, name or obj.__qualname__
        if mod.startswith('numpy._core'):
            mod = 'numpy.core' + mod[len('numpy._core'):]
        self.write(pickle.GLOBAL + mod.encode() + b'\n' + name.encode() + b'\n')
        self.memoize(obj)
    dispatch[type] = save_global


@pytest.fixture()
def saved_cfg():
    from fewshot_detection_b200.cfg import cfg
    saved = dict(cfg)
    yield cfg
    cfg.clear()
    cfg.update(saved)


def test_save_then_load_returns_the_vectors(tmp_path):
    from fewshot_detection_b200 import valid as VA
    dw = vectors()
    p = str(tmp_path / 'voc_novel0_.pkl')
    VA.save_reweighting_vectors(p, dw)
    with open(p, 'rb') as f:
        plain = pickle.load(f)
    assert isinstance(plain, list) and len(plain) == 1
    assert isinstance(plain[0], np.ndarray) and plain[0].dtype == np.float32 and plain[0].shape == (20, 64, 1, 1)
    assert np.array_equal(plain[0], dw[0].numpy())
    got = VA.load_reweighting_vectors(p, [(20, 64, 1, 1)])
    assert len(got) == 1 and got[0].dtype == np.float32 and np.array_equal(got[0], dw[0].numpy())
    assert np.array_equal(VA.load_reweighting_vectors(p)[0], dw[0].numpy())      # without shapes: the same list


def test_protocol_2_and_python_2_pickles_load(tmp_path):
    from fewshot_detection_b200 import valid as VA
    a = [vectors(seed=1)[0].numpy()]
    p2 = tmp_path / 'p2.pkl'
    p2.write_bytes(pickle.dumps(a, protocol=2))
    assert np.array_equal(VA.load_reweighting_vectors(str(p2), [(20, 64, 1, 1)])[0], a[0])
    buf = io.BytesIO()
    Py2Pickler(buf, 2).dump(a)
    py2 = tmp_path / 'py2.pkl'
    py2.write_bytes(buf.getvalue())
    with pytest.raises(UnicodeDecodeError):                   # the array bytes are not ASCII
        pickle.loads(buf.getvalue())
    got = VA.load_reweighting_vectors(str(py2), [(20, 64, 1, 1)])
    assert got[0].dtype == np.float32 and np.array_equal(got[0], a[0])


@pytest.mark.parametrize('case,content,named', [
    ('not a list', {'rws': np.zeros((20, 64, 1, 1), np.float32)}, 'dict'),
    ('a tuple', (np.zeros((20, 64, 1, 1), np.float32),), 'tuple'),
    ('tensors', [torch.zeros(20, 64, 1, 1)], 'Tensor'),
    ('two layers', [np.zeros((20, 64, 1, 1), np.float32)] * 2, '(20, 64, 1, 1), (20, 64, 1, 1)]'),
    ('no layer', [], 'shapes []'),
    ('wrong n_cls', [np.zeros((15, 64, 1, 1), np.float32)], '(15, 64, 1, 1)'),
    ('wrong C', [np.zeros((20, 1024, 1, 1), np.float32)], '(20, 1024, 1, 1)'),
    ('flat rows', [np.zeros((20, 64), np.float32)], '(20, 64)'),
    ('float64', [np.zeros((20, 64, 1, 1), np.float64)], 'float64'),
    ('nan', [np.where(np.arange(1280).reshape(20, 64, 1, 1) == 77, np.nan, 0).astype(np.float32)], 'non-finite'),
    ('inf', [np.where(np.arange(1280).reshape(20, 64, 1, 1) == 5, -np.inf, 0).astype(np.float32)], 'non-finite'),
])
def test_a_file_that_does_not_fit_raises(tmp_path, case, content, named):
    from fewshot_detection_b200 import valid as VA
    p = str(tmp_path / 'bad.pkl')
    with open(p, 'wb') as f:
        pickle.dump(content, f)
    with pytest.raises(ValueError) as e:
        VA.load_reweighting_vectors(p, [(20, 64, 1, 1)])
    msg = str(e.value)
    assert p in msg and named in msg, (case, msg)
    if case not in ('nan', 'inf'):
        assert '(20, 64, 1, 1)' in msg, (case, msg)                # the expected shape
    if case in ('nan', 'inf'):
        assert '(20, 64, 1, 1)' in msg                             # the layer's shape


def test_a_file_that_is_not_a_pickle_raises(tmp_path):
    from fewshot_detection_b200 import valid as VA
    p = tmp_path / 'junk.pkl'
    p.write_bytes(b'\x00not a pickle')
    with pytest.raises(ValueError, match='junk.pkl'):
        VA.load_reweighting_vectors(str(p), [(20, 64, 1, 1)])
    p.write_bytes(pickle.dumps([np.zeros((20, 64, 1, 1), np.float32)])[:-20])
    with pytest.raises(ValueError, match='junk.pkl'):
        VA.load_reweighting_vectors(str(p), [(20, 64, 1, 1)])


def test_reweighting_vector_shapes_of_the_shipped_and_mini_nets():
    from fewshot_detection_b200 import netcfg, valid as VA
    assert VA.reweighting_vector_shapes(netcfg.reweighting_net_blocks(), 20) == [(20, 1024, 1, 1)]
    assert VA.reweighting_vector_shapes(netcfg.mini_reweighting_blocks(64, 16, 512), 80) == [(80, 512, 1, 1)]


@pytest.mark.parametrize('tuning', [True, False])
def test_substituted_rows_are_the_base_classes(tmp_path, saved_cfg, tuning):
    """cfg/metatune.data (fine-tuning: every class is trained, so cfg.base_ids is all 20) and cfg/metayolo.data (base
    training) with novelid = 0: the rows replaced are the 15 classes that are not novel, in both."""
    from fewshot_detection_b200 import valid as VA
    cfg = saved_cfg
    novels = tmp_path / 'voc_novels.txt'
    novels.write_text(NOVELS)
    opts = {'metayolo': '1', 'metain_type': '2', 'data': 'voc', 'neg': '1', 'rand': '0', 'novel': str(novels),
            'novelid': '0', 'meta': 'data/voc_traindict_full.txt', 'backup': 'backup/metayolo', 'gpus': '1,2,3,4'}
    if tuning:
        opts.update(tuning='1', neg='0', max_epoch='2000', repeat='200', dynamic='0', scale='1',
                    meta='data/voc_traindict_bbox_5shot.txt', backup='backup/metatunetest1')
    cfg.tuning = False
    cfg.config_data(opts)
    assert len(cfg.classes) == 20 and cfg.novel_classes == ['bird', 'bus', 'cow', 'motorbike', 'sofa']
    assert cfg.base_ids == (list(range(20)) if tuning else BASE0)
    assert cfg._real_base_ids == BASE0
    dw, stored = vectors(seed=2), [vectors(seed=3)[0].numpy()]
    before = dw[0].clone()
    out = VA.substitute_base_rows(dw, stored, cfg._real_base_ids)
    assert out is dw
    changed = [i for i in range(20) if not torch.equal(dw[0][i], before[i])]
    assert changed == BASE0
    assert torch.equal(dw[0][BASE0], torch.from_numpy(stored[0])[BASE0])
    novel = [cfg.classes.index(c) for c in cfg.novel_classes]
    assert torch.equal(dw[0][novel], before[novel])


def test_substitution_refuses_vectors_that_do_not_fit():
    from fewshot_detection_b200 import valid as VA
    with pytest.raises(ValueError, match=r'\(15, 64, 1, 1\)'):
        VA.substitute_base_rows(vectors(), [np.zeros((15, 64, 1, 1), np.float32)], [0])
    with pytest.raises(ValueError, match='2 stored layers'):
        VA.substitute_base_rows(vectors(), [np.zeros((20, 64, 1, 1), np.float32)] * 2, [0])


def test_result_prefix():
    cli = tool('valid_ensemble_b200')
    w = os.path.join('backup', 'metatune_novel0_neg0', '000010.weights')
    assert cli.result_prefix(w, True) == os.path.join('results', 'metatune_novel0_neg0', 'ene_000010')
    assert cli.result_prefix(w) == os.path.join('results', 'metatune_novel0_neg0', 'ene000010')
    assert cli.result_prefix(w, False) == cli.result_prefix(w)


def command_files(root):
    """A `.data` file with 20 VOC classes and novel split 0, and mini cfgs whose reweighting vectors are 512 wide."""
    from fewshot_detection_b200 import netcfg
    novels = os.path.join(root, 'novels.txt')
    with open(novels, 'w') as f:
        f.write(NOVELS)
    data = os.path.join(root, 'meta.data')
    with open(data, 'w') as f:
        f.write('metayolo=1\nmetain_type=2\ndata=voc\nneg = 1\nrand = 0\nnovel = %s\nnovelid = 0\nmeta = unused.txt\n'
                'valid = unused.txt\n' % novels)
    netcfg.write_cfg(netcfg.mini_dynamic_blocks(128, 16), os.path.join(root, 'det.cfg'))
    netcfg.write_cfg(netcfg.mini_reweighting_blocks(64, 16, 512), os.path.join(root, 'ler.cfg'))
    return [data, os.path.join(root, 'det.cfg'), os.path.join(root, 'ler.cfg'), os.path.join(root, 'w.weights')]


def test_evaluation_command_refuses_a_bad_vectors_file_before_the_model(tmp_path, saved_cfg, capsys):
    """Every case fails in argument checking: no model, no GPU."""
    cli = tool('valid_ensemble_b200')
    args = command_files(str(tmp_path)) + ['--write-results']
    with pytest.raises(SystemExit) as e:
        cli.main(args + ['--base-rw', str(tmp_path / 'missing.pkl')])
    assert e.value.code == 2 and 'missing.pkl' in capsys.readouterr().err
    bad = str(tmp_path / 'c1024.pkl')
    with open(bad, 'wb') as f:
        pickle.dump([np.zeros((20, 1024, 1, 1), np.float32)], f)
    with pytest.raises(SystemExit) as e:
        cli.main(args + ['--base-rw', bad])
    err = capsys.readouterr().err
    assert e.value.code == 2 and '(20, 512, 1, 1)' in err and '(20, 1024, 1, 1)' in err, err
    good = str(tmp_path / 'c512.pkl')
    with open(good, 'wb') as f:
        pickle.dump([np.ones((20, 512, 1, 1), np.float32)], f)
    got = cli.load_base_rw(good, args[0], args[2])
    assert len(got) == 1 and got[0].shape == (20, 512, 1, 1)


def test_training_driver_refuses_eval_base_rw_without_an_evaluation(tmp_path, monkeypatch, capsys):
    cli = tool('train_meta_b200')
    args = ['train_meta_b200.py', 'a.data', 'det.cfg', 'ler.cfg', 'w.weights']
    rw = str(tmp_path / 'rw.pkl')
    with open(rw, 'wb') as f:
        pickle.dump([np.ones((20, 512, 1, 1), np.float32)], f)
    monkeypatch.setattr(sys, 'argv', args + ['--eval-base-rw', rw])
    assert cli.main() == 1
    assert '--eval-base-rw needs --eval-devkit or --eval-coco-annotations' in capsys.readouterr().out
    monkeypatch.setattr(sys, 'argv', args + ['--eval-devkit', str(tmp_path), '--eval-base-rw', str(tmp_path / 'no.pkl')])
    assert cli.main() == 1
    assert 'no.pkl' in capsys.readouterr().out

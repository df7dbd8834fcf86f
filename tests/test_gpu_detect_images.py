"""The detection pass on the GPU: fsdet_detect_select on real head outputs against the Python reference, the graphed
pass against the eager one, the selection against the evaluation's result lines, and the detection command end to
end."""
import os

import numpy as np
import pytest
import torch

from test_detect_select_host_emul import assert_select_equals, reference_select

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def model():
    from test_gpu_zz_eval_pass import make_model
    return make_model(501, True)


def vectors(m, sup, n_cls, seed):
    from test_gpu_zz_eval_pass import support_batches
    from fewshot_detection_b200 import valid as VA
    return VA.ensemble_dynamic_weights(m, support_batches(sup, n_cls, seed), n_cls)


def random_sizes(B, seed):
    rs = np.random.RandomState(seed)
    return [(int(rs.randint(32, 1200)), int(rs.randint(32, 1200))) for _ in range(B)]


def snapshot(m):
    return dict((k, v.detach().clone()) for k, v in m.state_dict().items())


def assert_unchanged(m, before):
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k


# the evaluation shapes of test_gpu_zz_eval_pass: voc64 (64 images x 20 classes) and coco8 (8 x 80)
@pytest.mark.parametrize('sup,B,n_cls', [pytest.param((64, 8), 64, 20, id='voc64'),
                                         pytest.param((64, 32), 8, 80, id='coco8')])
@pytest.mark.parametrize('conf', [0.005, 0.5])
def test_select_equals_reference_on_real_head_output(model, sup, B, n_cls, conf):
    from test_gpu_zz_eval_pass import query_batch
    from fewshot_detection_b200 import valid as VA
    dw = vectors(model, sup, n_cls, 11)
    sizes = random_sizes(B, B + n_cls)
    dets = VA.detect(model, query_batch(B, 12).cuda(), dw, n_cls, conf, 0.45)
    for max_det in (100, 1):
        got = dets.select(n_cls, sizes, max_det)
        assert_select_equals(got.host(), reference_select(dets, n_cls, sizes, max_det), max_det)
    total = got.host()[4]
    if conf == 0.005:
        assert (total > 100).any()                  # the cap binds
    print('conf %g: survivors per image %d..%d' % (conf, total.min(), total.max()))


def eager_padded(m, x, dw, n_cls, sizes, B, conf, nms, max_det):
    """What GraphedDetect computes for a batch of b <= B images: the eager pass over the batch padded to B with zero
    images (the forward's tiling depends on the batch size, so a pass over b images can differ in the last bits),
    narrowed to the b images."""
    from fewshot_detection_b200 import valid as VA
    b, side = x.size(0), x.size(-1)
    xp = torch.cat([x, torch.zeros(B - b, 3, side, side, device=x.device)]) if b < B else x
    return VA.detect_images(m, xp, dw, n_cls, list(sizes) + [(side, side)] * (B - b), conf, nms, max_det).narrow(b)


def test_graph_replay_equals_eager(model):
    from fewshot_detection_b200 import valid as VA
    from fewshot_detection_b200.graph import GraphedDetect
    n_cls, B, conf, nms, max_det = 20, 8, 0.005, 0.45, 100
    dw = vectors(model, (64,), n_cls, 21)
    before = snapshot(model)
    gd = GraphedDetect(model, dw, B, 416, n_cls, conf, nms, max_det)
    g = torch.Generator().manual_seed(22)
    # three full batches of different contents, a padded partial batch, and a second side
    batches = [(torch.rand(B, 3, 416, 416, generator=g), random_sizes(B, 1)),
               (torch.rand(B, 3, 416, 416, generator=g), random_sizes(B, 2)),
               (torch.rand(B, 3, 416, 416, generator=g) * 0.5, random_sizes(B, 3)),
               (torch.rand(5, 3, 416, 416, generator=g), random_sizes(5, 4)),
               (torch.rand(B, 3, 608, 608, generator=g), random_sizes(B, 5)),
               (torch.rand(3, 3, 608, 608, generator=g), random_sizes(3, 6))]
    counts = []
    for x, sizes in batches:
        x = x.cuda()
        got = gd(x, sizes).host()
        want = eager_padded(model, x, dw, n_cls, sizes, B, conf, nms, max_det).host()
        assert got[0].shape[0] == len(sizes)
        for a, b in zip(got, want):
            assert a.shape == b.shape and a.tobytes() == b.tobytes()
        counts.append(got[4].tolist())              # survivors before the cap: the batches differ
    assert gd.captures == 2 and sorted(gd.entries) == [(B, 416), (B, 608)]
    assert_unchanged(model, before)
    assert counts[0] != counts[1] and sum(map(sum, counts)) > 0
    print('graph == eager; survivors', counts)


@pytest.mark.parametrize('max_det', [100, 100000])
def test_selected_boxes_are_the_evaluation_lines(model, max_det):
    """conf 0.005 / NMS 0.45: per image and class, the selected boxes printed as valid.detection_lines prints them are
    its lines of that image with the highest probs, best first; all of them when the cap does not bind."""
    from test_gpu_zz_eval_pass import query_batch
    from fewshot_detection_b200 import valid as VA
    n_cls, B = 20, 16
    dw = vectors(model, (64,), n_cls, 31)
    sizes = random_sizes(B, 32)
    imgids = ['img%03d' % b for b in range(B)]
    dets = VA.detect(model, query_batch(B, 33).cuda(), dw, n_cls)
    lines = VA.detection_lines(dets, imgids, sizes, n_cls)
    result = dets.select(n_cls, sizes, max_det)
    per_image = result.lists()
    _, _, _, count, total = result.host()
    for b in range(B):
        assert int(total[b]) == sum(sum(1 for l in lines[i] if l.split()[0] == imgids[b]) for i in range(n_cls))
        for i in range(n_cls):
            mine = [l for l in lines[i] if l.split()[0] == imgids[b]]
            sel = ['%s %f %f %f %f %f\n' % ((imgids[b],) + tuple(r[1:])) for r in per_image[b] if r[0] == i]
            probs = [float(l.split()[1]) for l in sel]
            assert probs == sorted(probs, reverse=True)
            if int(total[b]) <= max_det:
                assert sorted(sel) == sorted(mine)
            else:
                rest = list(mine)
                for l in sel:
                    rest.remove(l)                  # every selected line is one of the image's lines
                assert not rest or not sel or max(float(l.split()[1]) for l in rest) <= min(probs)
    assert (total > max_det).any() == (max_det == 100)


def test_detect_command_end_to_end(tmp_path):
    from PIL import Image
    from fewshot_detection_b200 import netcfg, valid as VA
    from fewshot_detection_b200.cfg import cfg, parse_cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.dataset import DetectionBatcher
    from fewshot_detection_b200.image import decode_many
    from test_detect_command import tool
    from seeding import seeded_init
    saved = dict(cfg)
    try:
        root = str(tmp_path)
        det, ler = os.path.join(root, 'det.cfg'), os.path.join(root, 'ler.cfg')
        netcfg.write_cfg(netcfg.mini_dynamic_blocks(128, 16), det)
        netcfg.write_cfg(netcfg.mini_reweighting_blocks(64, 16, 512), ler)
        cfg.config_meta(parse_cfg(ler)[0])
        cfg.config_net(parse_cfg(det)[0])
        m = Darknet(parse_cfg(det), parse_cfg(ler))
        seeded_init(m, 7)
        weights = os.path.join(root, 'w.weights')
        m.save_weights(weights)
        names = ['cat', 'traffic light', 'dog']
        with open(os.path.join(root, 'c.names'), 'w') as f:
            f.write('\n'.join(names) + '\n')
        g = torch.Generator().manual_seed(8)
        rw = os.path.join(root, 'rw.pkl')
        VA.save_reweighting_vectors(rw, [torch.randn(3, 512, 1, 1, generator=g) * 0.1])
        rs = np.random.RandomState(9)
        paths = []
        for k, (w, h, ext) in enumerate([(200, 150, 'jpg'), (97, 311, 'png'), (640, 480, 'jpg'), (128, 128, 'png'),
                                         (33, 45, 'jpg')]):
            p = os.path.join(root, 'im%d.%s' % (k, ext))
            Image.fromarray(rs.randint(0, 256, (h, w, 3)).astype(np.uint8)).save(p)
            paths.append(p)
        out = os.path.join(root, 'out')
        cli = tool('detect_b200')
        args = [det, ler, weights] + paths + ['--rw', rw, '--names', os.path.join(root, 'c.names'), '--conf', '0.005',
                                             '--max-det', '7', '--batch-size', '3', '--out', out, '--draw']
        assert cli.main(args) == 0
        # the kernel's output for the same images, eagerly
        m2 = Darknet(parse_cfg(det), parse_cfg(ler))
        m2.load_weights(weights)
        m2 = m2.cuda().eval()
        dw = [torch.from_numpy(a).cuda() for a in VA.load_reweighting_vectors(rw)]
        want = []
        for s in (0, 3):
            arrays = decode_many(paths[s:s + 3])
            data, _ = DetectionBatcher([(a, np.zeros((0, 5))) for a in arrays], shape=(m2.width, m2.height),
                                       shuffle=False, train=False, batch_size=len(arrays)).batch(range(len(arrays)))
            sizes = [(a.shape[1], a.shape[0]) for a in arrays]
            want.extend(eager_padded(m2, data, dw, 3, sizes, 3, 0.005, 0.4, 7).lists(names))
        n_lines = 0
        for p, rows in zip(paths, want):
            stem = os.path.splitext(os.path.basename(p))[0]
            with open(os.path.join(out, stem + '.txt')) as f:
                got = [l.rstrip('\n').rsplit(' ', 5) for l in f]
            assert len(got) == len(rows)
            for g_, r in zip(got, rows):
                assert g_[0] == r[0] and [float(v) for v in g_[1:]] == list(r[1:])
            n_lines += len(rows)
            with Image.open(os.path.join(out, stem + '.jpg')) as im, Image.open(p) as src:
                assert im.size == src.size
        assert n_lines > 0
    finally:
        cfg.clear()
        cfg.update(saved)

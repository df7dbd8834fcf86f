"""coco_eval.py, the host COCO box evaluator (and the device's oracle): hand-computed answers for every rule of
pycocotools' evaluateImg / accumulate / summarize, the category mapping of coco.names and the results json."""
import io
import json

import numpy as np
import pytest

from fewshot_detection_b200 import coco_eval as C
from fewshot_detection_b200.cfg import COCO_NAMES

ONE = pytest.approx(1.0, abs=1e-15)                     # a perfect precision is 1 / (1 + eps)


def run(anns, dets, classes=('a',), novel=()):
    """anns[i]: image i's objects (class, [x, y, w, h], area or None for w*h, iscrowd); dets: (image, class, score,
    [x, y, w, h])."""
    names = ['img%d' % i for i in range(len(anns))]
    gt = {'image_ids': [100 + i for i in range(len(anns))], 'category_ids': [10 + k for k in range(len(classes))],
          'anns': [[(c, [float(v) for v in b], b[2] * b[3] if a is None else a, cr) for c, b, a, cr in objs]
                   for objs in anns]}
    results = [{'image_id': 100 + i, 'category_id': 10 + c, 'bbox': [float(v) for v in b], 'score': s}
               for i, c, s, b in dets]
    return C.coco_evaluate(gt, results, names, list(classes), novel_classes=novel)


def test_perfect_detections_give_one():
    boxes = [[5, 5, 20, 20], [10, 10, 60, 50], [0, 0, 200, 150]]              # small, medium, large
    anns = [[(0, b, None, 0), (1, [b[0] + 1, b[1], b[2], b[3]], None, 0)] for b in boxes]
    dets = [(i, c, 0.9 - 0.1 * c, o[1]) for i, objs in enumerate(anns) for c, o in enumerate(objs)]
    r = run(anns, dets, classes=('a', 'b'))
    assert r['all'] == pytest.approx([1.0] * 12, abs=1e-15)                # precision is tp / (tp + fp + eps)
    assert r['ap'] == pytest.approx({'a': 1.0, 'b': 1.0}, abs=1e-15)


def test_single_detection_at_iou_062():
    r = run([[(0, [0, 0, 100, 100], None, 0)]], [(0, 0, 0.8, [0, 0, 62, 100])])
    assert C.bbox_iou([[0, 0, 62, 100]], [[0, 0, 100, 100]], [0])[0, 0] == 0.62
    assert r['all'][0] == pytest.approx(0.3, abs=1e-15) and r['all'][1] == ONE and r['all'][2] == 0.0
    assert r['ap']['a'] == r['all'][0]


def test_crowd_ground_truth_absorbs_detections():
    crowd = [100, 100, 200, 200]
    anns = [[(0, [0, 0, 50, 50], None, 0), (0, crowd, None, 1)]]
    inside = [[110, 110, 40, 40], [150, 150, 60, 60]]
    # IoU with a crowd box is intersection over the detection's area
    assert C.bbox_iou(inside, [crowd], [1])[:, 0].tolist() == [1.0, 1.0]
    assert C.bbox_iou(inside, [crowd], [0])[0, 0] == 1600.0 / 40000.0
    dets = [(0, 0, 0.9, inside[0]), (0, 0, 0.8, inside[1]), (0, 0, 0.7, [0, 0, 50, 50])]
    r = run(anns, dets)
    assert r['all'][0] == ONE                                                 # the crowd matches are neither TP nor FP
    gt = [([0., 0., 50., 50.], 2500.0, 0), (crowd, 40000.0, 1)]
    e = C.evaluate_img([(0.9, inside[0]), (0.8, inside[1]), (0.7, [0, 0, 50, 50])], gt, [0, 1e10], 100, C.Params())
    assert e['dtMatches'].all() and e['dtIgnore'][:, :2].all() and not e['dtIgnore'][:, 2].any()
    assert e['gtIgnore'].tolist() == [False, True]


def test_area_field_not_box_area_picks_the_range():
    # a 40x40 box (1600, medium by box area) whose json area is 900 (small)
    r = run([[(0, [10, 10, 40, 40], 900.0, 0)]], [(0, 0, 0.9, [10, 10, 40, 40])])
    assert r['all'][3] == ONE and r['all'][4] == -1.0 and r['all'][5] == -1.0
    assert r['all'][9] == 1.0 and r['all'][10] == -1.0


def test_area_range_bounds_are_inclusive():
    # json areas exactly 32^2 and 96^2 are in both neighbouring ranges
    r = run([[(0, [0, 0, 32, 32], None, 0)], [(0, [0, 0, 96, 96], None, 0)]],
            [(0, 0, 0.9, [0, 0, 32, 32]), (1, 0, 0.8, [0, 0, 96, 96])])
    assert r['recall'][0, 0, 1:, 2].tolist() == [1.0, 1.0, 1.0]


def test_unmatched_detection_outside_the_range_is_ignored():
    anns = [[(0, [0, 0, 20, 20], None, 0)]]
    dets = [(0, 0, 0.9, [300, 300, 200, 200]), (0, 0, 0.5, [0, 0, 20, 20])]   # a large FP ranked first
    r = run(anns, dets)
    assert r['all'][0] == pytest.approx(0.5, abs=1e-12)                       # all: FP then TP
    assert r['all'][3] == ONE                                                 # small: the large FP is ignored


def test_equal_iou_goes_to_the_later_ground_truth():
    anns = [[(0, [0, 0, 100, 100], None, 0), (0, [50, 0, 100, 100], None, 0)]]
    d1, d2 = [25, 0, 100, 100], [0, 0, 100, 100]
    iou = C.bbox_iou([d1], [anns[0][0][1], anns[0][1][1]], [0, 0])
    assert iou[0, 0] == iou[0, 1] == 0.6
    r = run(anns, [(0, 0, 0.9, d1), (0, 0, 0.8, d2)])
    # t = .5, .55: d1 takes the later box, so d2 still finds the first one: precision 1 at every recall
    assert r['precision'][:2, :, 0, 0, 2].min() == ONE
    assert r['precision'][-1, 0, 0, 0, 2] == pytest.approx(0.5, abs=1e-15)                             # t = .95: d1 is an FP ranked first


def test_score_ties_across_images_follow_the_image_set_order():
    anns = [[(0, [0, 0, 50, 50], None, 0)], [(0, [0, 0, 50, 50], None, 0)]]
    dets = [(0, 0, 0.7, [200, 200, 50, 50]), (1, 0, 0.7, [0, 0, 50, 50])]     # image 0: FP, image 1: TP, equal score
    r = run(anns, dets)
    assert r['precision'][0, 0, 0, 0, 2] == pytest.approx(0.5, abs=1e-15)    # FP ranked first
    swapped = run(anns[::-1], [(1 - i, c, s, b) for i, c, s, b in dets])
    assert swapped['precision'][0, 0, 0, 0, 2] == ONE                        # TP ranked first


def test_max_dets_prefixes():
    boxes = [[0, 0, 50, 50], [100, 0, 50, 50], [200, 0, 50, 50]]
    r = run([[(0, b, None, 0) for b in boxes]], [(0, 0, 0.9 - 0.1 * k, b) for k, b in enumerate(boxes)])
    assert r['all'][6] == pytest.approx(1 / 3.0, abs=1e-15) and r['all'][7] == 1.0 and r['all'][8] == 1.0
    assert r['recall'][0, 0, 0].tolist() == [1 / 3.0, 1.0, 1.0]


def test_class_without_ground_truth_is_excluded():
    anns = [[(0, [0, 0, 50, 50], None, 0)]]
    dets = [(0, 0, 0.9, [0, 0, 50, 50]), (0, 1, 0.9, [0, 0, 50, 50])]
    r = run(anns, dets, classes=('a', 'b'), novel=('b',))
    assert (r['precision'][:, :, 1] == -1).all() and (r['recall'][:, 1] == -1).all()
    assert r['ap']['b'] == -1.0 and r['all'][0] == ONE and r['base'][0] == ONE and r['novel'] == [-1.0] * 12


def test_more_than_100_detections_per_image_are_cut():
    anns = [[(0, [0, 0, 50, 50], None, 0)]]
    dets = [(0, 0, 0.9, [500, 500, 5, 5])] * 100 + [(0, 0, 0.1, [0, 0, 50, 50])]
    r = run(anns, dets)
    assert r['all'][8] == 0.0 and r['all'][0] == 0.0


# ---- annotations and results json ---------------------------------------------------------------------------------------
COCO_JSON_NAMES = [C.COCO_ALIASES.get(n, n) for n in COCO_NAMES]


def instances(names, objs, cat_names=COCO_JSON_NAMES):
    ids = [k + 1 + k // 10 for k in range(len(cat_names))]                   # ascending ids with gaps, as COCO's
    cats = [{'id': i, 'name': n} for i, n in zip(ids, cat_names)]
    rs = np.random.RandomState(0)
    cats = [cats[k] for k in rs.permutation(len(cats))]                       # file order is not id order
    images = [{'id': 1000 - 7 * k, 'file_name': n + '.jpg'} for k, n in enumerate(names)]
    anns = [{'id': j + 1, 'image_id': 1000 - 7 * k, 'category_id': ids[c], 'bbox': b, 'area': a, 'iscrowd': cr}
            for j, (k, c, b, a, cr) in enumerate(objs)]
    return {'images': images, 'categories': cats, 'annotations': anns}, ids


def test_load_annotations_maps_coco_names_order(tmp_path):
    names = ['COCO_val2014_%012d' % k for k in (42, 73, 74)]
    objs = [(0, 3, [1, 2, 3, 4], 12.5, 0), (2, 79, [0.5, 0, 10, 10], 100, 1), (0, 4, [5, 5, 5, 5], 25, 0),
            (0, 3, [7, 7, 7, 7], 49, 0)]
    data, ids = instances(names, objs)
    p = tmp_path / 'instances.json'
    p.write_text(json.dumps(data))
    gt = C.load_coco_annotations(str(p), names[::-1], COCO_NAMES)
    assert gt['category_ids'] == ids and gt['image_ids'] == [1000 - 14, 1000 - 7, 1000]
    assert gt['anns'][2] == [(3, [1.0, 2.0, 3.0, 4.0], 12.5, 0), (4, [5.0, 5.0, 5.0, 5.0], 25, 0),
                             (3, [7.0, 7.0, 7.0, 7.0], 49, 0)]
    assert gt['anns'][0] == [(79, [0.5, 0.0, 10.0, 10.0], 100, 1)] and gt['anns'][1] == []
    assert COCO_NAMES[3] == 'motorbike' and COCO_NAMES[4] == 'aeroplane'


def test_load_annotations_rejects_a_name_mismatch(tmp_path):
    bad = list(COCO_JSON_NAMES)
    bad[17] = 'pony'
    data, _ = instances(['x'], [], cat_names=bad)
    p = tmp_path / 'instances.json'
    p.write_text(json.dumps(data))
    with pytest.raises(ValueError):
        C.load_coco_annotations(str(p), ['x'], COCO_NAMES)


def test_results_json_round_trips_exactly():
    rs = np.random.RandomState(1)
    recs = [('a', int(rs.randint(3)), float(s), [float(v) for v in rs.uniform(-5, 700, 4)])
            for s in rs.uniform(0, 1, 50) * rs.uniform(0, 1, 50)]
    recs.append(('b', 0, 0.1 + 0.2, [1 / 3.0, 2 ** -40, 1e-300, -0.0]))
    f = io.StringIO()
    C.write_coco_results(f, recs, {'a': 42, 'b': 7}, [1, 2, 3])
    back = json.loads(f.getvalue())
    assert [(r['image_id'], r['category_id']) for r in back] == [(42 if r[0] == 'a' else 7, r[1] + 1) for r in recs]
    assert all(x['score'] == r[2] and x['bbox'] == r[3] for x, r in zip(back, recs))
    assert repr(back[-1]['score']) == repr(0.1 + 0.2)


def test_summary_lines():
    lines = C.format_stats([0.5] * 12)
    assert len(lines) == 12
    assert lines[0] == ' Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 0.500'
    assert lines[6] == ' Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = 0.500'

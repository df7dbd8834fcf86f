"""fsdet_voc_merge / fsdet_coco_merge (csrc/eval_sort.cuh) without a GPU, compiled by g++ against
tools/host_emul/cuda_host_emul.h: the pools of separate gather sequences (one per rank of a sharded evaluation) merged
in rank order must be the pool of one sequence over the same batches, record for record, and score bit for bit the
same.  Also: an empty rank, a rank with images but no records, an image on two ranks (error bit 2) and a destination
too small (error bit 1, nothing written)."""
import ctypes

import numpy as np
import pytest

import test_coco_eval_host_emul as TC
import test_voc_eval_host_emul as TV
from emul_util import build_emul

P = TV.P


@pytest.fixture(scope='module')
def voc():
    lib = build_emul('voc_eval', 'voc_eval.cu')
    lib.emul_voc_workspace_bytes.restype = ctypes.c_size_t
    lib.emul_eval_merge_workspace_bytes.restype = ctypes.c_size_t
    return lib


@pytest.fixture(scope='module')
def coco():
    lib = build_emul('coco_eval', 'coco_eval.cu')
    lib.emul_coco_workspace_bytes.restype = ctypes.c_size_t
    lib.emul_eval_merge_workspace_bytes.restype = ctypes.c_size_t
    return lib


def stack(pools, key_dtype):
    """Padded per-source buffers as an all-gather leaves them: counters [R, 4], key [R, P], box [R, P, 4],
    groups [R, G, 4] (padding filled with garbage that must never be read)."""
    R = len(pools)
    Pn = max([1] + [int(p[3][0]) for p in pools])
    Gn = max([1] + [int(p[3][1]) for p in pools])
    key = np.full((R, Pn), 77, dtype=key_dtype)
    box = np.full((R, Pn, 4), -99.0)
    groups = np.full((R, Gn, 4), -5, dtype=np.int32)
    counters = np.zeros((R, 4), dtype=np.int64)
    for r, (k, b, g, c) in enumerate(pools):
        n, ng = int(c[0]), int(c[1])
        key[r, :n], box[r, :n], groups[r, :ng], counters[r] = k[:n], b[:n], g[:ng], c
    return counters, key, box, groups


def merge(lib, fn, pools, key_dtype, n_images, pool_cap=None, group_cap=None, slack=16):
    """Run the merge into fresh buffers with `slack` sentinel entries past the capacities."""
    counters, key, box, groups = stack(pools, key_dtype)
    total, gtotal = int(counters[:, 0].sum()), int(counters[:, 1].sum())
    pool_cap = total if pool_cap is None else pool_cap
    group_cap = gtotal if group_cap is None else group_cap
    dkey = np.full(pool_cap + slack, 55, dtype=key_dtype)
    dbox = np.full((pool_cap + slack, 4), 3.5)
    dgroups = np.full((group_cap + slack, 4), 9, dtype=np.int32)
    dcount = np.full(4, 123, dtype=np.int64)
    ws = np.zeros(lib.emul_eval_merge_workspace_bytes(len(pools), n_images), dtype=np.uint8)
    getattr(lib, fn)(len(pools), P(counters), P(key), P(box), ctypes.c_longlong(key.shape[1]), P(groups),
                     ctypes.c_longlong(groups.shape[1]), n_images, P(ws), P(dkey), P(dbox), ctypes.c_longlong(pool_cap),
                     P(dgroups), group_cap, P(dcount))
    return dkey, dbox, dgroups, dcount


# ---- VOC: pools laid out as fsdet_voc_gather lays them (batch, image, class; records in line order) ----------------
def voc_pool(per_class, names, images):
    index = dict((n, k) for k, n in enumerate(names))
    keys, boxes, groups = [], [], []
    for i in images:
        for c, lines in enumerate(per_class):
            mine = [l for l in lines if index[l[0]] == i]
            groups.append([len(keys), len(mine), i, c])
            for l in mine:
                keys.append((c << 20) | (TV.KEY_MASK - int(round(l[1] * 1e6))))
                boxes.append(l[2:])
    counters = np.array([len(keys), len(groups), 0, 0], dtype=np.int64)
    return (np.array(keys, dtype=np.uint32), np.array(boxes, dtype=np.float64).reshape(-1, 4),
            np.array(groups, dtype=np.int32).reshape(-1, 4), counters)


def voc_evaluate(lib, key, box, groups, counters, classes, names, recs):
    n, ng = int(counters[0]), int(counters[1])
    gt_ptr, gt_box, gt_diff = TV.V.gt_tables(classes, names, recs)
    n_cls, n_gt = len(classes), len(gt_diff)
    ws = np.zeros(max(1, lib.emul_voc_workspace_bytes(n, n_gt)), dtype=np.uint8)
    out = dict(flags=np.full(n, 9, np.uint8), order=np.full(n, -1, np.int32), rec=np.full(n, -7.0),
               prec=np.full(n, -7.0), cls_count=np.full(n_cls, -1, np.int32), npos=np.full(n_cls, -1, np.int32),
               ap07=np.full(n_cls, -7.0), ap_area=np.full(n_cls, -7.0))
    th = np.ascontiguousarray(TV.V.VOC07_THRESHOLDS)
    lib.emul_voc_evaluate(P(key[:n]), P(box[:n]), n, P(groups[:ng]), ng, P(gt_ptr), P(gt_box), P(gt_diff), n_gt, n_cls,
                          len(names), ctypes.c_double(0.5), P(th), P(ws), P(out['flags']), P(out['order']),
                          P(out['rec']), P(out['prec']), P(out['cls_count']), P(out['npos']), P(out['ap07']),
                          P(out['ap_area']))
    return out


def rank_blocks(batches, sizes):
    """Contiguous blocks of `batches` with the given numbers of batches per rank."""
    out, k = [], 0
    for s in sizes:
        out.append(batches[k:k + s])
        k += s
    assert k == len(batches)
    return out


@pytest.mark.parametrize('seed,split', [(0, (3, 1, 4, 2)), (1, (4, 0, 6)), (2, (10,)), (3, (0, 5, 5, 0))])
def test_voc_merge_equals_one_sequence(voc, seed, split):
    names, recs, classes, per_class = TV.synthetic_case(seed)
    batches = [list(range(k, min(k + 4, len(names)))) for k in range(0, len(names), 4)]
    one = voc_pool(per_class, names, [i for b in batches for i in b])
    pools = [voc_pool(per_class, names, [i for b in blk for i in b]) for blk in rank_blocks(batches, split)]
    key, box, groups, counters = merge(voc, 'emul_voc_merge', pools, np.uint32, len(names))
    n, ng = int(one[3][0]), int(one[3][1])
    assert counters.tolist() == [n, ng, 0, 0]
    assert np.array_equal(key[:n], one[0]) and np.array_equal(box[:n], one[1]) and np.array_equal(groups[:ng], one[2])
    assert (key[n:] == 55).all() and (box[n:] == 3.5).all() and (groups[ng:] == 9).all()
    a = voc_evaluate(voc, key, box, groups, counters, classes, names, recs)
    b = voc_evaluate(voc, one[0], one[1], one[2], one[3], classes, names, recs)
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    start = 0
    for c, name in enumerate(classes):                                  # and the host evaluator's numbers
        n = len(per_class[c])
        _, _, rec, prec, ap07, _ = TV.host_class_eval(per_class[c], recs, names, name)
        assert a['cls_count'][c] == n and a['ap07'][c] == ap07
        assert np.array_equal(a['rec'][start:start + n], rec, equal_nan=True)
        assert np.array_equal(a['prec'][start:start + n], prec)
        start += n


def test_voc_rank_with_images_but_no_records(voc):
    names, recs, classes, per_class = TV.synthetic_case(4)
    bare = set(names[8:12])
    per_class = [[l for l in lines if l[0] not in bare] for lines in per_class]
    blocks = [list(range(0, 8)), list(range(8, 12)), list(range(12, len(names)))]
    pools = [voc_pool(per_class, names, b) for b in blocks]
    assert pools[1][3][0] == 0 and pools[1][3][1] == 4 * len(classes)
    one = voc_pool(per_class, names, list(range(len(names))))
    key, box, groups, counters = merge(voc, 'emul_voc_merge', pools, np.uint32, len(names))
    assert counters.tolist() == one[3].tolist()
    assert np.array_equal(groups[:len(one[2])], one[2]) and np.array_equal(key[:len(one[0])], one[0])


def test_voc_image_on_two_ranks_and_overflow(voc):
    names, recs, classes, per_class = TV.synthetic_case(5)
    pools = [voc_pool(per_class, names, list(range(0, 10))), voc_pool(per_class, names, list(range(9, 20)))]
    _, _, _, counters = merge(voc, 'emul_voc_merge', pools, np.uint32, len(names))
    assert counters[3] == 2
    pools = [voc_pool(per_class, names, list(range(0, 10))), voc_pool(per_class, names, list(range(10, 20)))]
    total = int(sum(p[3][0] for p in pools))
    for pool_cap, group_cap in ((total - 1, None), (None, 20 * len(classes) - 1)):
        key, box, groups, counters = merge(voc, 'emul_voc_merge', pools, np.uint32, len(names), pool_cap, group_cap)
        assert counters.tolist() == [0, 0, 0, 1]
        assert (key == 55).all() and (box == 3.5).all() and (groups == 9).all()     # nothing written at all
    # a source that overflowed its own gather poisons the merge the same way
    bad = (pools[1][0], pools[1][1], pools[1][2], pools[1][3].copy())
    bad[3][3] = 1
    key, box, groups, counters = merge(voc, 'emul_voc_merge', [pools[0], bad], np.uint32, len(names))
    assert counters[3] & 1 and (key == 55).all()


def test_voc_malformed_group_is_flagged_not_followed(voc):
    names, recs, classes, per_class = TV.synthetic_case(6)
    k, b, g, c = voc_pool(per_class, names, list(range(0, 6)))
    g = g.copy()
    g[3, 0] = int(c[0])                        # runs past the source's records
    g[3, 1] = 5
    key, box, groups, counters = merge(voc, 'emul_voc_merge', [(k, b, g, c)], np.uint32, len(names))
    assert counters[3] == 4 and groups[3, 1] == 0
    assert (key[int(c[0]):] == 55).all()


# ---- COCO: pools from the emulated gather itself ---------------------------------------------------------------------
@pytest.mark.parametrize('seed,world', [(0, 3), (1, 16), (2, 1), (3, 4)])
def test_coco_merge_equals_one_gather_sequence(coco, seed, world):
    from fewshot_detection_b200.shard import shard_range
    n_cls = 6
    gt, sizes, rows = TC.synthetic_set(seed, n_cls=n_cls)
    assert max(len(r) for r in rows) > 100
    names = ['COCO_val2014_%012d' % i for i in gt['image_ids']]
    batches = TC.batches_of(len(names), seed)
    blocks = [batches[slice(*shard_range(len(batches), 1, world, r))] for r in range(world)]
    assert sum(len(b) for b in blocks) == len(batches)
    if world == 16:
        assert any(not b for b in blocks)                                  # ranks without batches
    one = TC.emul_gather(coco, gt, sizes, rows, n_cls, batches)
    pools = []
    for blk in blocks:
        imgs = [i for b in blk for i in b]
        cap = sum(min(len(rows[i * n_cls + c]), 100) for i in imgs for c in range(n_cls))
        pools.append(TC.emul_gather(coco, gt, sizes, rows, n_cls, blk, pool_cap=cap, group_cap=len(imgs) * n_cls))
    score, box, groups, counters = merge(coco, 'emul_coco_merge', pools, np.float64, len(names))
    n, ng = int(one[3][0]), int(one[3][1])
    assert counters.tolist() == [n, ng, 0, 0]
    assert np.array_equal(score[:n], one[0][:n]) and np.array_equal(box[:n], one[1][:n])
    assert np.array_equal(groups[:ng], one[2][:ng])
    a = TC.emul_evaluate(coco, score, box, groups, counters, gt, n_cls)
    b = TC.emul_evaluate(coco, one[0], one[1], one[2], one[3], gt, n_cls)
    TC.check_bit_equal(a, b)
    _, ref = TC.host_reference(gt, sizes, rows, names, n_cls, batches)
    TC.check_bit_equal(a, ref)


def test_coco_image_on_two_ranks_and_overflow(coco):
    n_cls = 3
    gt, sizes, rows = TC.synthetic_set(8, n_img=10, n_cls=n_cls, big_rows=1)
    pools = [TC.emul_gather(coco, gt, sizes, rows, n_cls, [[0, 1], [2, 3]]),
             TC.emul_gather(coco, gt, sizes, rows, n_cls, [[3, 4], [5]])]
    _, _, _, counters = merge(coco, 'emul_coco_merge', pools, np.float64, 10)
    assert counters[3] == 2
    pools[1] = TC.emul_gather(coco, gt, sizes, rows, n_cls, [[4], [5, 6]])
    total = int(pools[0][3][0] + pools[1][3][0])
    score, box, groups, counters = merge(coco, 'emul_coco_merge', pools, np.float64, 10, pool_cap=total - 1)
    assert counters.tolist() == [0, 0, 0, 1] and (score == 55).all() and (groups == 9).all()


def test_shard_plan():
    from fewshot_detection_b200.shard import shard_range
    for n, bs, world in [(4952, 64, 8), (10, 3, 4), (7, 3, 8), (0, 4, 2), (64, 64, 2), (65, 64, 2), (5, 1, 5)]:
        ranges = [shard_range(n, bs, world, r) for r in range(world)]
        assert ranges[0][0] == 0 and max(r[1] for r in ranges) == n
        for (a0, a1), (b0, b1) in zip(ranges, ranges[1:]):
            assert a1 == b0                                              # contiguous, in rank order
        for a, b in ranges:
            assert (a % bs == 0 or a == n) and (b % bs == 0 or b == n)   # whole batches only
        busy = [r for r in ranges if r[1] > r[0]]
        assert all(r[1] - r[0] == busy[0][1] - busy[0][0] for r in busy[:-1])
    assert shard_range(65, 64, 2, 1) == (64, 65) and shard_range(7, 3, 8, 5) == (7, 7)

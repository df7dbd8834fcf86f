"""Test-time augmentation kernels (csrc/detect.cu, voc_eval.cu, coco_eval.cu) without a GPU: the kernel sources
compiled by g++ against tools/host_emul/cuda_host_emul.h, on seeded candidate tables, bit for bit against the Python
oracle built from the reference's own pieces: per pass the box lists of get_region_boxes_v2 (x = xs / W, ...), the
mirror x = 1.0 - x on flipped passes, concatenation in pass order, and the reference's nms (oracle/utils.py) on the
concatenated list.

Also: the merged-record forms of the per-image selection and of the VOC and COCO gathers write the same bytes as
their single-pass counterparts on the merged table of one unflipped pass."""
import ctypes

import numpy as np
import pytest

from emul_util import build_emul

A = 5
REC = np.dtype([('x', '<f8'), ('y', '<f8'), ('w', '<f8'), ('h', '<f8'), ('det', '<f4'), ('cls', '<f4'), ('cid', '<i4'),
                ('src', '<i4')])
SENTINEL = 0x5a


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


@pytest.fixture(scope='module')
def emul():
    lib = build_emul('detect', 'detect.cu')
    lib.emul_nms_merged_workspace_bytes.restype = ctypes.c_size_t
    lib.emul_detect_select_workspace_bytes.restype = ctypes.c_size_t
    return lib


def aligned(nbytes):
    buf = np.zeros(nbytes + 256, dtype=np.uint8)
    off = (-buf.ctypes.data) % 256
    return buf[off:off + nbytes]


def pass_table(rs, N, G, counts, ties=False, clusters=None):
    """cand float32 [N, A*G*G, 8] / count of one pass on a G x G grid with counts[n] candidates in row n.  ties:
    det_conf from a few binary fractions (equal keys within and across passes).  clusters: boxes around that many
    centres per row (long rows whose survivors stay few)."""
    K = A * G * G
    cand = np.zeros((N, K, 8), dtype=np.float32)
    count = np.zeros(N, dtype=np.int32)
    for n in range(N):
        c = int(counts[n])
        count[n] = c
        if clusters:
            centre = rs.uniform(0.1, 0.9, (clusters, 2))[rs.randint(0, clusters, c)]
            xy = (centre + rs.normal(0, 0.01, (c, 2))) * G
            wh = rs.uniform(0.2, 0.3, (c, 2)) * G
        else:
            xy = rs.uniform(0, G, (c, 2))
            wh = rs.uniform(0.05, G / 3.0, (c, 2))
        cand[n, :c, 0:2] = xy
        cand[n, :c, 2:4] = wh
        cand[n, :c, 4] = rs.choice([0.5, 0.25, 0.75, 0.125], c) if ties else rs.uniform(0.005, 1, c)
        cand[n, :c, 5] = rs.uniform(0.01, 1, c)
        cand[n, :c, 6:8] = np.stack([np.zeros(c, np.int32), rs.permutation(K)[:c].astype(np.int32)], 1).view(np.float32)
    return cand, count


def oracle_rows(passes, tables):
    """Per row the reference's concatenated box list: [x, y, w, h, det, cls, cid, (pass, slot)] as Python floats."""
    N = tables[0][0].shape[0]
    rows = [[] for _ in range(N)]
    for p, ((G, flip), (cand, count)) in enumerate(zip(passes, tables)):
        for n in range(N):
            for t in range(int(count[n])):
                v = cand[n, t]
                box = [float(v[0]) / G, float(v[1]) / G, float(v[2]) / G, float(v[3]) / G, float(v[4]), float(v[5]),
                       int(v[6:7].view(np.int32)[0]), (p, t)]
                if flip:
                    box[0] = 1.0 - box[0]
                rows[n].append(box)
    return rows


def run_merge(emul, passes, tables, merged_cap, guard=64):
    """The merged table through emul_tta_merge, one call per pass; the buffer has `guard` sentinel records past the
    end.  Returns (records [N, merged_cap], count, overflow, guard bytes)."""
    N = tables[0][0].shape[0]
    buf = np.full((N * merged_cap + guard) * REC.itemsize, SENTINEL, dtype=np.uint8)
    count = np.zeros(N, dtype=np.int32)
    overflow = np.zeros(1, dtype=np.int32)
    for p, ((G, flip), (cand, cnt)) in enumerate(zip(passes, tables)):
        assert emul.emul_tta_merge(P(cand), P(cnt), N, cand.shape[1], G, G, flip, p, P(buf), P(count), merged_cap,
                                   P(overflow)) == 0
    rec = buf[:N * merged_cap * REC.itemsize].view(REC).reshape(N, merged_cap)
    return rec, count, int(overflow[0]), buf[N * merged_cap * REC.itemsize:]


def run_nms(emul, rec, count, thresh):
    N, cap = rec.shape
    ws = aligned(int(emul.emul_nms_merged_workspace_bytes(N, cap)))
    keep = np.full((N, cap), -1, dtype=np.int32)
    kc = np.full(N, -1, dtype=np.int32)
    assert emul.emul_nms_merged(P(rec), P(count), N, cap, ctypes.c_double(thresh), P(ws), P(keep), P(kc)) == 0
    return keep, kc


def assert_merged_equals(rec, count, want_rows):
    for n, row in enumerate(want_rows):
        assert int(count[n]) == len(row), (n, int(count[n]), len(row))
        got = rec[n, :len(row)]
        for k, b in enumerate(row):
            q = got[k]
            assert np.array([q['x'], q['y'], q['w'], q['h']]).tobytes() == np.array(b[:4], np.float64).tobytes(), (n, k)
            assert float(q['det']) == b[4] and float(q['cls']) == b[5] and int(q['cid']) == b[6], (n, k)
            assert int(q['src']) == (b[7][0] << 20 | b[7][1]), (n, k)


def assert_nms_equals(keep, kc, want_rows, thresh):
    from oracle import utils as OU
    for n, row in enumerate(want_rows):
        slot_of = dict((b[7], s) for s, b in enumerate(row))
        want = [slot_of[b[7]] for b in OU.nms([list(b) for b in row], thresh)]
        assert int(kc[n]) == len(want), (n, int(kc[n]), len(want))
        assert keep[n, :len(want)].tolist() == want, n


# (name, grids of the passes with their flips, rows, candidates per row and pass: 'full', 'rand' or a list, options)
CASES = [
    # rows 0 and 3 empty in every pass, row 4 empty in one; grids 10 / 13 / 19 (sides 320 / 416 / 608)
    ('empty-rows', [(13, 0), (13, 1), (19, 0), (10, 1)], 6, [[0, 200, 845, 0, 0, 17]] * 3 + [[0, 3, 500, 0, 9, 0]], {}),
    # 5 x 1805 = 9025 > 4096 candidates in a row, long clustered rows: survivors of earlier chunks suppress later ones
    ('above-4096', [(19, 0), (19, 1), (19, 0), (19, 1), (19, 0)], 2, 'full', dict(clusters=6)),
    # near the 16384 of the six-pass plan's double: 4 passes of 28 x 28 (side 896) = 15680 per row
    ('near-16k', [(28, 0), (28, 1), (28, 0), (28, 1)], 1, 'full', dict(clusters=4)),
    # equal det_conf within a pass and across passes: ties keep merged order
    ('ties', [(13, 0), (13, 1), (17, 0)], 4, 'rand', dict(ties=True)),
    # every pass flipped
    ('all-flipped', [(13, 1), (17, 1), (19, 1)], 3, 'rand', {}),
]


@pytest.mark.parametrize('name,passes,N,counts,opts', CASES, ids=[c[0] for c in CASES])
def test_merge_and_nms_equal_the_oracle(emul, name, passes, N, counts, opts):
    rs = np.random.RandomState(len(name) * 31 + N)
    tables = []
    for p, (G, _) in enumerate(passes):
        K = A * G * G
        if counts == 'full':
            c = [K - rs.randint(0, 5) for _ in range(N)]
        elif counts == 'rand':
            c = [rs.randint(0, K // 3) for _ in range(N)]
        else:
            c = [min(K, v) for v in counts[min(p, len(counts) - 1)]]
        tables.append(pass_table(rs, N, G, c, **opts))
    cap = sum(A * G * G for G, _ in passes)
    rec, count, overflow, guard = run_merge(emul, passes, tables, cap)
    want = oracle_rows(passes, tables)
    assert overflow == 0 and (guard == SENTINEL).all()
    assert_merged_equals(rec, count, want)
    if name == 'ties':
        dets = [b[4] for row in want for b in row]
        assert len(set(dets)) < len(dets)
    thresh = 0.45
    keep, kc = run_nms(emul, rec, count, thresh)
    assert_nms_equals(keep, kc, want, thresh)
    if name in ('above-4096', 'near-16k'):
        assert count.min() > 4096 and kc.min() > 1
    print('%s: rows of %s candidates, %s survivors' % (name, count.tolist(), kc.tolist()))


def test_merge_overflow_sets_the_flag_and_writes_nothing_past_the_end(emul):
    rs = np.random.RandomState(5)
    passes = [(13, 0), (13, 1), (10, 0)]
    N = 4
    tables = [pass_table(rs, N, G, [rs.randint(100, 400) for _ in range(N)]) for G, _ in passes]
    tables[1][1][2] = 0                               # row 2 of pass 1 is empty
    cap = 700
    rec, count, overflow, guard = run_merge(emul, passes, tables, cap)
    assert overflow == 1 and (guard == SENTINEL).all()
    # each row holds the passes that fit whole, in order; the rest of its capacity is untouched
    for n in range(N):
        fit = []
        used = 0
        for p in range(len(passes)):
            c = int(tables[p][1][n])
            if used + c <= cap:
                fit.append(p)
                used += c
        want = [b for b in oracle_rows(passes, tables)[n] if b[7][0] in fit]
        assert_merged_equals(rec[n:n + 1], count[n:n + 1], [want])
        assert (rec[n, used:].view(np.uint8) == SENTINEL).all()
    assert any(int(count[n]) < sum(int(t[1][n]) for t in tables) for n in range(N))   # the case does overflow


def test_merged_consumers_equal_single_pass_on_one_pass(emul):
    """One unflipped pass: fsdet_detect_select_merged, fsdet_voc_gather_merged and fsdet_coco_gather_merged write the
    bytes of fsdet_detect_select, fsdet_voc_gather and fsdet_coco_gather on the pass's own candidates."""
    voc = build_emul('voc_eval', 'voc_eval.cu')
    coco = build_emul('coco_eval', 'coco_eval.cu')
    rs = np.random.RandomState(9)
    B, n_cls, G = 3, 4, 13
    N, K = B * n_cls, A * G * G
    cand, count = pass_table(rs, N, G, [rs.randint(0, 300) for _ in range(N)], ties=True)
    keep = np.full((N, K), -1, dtype=np.int32)
    kc = np.zeros(N, dtype=np.int32)
    emul.emul_nms(P(cand), None, P(count), N, K, G, G, ctypes.c_double(0.45), P(keep), P(kc))
    rec, mcount, overflow, _ = run_merge(emul, [(G, 0)], [(cand, count)], K, guard=0)
    mkeep, mkc = run_nms(emul, rec, mcount, 0.45)
    assert overflow == 0 and np.array_equal(mcount, count)
    assert np.array_equal(mkc, kc) and all(mkeep[n, :kc[n]].tolist() == keep[n, :kc[n]].tolist() for n in range(N))
    assert kc.sum() > 50
    sizes = np.array([[500, 375], [333, 640], [1200, 31]], dtype=np.int32)
    # per-image selection
    outs = []
    for merged in (False, True):
        ws = aligned(int(emul.emul_detect_select_workspace_bytes(N, K)))
        score, box = np.full((B, 20), np.nan), np.full((B, 20, 4), np.nan)
        cls, cnt, tot = np.full((B, 20), 7, np.int32), np.full(B, -9, np.int32), np.full(B, -9, np.int32)
        if merged:
            emul.emul_detect_select_merged(P(rec), P(keep), P(kc), N, K, n_cls, P(sizes), 20, P(ws), P(score), P(box),
                                           P(cls), P(cnt), P(tot))
        else:
            emul.emul_detect_select(P(cand), P(keep), P(kc), N, K, G, G, n_cls, P(sizes), 20, P(ws), P(score), P(box),
                                    P(cls), P(cnt), P(tot))
        outs.append(b''.join(a.tobytes() for a in (score, box, cls, cnt, tot)))
    assert outs[0] == outs[1]
    # VOC and COCO gathers
    idx = np.array([2, 0, 1], dtype=np.int32)
    size = sizes.astype(np.float64)
    pool = int(kc.sum())
    outs = []
    for merged in (False, True):
        keys, boxes = np.zeros(pool, np.uint32), np.zeros((pool, 4))
        groups, counters = np.zeros((N, 4), np.int32), np.zeros(4, np.int64)
        if merged:
            voc.emul_voc_gather_merged(P(rec), P(keep), P(kc), N, K, n_cls, P(idx), P(size), P(keys), P(boxes),
                                       ctypes.c_longlong(pool), P(groups), N, P(counters))
        else:
            voc.emul_voc_gather(P(cand), P(keep), P(kc), N, K, G, G, n_cls, P(idx), P(size), P(keys), P(boxes),
                                ctypes.c_longlong(pool), P(groups), N, P(counters))
        assert counters[3] == 0 and counters[0] == pool
        outs.append(b''.join(a.tobytes() for a in (keys, boxes, groups, counters)))
    assert outs[0] == outs[1]
    outs = []
    for merged in (False, True):
        score, boxes = np.zeros(pool), np.zeros((pool, 4))
        groups, counters = np.zeros((N, 4), np.int32), np.zeros(4, np.int64)
        if merged:
            coco.emul_coco_gather_merged(P(rec), P(keep), P(kc), N, K, n_cls, P(idx), P(size), 100, P(score), P(boxes),
                                         ctypes.c_longlong(pool), P(groups), N, P(counters))
        else:
            coco.emul_coco_gather(P(cand), P(keep), P(kc), N, K, G, G, n_cls, P(idx), P(size), 100, P(score), P(boxes),
                                  ctypes.c_longlong(pool), P(groups), N, P(counters))
        assert counters[3] == 0
        outs.append(b''.join(a.tobytes() for a in (score, boxes, groups, counters)))
    assert outs[0] == outs[1]

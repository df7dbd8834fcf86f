"""Programmatic Darknet block lists for the networks the hot path is quoted on.

The reference's `Darknet(darknet_file, learnet_file)` accepts either a path to a
Darknet `.cfg` file or an already parsed list of block dicts
(darknet_meta.py:87-90).  The reference's `cfg/*.cfg` files are not part of this
repository, so the benchmark and the tests build the same architectures from the
compact specs below (architecture facts taken from cfg/darknet_dynamic.cfg,
cfg/reweighting_net.cfg and cfg/tiny-yolo-voc.cfg) in the exact dict format
`cfg.parse_cfg` produces (all values are strings, `type=` keys renamed
`_type`, conv blocks default `batch_normalize` to 0; cfg.py:198-228).
User supplied `.cfg` files keep working through `cfg.parse_cfg`.
"""

VOC_ANCHORS = "1.3221, 1.73145, 3.19275, 4.00944, 5.05587, 8.09892, 9.47112, 4.84053, 11.2364, 10.0071"
TINY_VOC_ANCHORS = "1.08,1.19,  3.42,4.41,  6.63,11.38,  9.42,5.11,  16.62,10.52"


def _conv(filters, size, bn=1, act='leaky', **extra):
    # parse_cfg's default for a missing key is the *int* 0 (cfg.py:213-214)
    # (an explicit `batch_normalize=0` line is passed as the string '0')
    b = {'type': 'convolutional', 'batch_normalize': bn if bn == '0' else (str(bn) if bn else 0)}
    b.update({'filters': str(filters), 'size': str(size), 'stride': '1', 'pad': '1',
              'activation': act})
    for k, v in extra.items():
        b[k] = str(v)
    return b


def _maxpool(size=2, stride=2):
    return {'type': 'maxpool', 'size': str(size), 'stride': str(stride)}


def _net(width, height, channels=3, batch=64):
    return {'type': 'net', 'batch': str(batch), 'subdivisions': '8', 'height': str(height),
            'width': str(width), 'channels': str(channels), 'momentum': '0.9',
            'decay': '0.0005', 'learning_rate': '0.001', 'max_batches': '80200',
            'policy': 'steps', 'steps': '-1,500,40000,60000', 'scales': '0.1,10,.1,.1'}


def _region(anchors, classes, num=5, jitter='.3'):
    return {'type': 'region', 'anchors': anchors, 'bias_match': '1', 'classes': str(classes),
            'coords': '4', 'num': str(num), 'softmax': '1', 'jitter': jitter, 'rescore': '1',
            'object_scale': '5', 'noobject_scale': '1', 'class_scale': '1',
            'coord_scale': '1', 'absolute': '1', 'thresh': '.6', 'random': '1'}


def darknet_dynamic_blocks(width=416, height=416, anchors=VOC_ANCHORS):
    """Detector of the meta model: Darknet-19 trunk + passthrough + dynamic 1x1
    + 1x1 head (cfg/darknet_dynamic.cfg:27-273)."""
    B = [_net(width, height)]
    B += [_conv(32, 3), _maxpool(), _conv(64, 3), _maxpool()]
    B += [_conv(128, 3), _conv(64, 1), _conv(128, 3), _maxpool()]
    B += [_conv(256, 3), _conv(128, 1), _conv(256, 3), _maxpool()]
    B += [_conv(512, 3), _conv(256, 1), _conv(512, 3), _conv(256, 1), _conv(512, 3), _maxpool()]
    B += [_conv(1024, 3), _conv(512, 1), _conv(1024, 3), _conv(512, 1), _conv(1024, 3)]
    B += [_conv(1024, 3), _conv(1024, 3)]
    B += [{'type': 'route', 'layers': '-9'}, _conv(64, 1), {'type': 'reorg', 'stride': '2'},
          {'type': 'route', 'layers': '-1,-4'}]
    B += [_conv(1024, 3)]
    B += [_conv(1024, 1, bn='0', act='linear', dynamic=1)]
    B += [_conv(30, 1, bn=0, act='linear')]
    B += [_region(anchors, classes=1)]
    return B


def reweighting_net_blocks(width=416, height=416, channels=4):
    """Support branch (cfg/reweighting_net.cfg:1-97)."""
    B = [{'type': 'learnet', 'feat_layer': '0', 'channels': str(channels),
          'height': str(height), 'width': str(width)}]
    for f in (32, 64, 128, 256, 512, 1024):
        B += [_conv(f, 3), _maxpool()]
    B += [_conv(1024, 3), {'type': 'globalmax'}]
    return B


def tiny_yolo_voc_blocks(width=416, height=416):
    """Plain YOLOv2-tiny (cfg/tiny-yolo-voc.cfg), BASELINE config #1."""
    B = [_net(width, height)]
    for f in (16, 32, 64, 128, 256):
        B += [_conv(f, 3), _maxpool()]
    B += [_conv(512, 3), _maxpool(2, 1), _conv(1024, 3), _conv(1024, 3)]
    B += [_conv(125, 1, bn=0, act='linear')]
    B += [_region(TINY_VOC_ANCHORS, classes=20, jitter='.2')]
    return B


def mini_dynamic_blocks(side=64, c=8):
    """Scaled-down detector with every layer *type* of darknet_dynamic (3x3/1x1
    conv+BN+leaky, maxpool, route, reorg, 2-way route, dynamic conv, head,
    region) for fast full-tensor parity tests. Stride 32 like the real one."""
    B = [_net(side, side)]
    B += [_conv(c, 3), _maxpool(), _conv(2 * c, 3), _maxpool()]
    B += [_conv(4 * c, 3), _conv(2 * c, 1), _conv(4 * c, 3), _maxpool()]
    B += [_conv(8 * c, 3), _maxpool()]
    B += [_conv(16 * c, 3), _conv(8 * c, 1), _conv(16 * c, 3), _maxpool()]      # blocks 10..12, pool 13
    B += [_conv(32 * c, 3), _conv(32 * c, 3)]                                   # 14, 15
    B += [{'type': 'route', 'layers': '-4'}, _conv(2 * c, 1), {'type': 'reorg', 'stride': '2'},
          {'type': 'route', 'layers': '-1,-4'}]                                 # 16(->12),17,18,19(->18,15)
    B += [_conv(32 * c, 3)]
    B += [_conv(32 * c, 1, bn='0', act='linear', dynamic=1)]
    B += [_conv(30, 1, bn=0, act='linear')]
    B += [_region(VOC_ANCHORS, classes=1)]
    return B


def mini_reweighting_blocks(side=64, c=8, out=256, channels=4):
    B = [{'type': 'learnet', 'feat_layer': '0', 'channels': str(channels),
          'height': str(side), 'width': str(side)}]
    for f in (c, 2 * c, 4 * c, 8 * c):
        B += [_conv(f, 3), _maxpool()]
    B += [_conv(out, 3), {'type': 'globalmax'}]
    return B


def mini_tiny_blocks(side=64, c=8):
    B = [_net(side, side)]
    for f in (c, 2 * c, 4 * c, 8 * c, 16 * c):
        B += [_conv(f, 3), _maxpool()]
    B += [_conv(32 * c, 3), _maxpool(2, 1), _conv(32 * c, 3)]
    B += [_conv(125, 1, bn=0, act='linear')]
    B += [_region(TINY_VOC_ANCHORS, classes=20)]
    return B


def write_cfg(blocks, path):
    """Serialise a block list as a Darknet `.cfg` file that `cfg.parse_cfg`
    reads back to the same list."""
    with open(path, 'w') as f:
        for b in blocks:
            f.write('[%s]\n' % b['type'])
            for k, v in b.items():
                if k == 'type':
                    continue
                if b['type'] == 'convolutional' and k == 'batch_normalize' and v == 0:
                    continue
                f.write('%s=%s\n' % ('type' if k == '_type' else k, v))
            f.write('\n')

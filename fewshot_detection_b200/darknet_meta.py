"""`Darknet(darknet_file, learnet_file)`: the meta-detector of the reference
(darknet_meta.py:86-482) on the H100-native engine.

Kept from the reference so that train_meta.py / valid_ensemble.py drop in:
constructor arguments (cfg path or parsed block list, darknet_meta.py:87-90),
attributes `.blocks .learnet_blocks .models .learnet_models .loss .width .height
.anchors .num_anchors .anchor_step .num_classes .header .seen`, methods
`forward(x, metax, mask, ids=None)`, `meta_forward`, `detect_forward`,
`load_weights`, `save_weights(outfile, cutoff=0)`, `print_network`,
`is_dynamic`, the ModuleList / Sequential(conv{i}, bn{i}, leaky{i}) tree (so
`parameters()` order, `state_dict()` keys and the Darknet weight stream are the
same), and `nn.Module` behaviour (.cuda(), .train(), .eval()).

New underneath: nn.Conv2d / nn.BatchNorm2d are only parameter containers here;
the forward and backward passes are executed by engine.NetRunner with
hand-written sm_90a kernels (libfsdet.so).  CUDA only - no CPU fallback.
"""
import numpy as np
import torch
import torch.nn as nn

from .cfg import cfg, parse_cfg, load_conv, load_conv_bn, save_conv, save_conv_bn
from .dynamic_conv import dynamic_conv2d
from .engine import NetRunner, run_network
from .pooling import GlobalMaxPool2d, MaxPoolStride1, MaxPool2x2, Reorg, EmptyModule
from .region_loss import RegionLossV2, RegionLoss


class _Build(object):
    """Running state while a block list is turned into modules: channel count of the current feature map, channel
    counts of every module built so far (routes look them up), convolution and dynamic-convolution counters."""

    def __init__(self, owner, loss_cls):
        self.owner, self.loss_cls = owner, loss_cls
        self.channels = 3
        self.history = []
        self.n_conv = 0
        self.n_dynamic = 0


def _make_convolutional(ctx, block):
    """nn.Sequential(conv{i}[, bn{i}][, leaky{i}]) - the names are the state_dict keys of the reference
    (darknet_meta.py:219-259).  Bias only without BatchNorm; pad = (k-1)//2 when `pad=1`."""
    ctx.n_conv += 1
    tag = str(ctx.n_conv)
    k, filters = int(block['size']), int(block['filters'])
    pad = (k - 1) // 2 if int(block['pad']) else 0
    has_bn = bool(int(block['batch_normalize']))
    if 'groups' in block and int(block['groups']) != 1:
        raise NotImplementedError('grouped convolution')
    if ctx.owner.is_dynamic(block):
        conv_cls = dynamic_conv2d(ctx.n_dynamic == 0, partial=int(block['partial']) if 'partial' in block else None)
        ctx.n_dynamic += 1
    else:
        conv_cls = nn.Conv2d
    use_bias = (not has_bn) and (bool(int(block['bias'])) if 'bias' in block else True)
    seq = nn.Sequential()
    seq.add_module('conv' + tag, conv_cls(ctx.channels, filters, k, int(block['stride']), pad, bias=use_bias))
    if has_bn:
        seq.add_module('bn' + tag, nn.BatchNorm2d(filters))
    if block['activation'] == 'leaky':
        seq.add_module('leaky' + tag, nn.LeakyReLU(0.1, inplace=True))
    elif block['activation'] == 'relu':
        raise NotImplementedError('relu activation')
    ctx.channels = filters
    return seq


def _make_maxpool(ctx, block):
    size, stride = int(block['size']), int(block['stride'])
    return MaxPool2x2(size, stride) if stride > 1 else MaxPoolStride1()


def _make_reorg(ctx, block):
    stride = int(block['stride'])
    ctx.channels = stride * stride * ctx.channels
    return Reorg(stride)


def _make_route(ctx, block):
    here = len(ctx.history)
    sources = [int(i) if int(i) > 0 else int(i) + here for i in block['layers'].split(',')]
    if len(sources) == 2:
        assert sources[0] == here - 1
    if len(sources) in (1, 2):
        ctx.channels = sum(ctx.history[i] for i in sources)
    return EmptyModule()


def _make_region(ctx, block):
    loss = ctx.loss_cls()
    loss.anchors = [float(i) for i in block['anchors'].split(',')]
    loss.num_classes = int(block['classes'])
    loss.num_anchors = int(block['num'])
    loss.anchor_step = len(loss.anchors) // loss.num_anchors
    for key in ('object_scale', 'noobject_scale', 'class_scale', 'coord_scale'):
        setattr(loss, key, float(block[key]))
    return loss


_BUILDERS = {
    'convolutional': _make_convolutional,
    'maxpool': _make_maxpool,
    'reorg': _make_reorg,
    'route': _make_route,
    'region': _make_region,
    'globalmax': lambda ctx, block: GlobalMaxPool2d(),
}


def create_network(owner, blocks, loss_cls):
    """Block list -> nn.ModuleList with one module per non-header block (darknet_meta.py:208-353 /
    darknet.py:134-245), through a table from block type to builder."""
    ctx = _Build(owner, loss_cls)
    models = nn.ModuleList()
    for block in blocks:
        kind = block['type']
        if kind in ('net', 'learnet'):
            ctx.channels = int(block['channels'])
            continue
        if kind not in _BUILDERS:
            raise NotImplementedError('block type %s is not on the supported hot path' % kind)
        models.append(_BUILDERS[kind](ctx, block))
        ctx.history.append(ctx.channels)
    return models


def _copy_blocks(blocks):
    return [dict(b) for b in blocks]


class Darknet(nn.Module):
    """replicas: R, the number of nn.DataParallel replicas one training step of the reference runs (its shipped configs
    train on 4 GPUs).  A train-mode `forward` then splits the query batch and the support batch into R contiguous
    chunks: every BatchNorm normalises each chunk by its own statistics (the running statistics follow replica 0),
    and replica r's query images are reweighted by replica r's vectors.  The output keeps the row order b * n_cls + c.
    Evaluation and the separate `meta_forward` / `detect_forward` calls are unaffected."""

    def __init__(self, darknet_file, learnet_file, replicas=1):
        super(Darknet, self).__init__()
        if int(replicas) < 1:
            raise ValueError('replicas must be >= 1, got %r' % (replicas,))
        self.replicas = int(replicas)
        self.blocks = darknet_file if isinstance(darknet_file, list) else parse_cfg(darknet_file)
        self.learnet_blocks = learnet_file if isinstance(learnet_file, list) else parse_cfg(learnet_file)
        self.models = create_network(self, self.blocks, RegionLossV2)
        self.learnet_models = create_network(self, self.learnet_blocks, RegionLossV2)
        self.loss = self.models[len(self.models) - 1]

        self.width = int(self.blocks[0]['width'])
        self.height = int(self.blocks[0]['height'])

        if self.blocks[(len(self.blocks) - 1)]['type'] == 'region':
            self.anchors = self.loss.anchors
            self.num_anchors = self.loss.num_anchors
            self.anchor_step = self.loss.anchor_step
            self.num_classes = self.loss.num_classes

        self.header = torch.IntTensor([0, 0, 0, 0])
        self.seen = 0
        if int(self.learnet_blocks[0].get('feat_layer', 0)) != 0:
            raise NotImplementedError('[learnet] feat_layer != 0 (shared trunk layers) is not used by the shipped cfgs')
        self._det = NetRunner(self.blocks, self.models)
        self._ler = NetRunner(self.learnet_blocks, self.learnet_models)

    # ------------------------------------------------------------------ forward
    def _params(self, models):
        return [p for p in models.parameters()]

    def meta_forward(self, metax, mask):
        """Support branch (darknet_meta.py:107-128): returns [ [n_cls, C, 1, 1] ]."""
        if cfg.metain_type in [2, 3]:
            inputs = [metax, mask]
        else:
            inputs = [metax]
        dw = run_network(self._ler, inputs, None, self._params(self.learnet_models), self.training)
        return [dw]

    def detect_forward(self, x, dynamic_weights):
        """Query branch (darknet_meta.py:130-195): [B,3,H,W] -> [B*n_cls, A*(5+nC), H/32, W/32]."""
        self.loss = None  # the reference resets it here (darknet_meta.py:134)
        dw = dynamic_weights[0] if isinstance(dynamic_weights, (list, tuple)) else dynamic_weights
        return run_network(self._det, [x], dw, self._params(self.models), self.training)

    def forward(self, x, metax, mask, ids=None):
        R = self.replicas if self.training else 1
        if R == 1:
            dynamic_weights = self.meta_forward(metax, mask)
            return self.detect_forward(x, dynamic_weights)
        if x.shape[0] % R or metax.shape[0] % R:
            raise ValueError('%d replicas need a query batch and a support batch divisible by %d, got x %s and metax %s'
                             % (R, R, tuple(x.shape), tuple(metax.shape)))
        inputs = [metax, mask] if cfg.metain_type in [2, 3] else [metax]
        dw = run_network(self._ler, inputs, None, self._params(self.learnet_models), True, segments=R)
        self.loss = None
        return run_network(self._det, [x], dw, self._params(self.models), True, segments=R)

    def print_network(self):
        for name, blocks in (('detector', self.blocks), ('reweighting net', self.learnet_blocks)):
            print('--- %s' % name)
            for i, b in enumerate(blocks):
                print('%3d %-14s %s' % (i - 1, b['type'], ' '.join('%s=%s' % kv for kv in b.items() if kv[0] != 'type')))

    def is_dynamic(self, block):
        return 'dynamic' in block and int(block['dynamic']) == 1

    # --------------------------------------------------------------- weight IO
    def _weight_stream(self):
        """The Darknet weight stream's order (darknet_meta.py:355-479): every convolution that owns weights as
        (position, conv, bn-or-None) - detector blocks first, then the reweighting net.  `position` is the 1-based
        block counter `save_weights(cutoff=)` counts in: detector block i sits at i, learnet block j at
        len(self.blocks) + j (the learnet header occupies a position of its own)."""
        for offset, blocks, models in ((0, self.blocks, self.models), (len(self.blocks), self.learnet_blocks, self.learnet_models)):
            for i, block in enumerate(blocks):
                if i == 0 or block['type'] != 'convolutional':
                    continue
                seq = models[i - 1]
                if self.is_dynamic(block) and seq[0].weight is None:
                    continue                                    # the dynamic convolution's weights are its input
                yield offset + i, seq[0], (seq[1] if int(block['batch_normalize']) else None)

    def load_weights(self, weightfile):
        """header int32[4] (its last entry is `seen`) + float32 stream.  Loading stops silently where the stream
        ends - that is how darknet19_448.conv.23 initialises only the trunk (darknet_meta.py:367-368)."""
        with open(weightfile, 'rb') as fp:
            header = np.fromfile(fp, count=4, dtype=np.int32)
            buf = np.fromfile(fp, dtype=np.float32)
        self.header = torch.from_numpy(header)
        self.seen = int(self.header[3])
        start = 0
        for _, conv, bn in self._weight_stream():
            if start >= buf.size:
                break
            start = load_conv_bn(buf, start, conv, bn) if bn is not None else load_conv(buf, start, conv)

    def save_weights(self, outfile, cutoff=0):
        """Writes the stream up to block position `cutoff` (0 = everything), darknet_meta.py:413-479."""
        if cutoff <= 0:
            cutoff = len(self.blocks) - 1 + len(self.learnet_blocks)
        with open(outfile, 'wb') as fp:
            self.header[3] = int(self.seen)
            self.header.numpy().tofile(fp)
            for position, conv, bn in self._weight_stream():
                if position > cutoff:
                    break
                if bn is not None:
                    save_conv_bn(fp, conv, bn)
                else:
                    save_conv(fp, conv)

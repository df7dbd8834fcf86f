"""`Darknet(cfgfile)`: the plain YOLOv2 cfg interpreter of the reference
(darknet.py:61-341) on the H100-native engine (BASELINE config #1,
cfg/tiny-yolo-voc.cfg).  Same surface: `.blocks .models .loss .width .height
.anchors .num_anchors .anchor_step .num_classes .header .seen`, `forward(x)`,
`load_weights`, `save_weights`, `print_network`.  CUDA only."""
import numpy as np
import torch
import torch.nn as nn

from .cfg import parse_cfg, load_conv, load_conv_bn, save_conv, save_conv_bn
from .darknet_meta import create_network
from .engine import NetRunner, run_network
from .region_loss import RegionLoss


class Darknet(nn.Module):
    def __init__(self, cfgfile):
        super(Darknet, self).__init__()
        self.blocks = cfgfile if isinstance(cfgfile, list) else parse_cfg(cfgfile)
        self.models = create_network(self, self.blocks, RegionLoss)
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
        self._net = NetRunner(self.blocks, self.models)

    def is_dynamic(self, block):
        return False

    def forward(self, x):
        self.loss = None  # darknet.py:82
        return run_network(self._net, [x], None, list(self.models.parameters()), self.training)

    def print_network(self):
        for i, b in enumerate(self.blocks):
            print('%3d %-14s %s' % (i - 1, b['type'], ' '.join('%s=%s' % kv for kv in b.items() if kv[0] != 'type')))

    def load_weights(self, weightfile):
        """darknet.py:247-290."""
        with open(weightfile, 'rb') as fp:
            header = np.fromfile(fp, count=4, dtype=np.int32)
            self.header = torch.from_numpy(header)
            self.seen = int(self.header[3])
            buf = np.fromfile(fp, dtype=np.float32)
        start = 0
        ind = -2
        for block in self.blocks:
            if start >= buf.size:
                break
            ind = ind + 1
            if block['type'] == 'convolutional':
                model = self.models[ind]
                if int(block['batch_normalize']):
                    start = load_conv_bn(buf, start, model[0], model[1])
                else:
                    start = load_conv(buf, start, model[0])

    def save_weights(self, outfile, cutoff=0):
        """darknet.py:292-341."""
        if cutoff <= 0:
            cutoff = len(self.blocks) - 1
        with open(outfile, 'wb') as fp:
            self.header[3] = int(self.seen)
            self.header.numpy().tofile(fp)
            ind = -1
            for blockId in range(1, cutoff + 1):
                ind = ind + 1
                block = self.blocks[blockId]
                if block['type'] == 'convolutional':
                    model = self.models[ind]
                    if int(block['batch_normalize']):
                        save_conv_bn(fp, model[0], model[1])
                    else:
                        save_conv(fp, model[0])

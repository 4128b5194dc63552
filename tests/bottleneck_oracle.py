"""Test helper: CPU / fp32 plain-PyTorch restatement of the Bottleneck backbones (DLA-46-C, DLA-60, DLA-102, DLA-169 of
cubercnn/modeling/backbone/dla.py:71-110,156-230,324-450 and the torchvision ResNet-50 / 101 of resnet.py:12-63), on top of
oracle/cubercnn_oracle, whose heads, RPN and losses it reuses unchanged.  Pinned against the reference's own code by
tests/golden/make_bottleneck_golden.py + tests/test_bottleneck_cpu.py; the fp32 side of tests/test_bottleneck_gpu.py and
of tests/tools/bench_backbones.py.

The DLA-34 / ResNet-18 / 34 cases stay with oracle.cubercnn_oracle.build_model."""
import math

import torch
import torch.nn.functional as F
from torch import nn

import oracle.cubercnn_oracle as co  # noqa: F401  (puts oracle/d2lite on sys.path)
from detectron2.modeling.backbone import FPN, Backbone, LastLevelMaxPool  # noqa: E402
from detectron2.modeling.meta_arch.rcnn import GeneralizedRCNN  # noqa: E402
from oracle.cubercnn_oracle import model as _model  # noqa: E402

# name -> (config file, config overrides, golden image size (H, W))
CASES = {
    "resnet50": ("cubercnn_ResNet34_FPN.yaml", ["MODEL.RESNETS.DEPTH", 50], (128, 128)),
    "resnet101": ("cubercnn_ResNet34_FPN.yaml", ["MODEL.RESNETS.DEPTH", 101], (128, 128)),
    "dla46_c": ("cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla46_c"], (128, 160)),
    "dla60": ("cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla60"], (128, 160)),
    "dla102": ("cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla102"], (128, 160)),
    "dla169": ("cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla169"], (128, 160)),
}

# dla.py:324-415: levels of level2..level5, channels of base_layer..level5, root_residual
DLA_TYPES = {
    "dla46_c": ((1, 2, 2, 1), (16, 32, 64, 64, 128, 256), False),
    "dla60": ((1, 2, 3, 1), (16, 32, 128, 256, 512, 1024), False),
    "dla102": ((1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), True),
    "dla169": ((2, 3, 5, 1), (16, 32, 128, 256, 512, 1024), True),
}


def _cbr(cin, cout, k, stride=1):
    return [nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False), nn.BatchNorm2d(cout),
            nn.ReLU(inplace=True)]


class Bottleneck(nn.Module):
    def __init__(self, cin, cout, stride=1):
        super().__init__()
        mid = cout // 2
        self.conv1 = nn.Conv2d(cin, mid, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(mid)
        self.conv2 = nn.Conv2d(mid, mid, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(mid)
        self.conv3 = nn.Conv2d(mid, cout, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(cout)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x, residual=None):
        residual = x if residual is None else residual
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.relu(self.bn2(self.conv2(y)))
        return self.relu(self.bn3(self.conv3(y)) + residual)


class Root(nn.Module):
    def __init__(self, cin, cout, residual):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self.relu = nn.ReLU(inplace=True)
        self.residual = residual

    def forward(self, *xs):
        y = self.bn(self.conv(torch.cat(xs, 1)))
        return self.relu(y + xs[0] if self.residual else y)


class Tree(nn.Module):
    def __init__(self, levels, cin, cout, stride=1, level_root=False, root_dim=0, root_residual=False):
        super().__init__()
        if root_dim == 0:
            root_dim = 2 * cout
        if level_root:
            root_dim += cin
        if levels == 1:
            self.tree1 = Bottleneck(cin, cout, stride)
            self.tree2 = Bottleneck(cout, cout, 1)
            self.root = Root(root_dim, cout, root_residual)
        else:
            self.tree1 = Tree(levels - 1, cin, cout, stride, root_dim=0, root_residual=root_residual)
            self.tree2 = Tree(levels - 1, cout, cout, root_dim=root_dim + cout, root_residual=root_residual)
        self.level_root, self.levels = level_root, levels
        self.downsample = nn.MaxPool2d(stride, stride=stride) if stride > 1 else None
        self.project = None
        if cin != cout:
            # for levels >= 2 the projected residual goes to an inner Tree that ignores it (dla.py:217-230): the
            # parameters exist (state_dict parity) and receive no gradient; train mode still moves the BN statistics
            self.project = nn.Sequential(nn.Conv2d(cin, cout, 1, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x, residual=None, children=None):
        children = [] if children is None else children
        bottom = self.downsample(x) if self.downsample else x
        residual = self.project(bottom) if self.project else bottom
        if self.level_root:
            children.append(bottom)
        if self.levels == 1:
            x1 = self.tree1(x, residual)
            return self.root(self.tree2(x1), x1, *children)
        x1 = self.tree1(x, residual)
        children.append(x1)
        return self.tree2(x1, children=children)


class DLABackbone(Backbone):
    def __init__(self, dla_type):
        super().__init__()
        levels, c, root_residual = DLA_TYPES[dla_type]
        self.base_layer = nn.Sequential(*_cbr(3, c[0], 7))
        self.level0 = nn.Sequential(*_cbr(c[0], c[0], 3))
        self.level1 = nn.Sequential(*_cbr(c[0], c[1], 3, stride=2))
        for i in range(2, 6):
            setattr(self, "level%d" % i, Tree(levels[i - 2], c[i - 1], c[i], 2, level_root=i > 2,
                                              root_residual=root_residual))
        for m in self.modules():                      # dla.py:262-268
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        self._out_feature_channels = {"p2": c[2], "p3": c[3], "p4": c[4], "p5": c[5], "p6": c[5]}
        self._out_feature_strides = {"p2": 4, "p3": 8, "p4": 16, "p5": 32, "p6": 64}
        self._out_features = ["p2", "p3", "p4", "p5", "p6"]

    def forward(self, x):
        x = self.level1(self.level0(self.base_layer(x)))
        out = {}
        for i, name in zip(range(2, 6), ["p2", "p3", "p4", "p5"]):
            x = getattr(self, "level%d" % i)(x)
            out[name] = x
        out["p6"] = F.max_pool2d(x, kernel_size=1, stride=2, padding=0)
        return out


class TVResNetBackbone(Backbone):
    """torchvision ResNet-50 / 101: the modules (names, same-seed init) and forward of torchvision's Bottleneck."""

    def __init__(self, depth):
        super().__init__()
        from torchvision import models
        if depth not in (50, 101):
            raise ValueError("No configuration currently supporting depth of {}".format(depth))
        base = getattr(models, "resnet%d" % depth)(weights=None)
        for k in ("conv1", "bn1", "relu", "maxpool", "layer1", "layer2", "layer3", "layer4"):
            setattr(self, k, getattr(base, k))
        self._out_feature_channels = {"p2": 256, "p3": 512, "p4": 1024, "p5": 2048, "p6": 2048}
        self._out_feature_strides = {"p2": 4, "p3": 8, "p4": 16, "p5": 32, "p6": 64}
        self._out_features = ["p2", "p3", "p4", "p5", "p6"]

    def forward(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        out = {}
        for name, layer in zip(["p2", "p3", "p4", "p5"], [self.layer1, self.layer2, self.layer3, self.layer4]):
            x = layer(x)
            out[name] = x
        out["p6"] = F.max_pool2d(x, kernel_size=1, stride=2, padding=0)
        return out


def build_backbone(cfg):
    assert cfg.MODEL.WEIGHTS_PRETRAIN + cfg.MODEL.WEIGHTS != "", "no network: set MODEL.WEIGHTS_PRETRAIN non-empty"
    kw = dict(in_features=cfg.MODEL.FPN.IN_FEATURES, out_channels=cfg.MODEL.FPN.OUT_CHANNELS,
              norm=cfg.MODEL.FPN.NORM, fuse_type=cfg.MODEL.FPN.FUSE_TYPE)
    name = cfg.MODEL.BACKBONE.NAME
    if name == "build_dla_from_vision_fpn_backbone":
        return FPN(bottom_up=DLABackbone(cfg.MODEL.DLA.TYPE), **kw)
    if name == "build_resnet_from_vision_fpn_backbone":
        assert cfg.MODEL.RESNETS.TORCHVISION
        return FPN(bottom_up=TVResNetBackbone(cfg.MODEL.RESNETS.DEPTH), top_block=LastLevelMaxPool(), **kw)
    raise NotImplementedError(name)


class RCNN3D(_model.RCNN3D):
    """oracle.cubercnn_oracle.model.RCNN3D with a Bottleneck bottom-up; construction order (backbone, RPN, ROI heads) kept
    for the same-seed initialisation."""

    def __init__(self, cfg, priors=None):
        backbone = build_backbone(cfg)
        shape = backbone.output_shape()
        GeneralizedRCNN.__init__(self, backbone=backbone, proposal_generator=_model.RPNWithIgnore(cfg, shape),
                                 roi_heads=_model.ROIHeads3D(cfg, shape, priors=priors), pixel_mean=cfg.MODEL.PIXEL_MEAN,
                                 pixel_std=cfg.MODEL.PIXEL_STD, input_format=cfg.INPUT.FORMAT, vis_period=0)


def load_cfg(name):
    cfg_file, opts, _ = CASES[name]
    return co.load_cfg(cfg_file, list(opts))


def build_model(cfg, priors=None):
    model = RCNN3D(cfg, priors=priors)
    model.to(torch.device(cfg.MODEL.DEVICE))
    return model

"""DLA / torchvision ResNet bottom-ups + FPN on the wgmma convolution kernels (NHWC bf16).

Mirrors the module tree, parameter names and initialisation order of
cubercnn/modeling/backbone/dla.py:40-110,156-415,417-507 and resnet.py:12-96 (+ detectron2 FPN), so a
reference checkpoint's state_dict loads unchanged and the same seed gives the same initial weights.  The
nn.Conv2d / nn.BatchNorm2d modules below are PARAMETER HOLDERS (their forward is never called — every
convolution / BatchNorm / pooling runs through omni3d_b200.nnfunc on libc3d.so).
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from ..nnfunc import CatChannels, ConvBias, ConvBNAct, MaxPool2, MaxPool3s2, fork
from .registry import BACKBONE_REGISTRY


_fold_cache = {}


def set_bn_folding(model, enable=True):
    """mark every BatchNorm2d of `model`: in eval mode (and under no_grad) its conv+BN pair runs as ONE convolution with the
    BatchNorm folded into weight and bias (omni3d_b200.checkpoint.fold_batchnorm; SURVEY 8f-4)."""
    for m in model.modules():
        if isinstance(m, nn.BatchNorm2d):
            m._c3d_fold = bool(enable)
    _fold_cache.clear()


def _folded(conv, bn, cin):
    """bf16 OHWI pack of w * gamma * rstd and the fp32 bias beta - mean * gamma * rstd, cached per parameter / statistics
    version (load_state_dict and optimizer steps bump them; the trainer's raw-pointer updates bump nnfunc's epoch)."""
    from .. import conv as K
    from .. import nnfunc
    from ..checkpoint import folded_conv_params
    ts = (conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)
    ver = tuple((t.data_ptr(), t._version) for t in ts) + (nnfunc._epoch, cin)
    hit = _fold_cache.get(id(bn))
    if hit is None or hit[0] != ver or hit[3] is not bn:
        w, b = folded_conv_params(conv.weight.detach(), bn)
        if w.shape[1] != cin:
            w = F.pad(w, (0, 0, 0, 0, 0, cin - w.shape[1]))
        wp = K.pack_conv_weight(w, want_dgrad=False)[0]
        hit = (ver, wp, b.contiguous(), bn)
        _fold_cache[id(bn)] = hit
    return hit[1], hit[2]


def conv_bn(x, conv, bn, residual=None, relu=True):
    """x NHWC bf16 -> [relu](BN(conv(x)) [+ residual]) through the fused kernels."""
    if not bn.training and getattr(bn, "_c3d_fold", False) and not torch.is_grad_enabled():
        from .. import conv as K
        wp, b = _folded(conv, bn, x.shape[-1])
        res = residual.contiguous() if residual is not None else None
        return K.conv2d_fwd(x.contiguous(), wp, b, conv.stride[0], conv.padding[0], relu=relu, addend=res)
    w = conv.weight
    if w.shape[1] != x.shape[-1]:                       # stem: Cin 3 zero-padded to the 16 the TMA box needs
        w = F.pad(w, (0, 0, 0, 0, 0, x.shape[-1] - w.shape[1]))
    return ConvBNAct.apply(x, w, bn.weight, bn.bias, bn.running_mean, bn.running_var, residual, conv.stride[0],
                           conv.padding[0], relu, bn.training, bn.eps, bn.momentum)


class BasicBlock(nn.Module):
    def __init__(self, cin, cout, stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout)

    def forward(self, x, residual=None):
        if residual is None:
            x, residual = fork(x, 2)            # conv1 and the identity shortcut: one gradient buffer, no add pass
        y = conv_bn(x, self.conv1, self.bn1)
        return conv_bn(y, self.conv2, self.bn2, residual=residual)


class Bottleneck(nn.Module):
    """dla.py:71-109: 1x1 -> 3x3 (stride) -> 1x1 over planes // 2 channels, the residual added in the last conv's epilogue."""

    def __init__(self, cin, cout, stride=1):
        super().__init__()
        mid = cout // 2
        self.conv1 = nn.Conv2d(cin, mid, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(mid)
        self.conv2 = nn.Conv2d(mid, mid, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(mid)
        self.conv3 = nn.Conv2d(mid, cout, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(cout)

    def forward(self, x, residual=None):
        if residual is None:
            x, residual = fork(x, 2)
        y = conv_bn(x, self.conv1, self.bn1)
        y = conv_bn(y, self.conv2, self.bn2)
        return conv_bn(y, self.conv3, self.bn3, residual=residual)


class Root(nn.Module):
    """dla.py:156-174; with `residual` (DLA-102 / 169) the first child is added before the ReLU."""

    def __init__(self, cin, cout, residual=False):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self.residual = residual

    def forward(self, *xs):
        res = None
        if self.residual:
            first, res = fork(xs[0], 2)
            xs = (first,) + xs[1:]
        cat = CatChannels.apply(*xs) if torch.is_grad_enabled() else torch.cat(xs, dim=-1)
        return conv_bn(cat, self.conv, self.bn, residual=res)


class Tree(nn.Module):
    """dla.py:177-230 for any `levels`.  A nested tree gets the stride and pools its own input.  For levels >= 2 the
    `project` is dead weight in the reference (its output is handed to an inner Tree that recomputes its own residual):
    parameters kept, never computed (omni3d_b200.train.unused_parameter_names)."""

    def __init__(self, levels, block, cin, cout, stride=1, level_root=False, root_dim=0, root_residual=False):
        super().__init__()
        root_dim = 2 * cout if root_dim == 0 else root_dim
        if level_root:
            root_dim += cin
        if levels == 1:
            self.tree1 = block(cin, cout, stride)
            self.tree2 = block(cout, cout, 1)
            self.root = Root(root_dim, cout, root_residual)
        else:
            self.tree1 = Tree(levels - 1, block, cin, cout, stride, root_residual=root_residual)
            self.tree2 = Tree(levels - 1, block, cout, cout, root_dim=root_dim + cout, root_residual=root_residual)
        self.levels, self.level_root, self.stride = levels, level_root, stride
        self.project = None
        if cin != cout:
            self.project = nn.Sequential(nn.Conv2d(cin, cout, 1, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x, children=None):
        children = [] if children is None else children
        # every tensor with more than one consumer is forked (nnfunc.fork): its consumers share one gradient buffer
        n_bottom = int(self.level_root) + int(self.levels == 1)      # children list, project / identity residual
        if self.stride > 1:
            if n_bottom:
                x, xp = fork(x, 2)
                bottoms = list(fork(MaxPool2.apply(xp), n_bottom))
            else:
                bottoms = []                     # (levels >= 2 without level_root: the pooled map is never used)
        else:
            x, *bottoms = fork(x, 1 + n_bottom)
        if self.level_root:
            children.append(bottoms.pop())
        if self.levels == 1:
            bottom = bottoms.pop()
            residual = conv_bn(bottom, self.project[0], self.project[1], relu=False) if self.project else bottom
            x1 = self.tree1(x, residual)
            x1a, x1b, x1c = fork(x1, 3)          # tree2.conv1, tree2's shortcut, Root
            x2 = self.tree2(x1a, x1b)
            return self.root(x2, x1c, *children)
        x1a, x1b = fork(self.tree1(x), 2)
        children.append(x1b)
        return self.tree2(x1a, children=children)


# dla.py:312-415: levels of level2..level5, channels of base_layer..level5, block, root_residual.  level0 and level1 are one
# 3x3 conv each in every type.  The DLA-X types need grouped 3x3 convolutions, which no kernel here computes.
DLA_TYPES = {
    "dla34": ((1, 2, 2, 1), (16, 32, 64, 128, 256, 512), BasicBlock, False),
    "dla46_c": ((1, 2, 2, 1), (16, 32, 64, 64, 128, 256), Bottleneck, False),
    "dla60": ((1, 2, 3, 1), (16, 32, 128, 256, 512, 1024), Bottleneck, False),
    "dla102": ((1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), Bottleneck, True),
    "dla169": ((2, 3, 5, 1), (16, 32, 128, 256, 512, 1024), Bottleneck, True),
}
DLA_GROUPED_TYPES = ("dla46x_c", "dla60x_c", "dla60x", "dla102x", "dla102x2")


class DLA(nn.Module):
    strides = {"p2": 4, "p3": 8, "p4": 16, "p5": 32, "p6": 64}
    # the 7x7 stride-1 stem runs on the rolling-halo kernel, which takes the image as NHWC8 (3 real channels)
    stem_cpad = 8

    def __init__(self, dla_type="dla34"):
        super().__init__()
        levels, c, block, root_residual = DLA_TYPES[dla_type]
        self.out_channels = {"p2": c[2], "p3": c[3], "p4": c[4], "p5": c[5], "p6": c[5]}      # dla.py:421-450

        def cbr(cin, cout, k, stride=1):
            return nn.Sequential(nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False),
                                 nn.BatchNorm2d(cout), nn.ReLU(inplace=True))
        self.base_layer = cbr(3, c[0], 7)
        self.level0 = cbr(c[0], c[0], 3)
        self.level1 = cbr(c[0], c[1], 3, stride=2)
        for i in range(2, 6):
            setattr(self, "level%d" % i, Tree(levels[i - 2], block, c[i - 1], c[i], 2, level_root=i > 2,
                                              root_residual=root_residual))
        for m in self.modules():            # dla.py:262-268
            if isinstance(m, nn.Conv2d):
                m.weight.data.normal_(0, math.sqrt(2.0 / (m.kernel_size[0] * m.kernel_size[1] * m.out_channels)))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    def forward(self, x):
        for seq in (self.base_layer, self.level0, self.level1):
            x = conv_bn(x, seq[0], seq[1])
        out = {}
        for i, name in zip(range(2, 6), ("p2", "p3", "p4", "p5")):
            x, out[name] = fork(getattr(self, "level%d" % i)(x), 2)      # next level (p5: the p6 subsample) + FPN lateral
        out["p6"] = x[:, ::2, ::2, :].contiguous()        # F.max_pool2d(k=1, s=2), dla.py:474
        return out


class TVResNet(nn.Module):
    """torchvision ResNet-18/34 (BasicBlock) and ResNet-50/101 (Bottleneck) topologies (resnet.py:12-63); parameter names
    and same-seed initialisation of torchvision."""
    strides = DLA.strides
    OUT_CHANNELS = {18: 64, 34: 64, 50: 256, 101: 256}          # p2 width; doubles per stage, p6 = p5 (resnet.py:16-27)

    def __init__(self, depth):
        super().__init__()
        from torchvision import models
        if depth not in self.OUT_CHANNELS:
            raise ValueError("No configuration currently supporting depth of {}".format(depth))
        base = getattr(models, "resnet%d" % depth)(weights=None)
        for k in ("conv1", "bn1", "layer1", "layer2", "layer3", "layer4"):
            setattr(self, k, getattr(base, k))
        c = self.OUT_CHANNELS[depth]
        self.out_channels = {"p2": c, "p3": 2 * c, "p4": 4 * c, "p5": 8 * c, "p6": 8 * c}

    def forward(self, x):
        x = conv_bn(x, self.conv1, self.bn1)
        x = MaxPool3s2.apply(x)              # 3x3 stride-2 pad-1 max pool of the torchvision stem (c3d_maxpool3s2_*)
        out = {}
        for name, layer in zip(("p2", "p3", "p4", "p5"), (self.layer1, self.layer2, self.layer3, self.layer4)):
            for blk in layer:
                x, idn = fork(x, 2)              # conv1 + shortcut (identity or 1x1 downsample)
                if blk.downsample is not None:
                    idn = conv_bn(idn, blk.downsample[0], blk.downsample[1], relu=False)
                y = conv_bn(x, blk.conv1, blk.bn1)
                if hasattr(blk, "conv3"):        # torchvision Bottleneck: 1x1, 3x3 carrying the stride, 1x1 + residual
                    y = conv_bn(y, blk.conv2, blk.bn2)
                    x = conv_bn(y, blk.conv3, blk.bn3, residual=idn)
                else:
                    x = conv_bn(y, blk.conv2, blk.bn2, residual=idn)
            x, out[name] = fork(x, 2)
        out["p6"] = x[:, ::2, ::2, :].contiguous()
        return out


class FPN(nn.Module):
    """detectron2 FPN (SURVEY A.2): fpn_lateral{2..6} 1x1 + fpn_output{2..6} 3x3, both with bias; the
    nearest-x2 upsample + sum of the top-down path is fused into the lateral conv's epilogue."""

    def __init__(self, bottom_up, in_features, out_channels, make_p7=False):
        super().__init__()
        self.bottom_up = bottom_up
        self.in_features = tuple(in_features)
        self.stages = [int(math.log2(bottom_up.strides[f])) for f in in_features]
        for f, s in zip(in_features, self.stages):
            lat = nn.Conv2d(bottom_up.out_channels[f], out_channels, 1)
            out = nn.Conv2d(out_channels, out_channels, 3, padding=1)
            for m in (lat, out):        # c2_xavier_fill
                nn.init.kaiming_uniform_(m.weight, a=1)
                nn.init.constant_(m.bias, 0)
            self.add_module("fpn_lateral%d" % s, lat)
            self.add_module("fpn_output%d" % s, out)
        self.split_backward, self.cut = False, None
        self.size_divisibility = bottom_up.strides[in_features[-1]]
        self._out_features = ["p%d" % s for s in self.stages]
        self.out_strides = {"p%d" % s: 2 ** s for s in self.stages}
        self.out_channels = out_channels
        # ResNet variant: LastLevelMaxPool emits an unused p7 (SURVEY A.2) — never computed here.

    def forward(self, x):
        feats = self.bottom_up(x)
        self.cut = None
        if self.split_backward and torch.is_grad_enabled():
            # FlatSGDTrainer's two-stage backward: the autograd graph is CUT at the bottom-up outputs — stage 1
            # (loss.backward()) stops at detached leaves, stage 2 feeds their gradients into the backbone's own graph
            leaves = {k: v.detach().requires_grad_(True) for k, v in feats.items()}
            self.cut = (feats, leaves)
            feats = leaves
        results, prev = {}, None
        for f, s in reversed(list(zip(self.in_features, self.stages))):
            lat, outc = getattr(self, "fpn_lateral%d" % s), getattr(self, "fpn_output%d" % s)
            prev = ConvBias.apply(feats[f], lat.weight, lat.bias, prev, 1, 0, False, False)
            prev_out, prev = fork(prev, 2) if s != self.stages[0] else (prev, None)     # output conv + next lateral's addend
            results["p%d" % s] = ConvBias.apply(prev_out, outc.weight, outc.bias, None, 1, 1, False, False)
        return {k: results[k] for k in self._out_features}


def _check_weights(cfg):
    if cfg.MODEL.WEIGHTS_PRETRAIN + cfg.MODEL.WEIGHTS == "":
        raise RuntimeError("ImageNet download (dla.py:494-496 / resnet.py:76-79) is impossible offline: set "
                           "MODEL.WEIGHTS_PRETRAIN (or MODEL.WEIGHTS) to a non-empty value for random init")


@BACKBONE_REGISTRY.register()
def build_dla_from_vision_fpn_backbone(cfg, input_shape=None, priors=None):
    _check_weights(cfg)
    t = cfg.MODEL.DLA.TYPE
    if t in DLA_GROUPED_TYPES:
        raise NotImplementedError("MODEL.DLA.TYPE %s needs grouped 3x3 convolutions, which the accelerated path does not "
                                  "compute; supported: %s" % (t, ", ".join(DLA_TYPES)))
    if t not in DLA_TYPES:
        raise NotImplementedError("unknown MODEL.DLA.TYPE %s; supported: %s" % (t, ", ".join(DLA_TYPES)))
    if cfg.MODEL.FPN.NORM != "" or cfg.MODEL.FPN.FUSE_TYPE != "sum":
        raise NotImplementedError("FPN NORM/FUSE_TYPE other than ''/'sum'")
    return FPN(DLA(t), cfg.MODEL.FPN.IN_FEATURES, cfg.MODEL.FPN.OUT_CHANNELS)


@BACKBONE_REGISTRY.register()
def build_resnet_from_vision_fpn_backbone(cfg, input_shape=None, priors=None):
    _check_weights(cfg)
    if not cfg.MODEL.RESNETS.TORCHVISION:
        raise NotImplementedError("MSRA ResNet builder is out of scope (config.py:141 default is torchvision)")
    return FPN(TVResNet(cfg.MODEL.RESNETS.DEPTH), cfg.MODEL.FPN.IN_FEATURES, cfg.MODEL.FPN.OUT_CHANNELS, make_p7=True)


for _n in ("build_densenet_fpn_backbone", "build_mnasnet_fpn_backbone", "build_shufflenet_fpn_backbone"):
    def _unsupported(cfg, input_shape=None, priors=None, _n=_n):
        raise NotImplementedError(f"{_n}: registered for config compatibility; not on the accelerated path")
    BACKBONE_REGISTRY.register(_unsupported, name=_n)

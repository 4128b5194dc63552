"""CPU tests of the Bottleneck backbones (torchvision ResNet-50 / 101, DLA-46-C, DLA-60, DLA-102, DLA-169): the fp32
oracle (tests/bottleneck_oracle.py) against the fixture produced by the reference's own code
(tests/golden/make_bottleneck_golden.py); the product model's state_dict, same-seed init and unused-parameter set against
the same fixture; the types that stay unsupported; and every convolution of each backbone at batch 32 @ 640x640 against
the argument checks and kernel selection of c3d_conv2d / c3d_conv2d_wgrad (the mirror in tests/conv_cases.py)."""
import os

import pytest
import torch
import torch.nn.functional as F

import bottleneck_oracle as bo
import conv_cases as cc
from omni3d_b200 import synth
from oracle import model_io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests/golden/bottleneck_golden.pt"), weights_only=False)
TYPES = list(bo.CASES)


def _product(name, seed=0):
    from omni3d_b200 import cubercnn as pc
    cfg_file, opts, _ = bo.CASES[name]
    cfg = pc.load_cfg(cfg_file, ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cpu"] + list(opts))
    torch.manual_seed(seed)
    return pc.build_model(cfg)


def test_golden_covers_every_type():
    assert sorted(GOLD) == sorted(TYPES)


@pytest.mark.parametrize("name", TYPES)
def test_oracle_matches_reference_run(name):
    """the comparisons and tolerances of test_model_oracle.py::test_oracle_matches_reference_run"""
    from detectron2.utils.events import EventStorage
    _, _, (H, W) = bo.CASES[name]
    g = GOLD[name]
    torch.manual_seed(0)
    model = bo.build_model(bo.load_cfg(name))
    sd = model.state_dict()
    assert set(sd) == set(g["init_sum"]), "state_dict key names differ from the reference"
    assert sum(p.numel() for p in model.parameters()) == g["n_params"]
    for k, v in sd.items():
        assert float(v.double().sum()) == pytest.approx(g["init_sum"][k], rel=1e-13, abs=1e-15), k
        assert float(v.double().abs().sum()) == pytest.approx(g["init_abs"][k], rel=1e-13, abs=1e-15), k
    model.train()
    torch.manual_seed(123)
    with EventStorage(0) as st:
        losses = model(model_io.to_d2_inputs(synth.make_batch(2, H, W, num_gt=4, seed=1)))
        sum(losses.values()).backward()
        scalars = st.latest()
    assert list(losses) == list(g["losses"])
    for k in losses:
        assert torch.allclose(losses[k].detach(), g["losses"][k], rtol=1e-5, atol=1e-7), k
    assert set(scalars) == set(g["scalars"])
    for k, v in scalars.items():
        assert v == pytest.approx(g["scalars"][k], rel=1e-5, abs=1e-7), k
    assert sorted(n for n, p in model.named_parameters() if p.grad is None) == g["no_grad"]
    for n, p in model.named_parameters():
        if p.grad is not None:
            ref = g["grad_norm"][n]
            assert abs(float(p.grad.double().norm()) - ref) <= 1e-4 * ref + 1e-7, n
    model.eval()
    with torch.no_grad():
        res = model(model_io.to_d2_inputs(synth.make_batch(2, H, W, with_gt=False, seed=3)))
    for r, d in zip(res, g["detections"]):
        f = r["instances"].get_fields()
        assert set(f) == set(d)
        for k, v in f.items():
            v = v.tensor if hasattr(v, "tensor") else v
            if v.is_floating_point():
                assert v.shape == d[k].shape and torch.allclose(v, d[k], rtol=1e-4, atol=1e-5), (k, float((v - d[k]).abs().max()))
            else:
                assert torch.equal(v, d[k]), k


@pytest.mark.parametrize("name", TYPES)
def test_product_state_dict_and_unused_set_match_reference(name):
    """a reference checkpoint loads unchanged (same keys, shapes), the same seed gives the reference's initial weights, and
    the trainer's unused region is exactly the set of parameters the reference never gives a gradient"""
    from omni3d_b200.train import unused_parameter_names
    g = GOLD[name]
    model = _product(name)
    sd = model.state_dict()
    assert set(sd) == set(g["init_sum"])
    assert sum(p.numel() for p in model.parameters()) == g["n_params"]
    for k, v in sd.items():
        assert float(v.double().sum()) == pytest.approx(g["init_sum"][k], rel=1e-13, abs=1e-15), k
        assert float(v.double().abs().sum()) == pytest.approx(g["init_abs"][k], rel=1e-13, abs=1e-15), k
    assert sorted(unused_parameter_names(model)) == g["no_grad"]


@pytest.mark.parametrize("name,cfg_file", [("dla34", "cubercnn_DLA34_FPN.yaml"), ("resnet34", "cubercnn_ResNet34_FPN.yaml")])
def test_unused_set_unchanged_for_basicblock_backbones(name, cfg_file):
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import unused_parameter_names
    no_grad = torch.load(os.path.join(ROOT, "tests/golden/model_golden.pt"), weights_only=False)[name]["no_grad"]
    torch.manual_seed(0)
    model = pc.build_model(pc.load_cfg(cfg_file, ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cpu"]))
    assert sorted(unused_parameter_names(model)) == no_grad


@pytest.mark.parametrize("dla_type", ["dla46x_c", "dla60x_c", "dla60x", "dla102x", "dla102x2"])
def test_grouped_dla_types_raise(dla_type):
    from omni3d_b200 import cubercnn as pc
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cpu",
                                                  "MODEL.DLA.TYPE", dla_type])
    with pytest.raises(NotImplementedError, match="grouped 3x3 convolutions"):
        pc.build_model(cfg)


@pytest.mark.parametrize("depth", [152, 26])
def test_other_resnet_depths_raise(depth):
    from omni3d_b200 import cubercnn as pc
    cfg = pc.load_cfg("cubercnn_ResNet34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cpu",
                                                     "MODEL.RESNETS.DEPTH", depth])
    with pytest.raises(ValueError, match="No configuration currently supporting depth of %d" % depth):
        pc.build_model(cfg)


# ---- kernel coverage ------------------------------------------------------------------------------------------------
def _trace_convs(model, N, H, W):
    """every convolution the backbone + FPN forward launches, as (N, H, W, Cin, Cout, k, stride, pad, is_stem), found by
    running the product modules' own forward on meta tensors with the libc3d calls replaced by shape bookkeeping"""
    from omni3d_b200.cubercnn import backbone as B
    convs = []

    def conv(x, cout, k, s, p):
        Nn, Hh, Ww, C = x.shape
        convs.append((Nn, Hh, Ww, C, cout, k, s, p, not convs))          # the first one is the stem
        return torch.empty(Nn, (Hh + 2 * p - k) // s + 1, (Ww + 2 * p - k) // s + 1, cout, device="meta")

    def conv_bn(x, c, bn, residual=None, relu=True):
        return conv(x, c.out_channels, c.kernel_size[0], c.stride[0], c.padding[0])

    class ConvBias:
        @staticmethod
        def apply(x, w, b, addend, stride, pad, *a):
            return conv(x, w.shape[0], w.shape[2], stride, pad)

    def pool(k, s, p):
        class Pool:
            @staticmethod
            def apply(x):
                return F.max_pool2d(x.permute(0, 3, 1, 2), k, s, p).permute(0, 2, 3, 1)
        return Pool

    saved = {k: getattr(B, k) for k in ("conv_bn", "ConvBias", "MaxPool2", "MaxPool3s2")}
    B.conv_bn, B.ConvBias, B.MaxPool2, B.MaxPool3s2 = conv_bn, ConvBias, pool(2, 2, 0), pool(3, 2, 1)
    try:
        cpad = getattr(model.backbone.bottom_up, "stem_cpad", 16)
        with torch.no_grad():
            model.backbone(torch.empty(N, H, W, cpad, device="meta"))
    finally:
        for k, v in saved.items():
            setattr(B, k, v)
    return convs


def _fwd_ok(d):
    """c3d_conv2d_fwd's argument checks and a compiled instance for the selection"""
    inst = cc.fwd_instance(d)
    if inst[0] == "halo":
        return inst[1:] in cc.HALO_FWD + cc.HALO_FWD_GENERIC
    return d.Cin % 16 == 0 and d.Cout % 16 == 0 and d.stride in (1, 2) and inst[1:] in cc.GEMM_FWD


def _wgrad_ok(d):
    (inst, buckets, _) = cc.wgrad_plan(d)
    if inst[0] == "halo":
        return inst[1:] in cc.HALO_WGRAD
    return (d.Cin % 16 == 0 and d.Cout % 16 == 0 and d.stride in (1, 2) and inst[1] in cc.WGRAD_WIDTHS
            and inst[2] in cc.WGRAD_WIDTHS and buckets <= set(cc.WGRAD_NCOLS))


def _dgrad_descs(c):
    """the stride-1 convolutions nnfunc._dgrad launches for the data gradient of case c"""
    Ho, Wo = cc.out_size(cc.desc(c.N, c.H, c.W, c.Cin, c.Cout, c.k, c.s, c.p))
    route = cc.dgrad_route(c, False)
    if route == "stride1":
        return route, [cc.dgrad_desc(c)]
    if route == "merged":
        return route, [cc.desc(c.N, Ho, Wo, c.Cout, 4 * c.Cin, 2, 1, 0, out_hw=(Ho, Wo), y_split_c=2 * c.Cin)]
    if route == "separate":
        return route, [cc.desc(c.N, Ho, Wo, c.Cout, c.Cin, 2, 1, 0, out_hw=(Ho, Wo))]
    return route, [cc.desc(c.N, c.H, c.W, c.Cout, c.Cin, c.k, 1, c.k - 1 - c.p)]       # zero_stuff2: dy scattered to H x W


@pytest.mark.parametrize("name", TYPES)
def test_every_conv_at_batch32_640_has_a_kernel(name):
    model = _product(name)
    convs = _trace_convs(model, 32, 640, 640)
    # every Conv2d of the backbone and FPN is launched, except the `project` of the trees with levels >= 2
    from omni3d_b200.train import unused_parameter_names
    dead = [n for n in unused_parameter_names(model) if n.endswith("project.0.weight")]
    assert len(convs) == sum(1 for m in model.backbone.modules() if isinstance(m, torch.nn.Conv2d)) - len(dead)
    routes = set()
    for (N, H, W, Cin, Cout, k, s, p, stem) in convs:
        c = cc._case(N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=k, s=s, p=p)
        d = cc.fwd_desc(c)
        tag = cc.case_id(c)
        assert _fwd_ok(d), ("forward", tag, cc.fwd_instance(d))
        assert _wgrad_ok(d), ("weight gradient", tag, cc.wgrad_plan(d)[0])
        if stem:                                    # the image needs no data gradient
            continue
        route, descs = _dgrad_descs(c)
        assert route in cc.DGRAD_ROUTES
        routes.add(route)
        for g in descs:
            assert _fwd_ok(g), ("data gradient", route, tag, cc.fwd_instance(g))
    if name.startswith("resnet"):                   # the three 1x1 / stride-2 downsample shortcuts
        assert sum(1 for cv in convs if cv[5] == 1 and cv[6] == 2) == 3 and "zero_stuff2" in routes


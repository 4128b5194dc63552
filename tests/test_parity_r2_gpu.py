"""Round-2 parity tests (VERDICT r1 'what's weak' 1-5): the convolution kernels at the BASELINE shapes that produce the
headline number (multi-tile persistent CTAs, persistent tile loop, full split-K, halo-ring wrap), ResNet34-FPN against
the oracle, a 640x640 model step, the 3x3/s2 max pool, and the packed-weight cache across CUDA-graph replays."""
import os

import pytest
import torch
import torch.nn.functional as F

from omni3d_b200 import synth

pytestmark = pytest.mark.gpu


def _r(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


# name, N, H, W, Cin, Cout, k, stride, pad  — BASELINE configs[1] layer shapes (batch 32 @ 640^2)
REAL_SHAPES = [
    ("fpn_out_256@160", 32, 160, 160, 256, 256, 3, 1, 1),      # top kernel: persistent BN=256, 6400 m-tiles / 132 CTAs
    ("level0_16@640", 32, 640, 640, 16, 16, 3, 1, 1),          # rolling-halo kernel, ring cycles through 640 rows
    ("l3_128@80", 32, 80, 80, 128, 128, 3, 1, 1),
    ("l2_s2_64to128@160", 32, 160, 160, 64, 128, 3, 2, 1),     # stride-2 entry conv (phase-decomposed data gradient)
    ("root_448to128@80", 32, 80, 80, 448, 128, 1, 1, 0),       # Root 1x1, K = 448
    ("l5_512@20", 32, 20, 20, 512, 512, 3, 1, 1),
    ("fpn_lat_64to256@160", 32, 160, 160, 64, 256, 1, 1, 0),
    ("level1_16to32_s2@640", 32, 640, 640, 16, 32, 3, 2, 1),   # data gradient = ONE merged 2x2 conv of dy (split channel placement)
    ("l2_entry_32to64_s2@320", 32, 320, 320, 32, 64, 3, 2, 1),  # merged data gradient, 4*32 = 128 channels
]


@pytest.mark.parametrize("name,N,H,W,Cin,Cout,k,s,p", REAL_SHAPES, ids=[r[0] for r in REAL_SHAPES])
def test_conv_real_shapes_vs_torch_fp32(name, N, H, W, Cin, Cout, k, s, p):
    """fwd / dgrad / wgrad of the wgmma kernels at the batch-32 640x640 shapes vs F.conv2d in fp32 (TF32 off) on the
    same bf16-rounded operands.  Outputs are bf16 => 2^-8 relative; the fp32 weight gradient agrees to accumulation order."""
    from omni3d_b200.nnfunc import ConvBias
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = _r(N, H, W, Cin).bfloat16().requires_grad_(True)
    w = (_r(Cout, Cin, k, k, seed=1) / (k * k * Cin) ** 0.5).requires_grad_(True)
    b = _r(Cout, seed=2).requires_grad_(True)
    y = ConvBias.apply(x, w, b, None, s, p, True, False)
    dy = _r(*y.shape, seed=3).bfloat16()
    y.backward(dy)
    with torch.no_grad():
        wr = w.detach().bfloat16().float()
        # reference in image chunks (fp32 NCHW copies of a 32 x 640 x 640 map are large); wgrad accumulates in fp64
        gw = torch.zeros_like(wr, dtype=torch.float64)
        gb = torch.zeros(Cout, device="cuda", dtype=torch.float64)
        e_y = e_x = 0.0
        m_y = m_x = 0.0
        step = 4
        for i in range(0, N, step):
            xr = x.detach()[i:i + step].float().permute(0, 3, 1, 2).requires_grad_(True)
            wv = wr.clone().requires_grad_(True)
            bv = b.detach().clone().requires_grad_(True)
            with torch.enable_grad():
                yl = F.conv2d(xr, wv, bv, s, p)
                yr = F.relu(yl)
                # the backward is compared under the PRODUCT's ReLU mask: among 10^7..10^8 outputs a few pre-activations lie
                # within fp32 summation-order noise of 0, and one flipped mask bit moves a whole gradient row by O(|dy| |w|)
                mask = (y.detach()[i:i + step] > 0).permute(0, 3, 1, 2)
                yl.backward(dy[i:i + step].float().permute(0, 3, 1, 2) * mask)
            flips = ((yr > 0) != mask).float().mean().item()
            assert flips < 1e-4, (name, "relu mask disagreement", flips)
            e_y = max(e_y, (y.detach()[i:i + step].float() - yr.permute(0, 2, 3, 1)).abs().max().item())
            m_y = max(m_y, yr.abs().max().item())
            e_x = max(e_x, (x.grad[i:i + step].float() - xr.grad.permute(0, 2, 3, 1)).abs().max().item())
            m_x = max(m_x, xr.grad.abs().max().item())
            gw += wv.grad.double()
            gb += bv.grad.double()
    assert e_y <= 1.2e-2 * m_y + 1e-3, (name, "fwd", e_y, m_y)
    assert e_x <= 1.2e-2 * m_x + 1e-3, (name, "dgrad", e_x, m_x)
    # dz = dy * relu-mask is rounded to bf16 once before the weight-gradient GEMM (same in the reference graph up to that
    # rounding): relative Frobenius error of the full gradient
    assert _rel(w.grad.double(), gw) <= 6e-3, (name, "wgrad", _rel(w.grad.double(), gw))
    assert _rel(b.grad.double(), gb) <= 6e-3, (name, "dbias")


def test_conv_bn_stats_real_shape():
    """per-tile BatchNorm partial sums of the persistent kernel at a multi-tile-per-CTA shape vs fp64 sums."""
    from omni3d_b200 import conv as K
    x = _r(32, 80, 80, 128).bfloat16()
    w = (_r(128, 3, 3, 128, seed=1) / (9 * 128) ** 0.5).bfloat16()
    y, stats = K.conv2d_fwd(x, w, stride=1, pad=1, want_stats=True)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, 1, 1)
    tot = stats.double().sum(0)
    s1, s2 = ref.double().sum((0, 2, 3)), (ref.double() ** 2).sum((0, 2, 3))
    assert (tot[0] - s1).abs().max().item() <= 1e-3 * ref.abs().sum((0, 2, 3)).max().item()
    assert (tot[1] - s2).abs().max().item() <= 1e-3 * s2.max().item()
    assert (y.float() - ref.permute(0, 2, 3, 1)).abs().max().item() <= 1.2e-2 * ref.abs().max().item()


@pytest.mark.parametrize("N,H,W,C", [(2, 64, 96, 64), (1, 33, 47, 16), (3, 8, 8, 128)])
def test_maxpool3s2_vs_torch(N, H, W, C):
    from omni3d_b200.nnfunc import MaxPool3s2
    x = _r(N, H, W, C).bfloat16()
    x[0, :4, :4] = 1.0                       # ties: the first maximal element of a window receives the gradient
    x = x.requires_grad_(True)
    y = MaxPool3s2.apply(x)
    dy = _r(*y.shape, seed=1).bfloat16()
    y.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.max_pool2d(xr, 3, 2, 1)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert torch.equal(y.float(), yr.permute(0, 2, 3, 1))
    # sums of up to 4 bf16 gradients, rounded to bf16 once
    assert (x.grad.float() - xr.grad.permute(0, 2, 3, 1)).abs().max().item() <= 2e-2 * xr.grad.abs().max().item()


# ---- ResNet34-FPN (SURVEY 8a-3, BASELINE configs[3]) ----------------------------------------------------------------
@pytest.fixture(scope="module")
def rpair():
    from omni3d_b200 import cubercnn as pc
    from oracle import cubercnn_oracle as co
    torch.manual_seed(0)
    orc = co.build_model(co.load_cfg("cubercnn_ResNet34_FPN.yaml"))
    torch.manual_seed(0)
    prod = pc.build_model(pc.load_cfg("cubercnn_ResNet34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none"]))
    sd = orc.state_dict()
    assert set(sd) == set(prod.state_dict())
    prod.load_state_dict(sd)
    return prod, orc


def _freeze_bn(m):
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eval()


def test_resnet34_fpn_features_frozen_bn(rpair):
    """resnet.py:43-63 + FPN: features of the product path vs the fp32 oracle with BatchNorm on running statistics."""
    prod, orc = rpair
    from oracle import model_io
    items = synth.make_batch(2, 128, 192, with_gt=False, seed=7)
    _freeze_bn(prod); _freeze_bn(orc)
    with torch.no_grad():
        x, _ = prod.preprocess_image(items)
        feats = prod.backbone(x)
        ref = orc.backbone(orc.preprocess_image(model_io.to_d2_inputs(items)).tensor)
    for k in feats:
        assert _rel(feats[k].float().cpu().permute(0, 3, 1, 2), ref[k]) < 3e-2, k


def test_resnet34_train_losses_with_injected_sampling(rpair):
    """all 10 losses of a ResNet34-FPN train forward vs the oracle (the oracle's sampling decisions injected)."""
    prod, orc = rpair
    from oracle_capture import run_oracle_train, to_injection
    for m in orc.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
    prod.load_state_dict(orc.state_dict())
    items = synth.make_batch(2, 128, 192, num_gt=4, seed=1)
    ref_losses, _, cap = run_oracle_train(orc, items)
    prod.train(); prod.zero_grad()
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    assert set(losses) == set(ref_losses)
    for k, v in ref_losses.items():
        got, ref = float(losses[k].detach()), float(v.detach())
        assert abs(got - ref) <= 5e-2 * abs(ref) + 1e-5, (k, got, ref)
    sum(losses.values()).backward()
    assert all(torch.isfinite(p.grad).all() for p in prod.parameters() if p.grad is not None)


# ---- one model step at the BASELINE image size -----------------------------------------------------------------------
def test_dla34_losses_640x640_vs_oracle():
    """2 x 640x640 (the bench's image size: 5 FPN levels up to 160x160, 102 300 anchors / image, multi-tile persistent
    convs, the halo ring over 640 rows): all 10 losses vs the fp32 CPU oracle, relative tolerance only."""
    from omni3d_b200 import cubercnn as pc
    from oracle import cubercnn_oracle as co
    from oracle_capture import run_oracle_train, to_injection
    torch.manual_seed(0)
    orc = co.build_model(co.load_cfg("cubercnn_DLA34_FPN.yaml"))
    torch.manual_seed(0)
    prod = pc.build_model(pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none"]))
    items = synth.make_batch(2, 640, 640, num_gt=8, seed=5)
    ref_losses, _, cap = run_oracle_train(orc, items)
    prod.train()
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    assert set(losses) == set(ref_losses)
    for k, v in ref_losses.items():
        got, ref = float(losses[k].detach()), float(v.detach())
        # the chamfer-based terms take an argmin over corner pairs on a handful of foreground RoIs: one bf16-induced flip moves
        # them by whole percents (cf. test_train_losses_and_grads_frozen_bn)
        rtol = 8e-2 if k in ("Cube/loss_joint", "Cube/loss_pose") else 5e-2
        assert abs(got - ref) <= rtol * abs(ref) + 1e-5, (k, got, ref)
    sum(losses.values()).backward()
    assert all(torch.isfinite(p.grad).all() for p in prod.parameters() if p.grad is not None)


# ---- ADVICE r1 (high): packed bf16 weights across CUDA-graph replays / load_state_dict ------------------------------
def test_eval_after_graph_steps_uses_current_weights():
    """graph steps -> eval -> graph steps -> eval must equal a freshly built model loaded with the same state_dict (the
    replayed SGD kernel rewrites the parameter arena through raw pointers: tensor._version never moves)."""
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import FlatSGDTrainer
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "SOLVER.BASE_LR", 0.004,
                                                  "SOLVER.WARMUP_ITERS", 0, "SOLVER.IMS_PER_BATCH", 2])
    torch.manual_seed(0)
    model = pc.build_model(cfg).train()
    tr = FlatSGDTrainer(cfg, model, use_graph=True)
    batches = [synth.make_batch(2, 128, 192, num_gt=4, seed=30 + j, image_dtype=torch.uint8) for j in range(2)]
    probe = synth.make_batch(1, 128, 192, with_gt=False, seed=99)

    def eval_feats(m):
        m.eval()
        with torch.no_grad():
            x, _ = m.preprocess_image(probe)
            f = m.backbone(x)
        m.train()
        return {k: v.float().clone() for k, v in f.items()}

    for i in range(4):
        tr.step(batches[i % 2])
    assert tr.graph is not None
    f1 = eval_feats(model)
    for i in range(3):
        tr.step(batches[i % 2])
    torch.cuda.synchronize()
    f2 = eval_feats(model)
    fresh = pc.build_model(cfg)
    fresh.load_state_dict(model.state_dict())
    f3 = eval_feats(fresh)
    assert any(not torch.equal(f1[k], f2[k]) for k in f1), "the training steps did not move the features"
    for k in f2:
        assert torch.equal(f2[k], f3[k]), k
    # second model of the same shapes / load_state_dict into a warmed-up model (ADVICE medium: derived temporaries)
    other = pc.build_model(cfg)
    torch.manual_seed(7)
    for p in other.parameters():
        p.data.normal_(0, 0.05)
    f4 = eval_feats(other)
    fresh.load_state_dict(other.state_dict())
    f5 = eval_feats(fresh)
    for k in f4:
        assert torch.equal(f4[k], f5[k]), k


def test_trainer_state_dict_roundtrip():
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import FlatSGDTrainer
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "SOLVER.BASE_LR", 0.01,
                                                  "SOLVER.IMS_PER_BATCH", 2])
    torch.manual_seed(0)
    model = pc.build_model(cfg).train()
    tr = FlatSGDTrainer(cfg, model, use_graph=False)
    batch = synth.make_batch(2, 128, 192, num_gt=4, seed=3, image_dtype=torch.uint8)
    for _ in range(2):
        tr.step(batch)
    sd, msd = tr.state_dict(), {k: v.clone() for k, v in model.state_dict().items()}
    assert sd["iteration"] == 2 and float(sd["momentum"].abs().sum()) > 0
    torch.manual_seed(1)
    model2 = pc.build_model(cfg).train()
    model2.load_state_dict(msd)
    tr2 = FlatSGDTrainer(cfg, model2, use_graph=False)
    tr2.load_state_dict(sd)
    assert tr2.iteration == 2 and torch.equal(tr2.flat_m, tr.flat_m) and torch.equal(tr2.flat_p, tr.flat_p)
    with pytest.raises(NotImplementedError):
        FlatSGDTrainer(pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "SOLVER.NESTEROV", True]), model2)


# ---- FC layers on the wgmma GEMM (VERDICT r1 next#4; SURVEY 8a-9 / 8a-10) ------------------------------------------
@pytest.mark.parametrize("rows,C,PP,N,relu,out_fp32", [(384, 64, 4, 256, True, False), (1000, 1024, 1, 256, False, True),
                                                       (4096, 1024, 1, 768, False, True), (16384, 256, 49, 1024, True, False),
                                                       (200, 128, 1, 64, True, False)])
def test_linear_act_vs_torch(rows, C, PP, N, relu, out_fp32):
    """c3d_linear_fwd/_dgrad/_wgrad (+ bias/ReLU epilogue, (c,p)->(p,c) feature re-ordering of the fc1 weights, weight
    gradient written in the master's order) vs fp32 torch on the same bf16-rounded operands."""
    from omni3d_b200.nnfunc import LinearAct
    torch.backends.cuda.matmul.allow_tf32 = False
    K = C * PP
    x = _r(rows, K).bfloat16().requires_grad_(True)                      # (p, c)-ordered features (NHWC-flattened RoI)
    w = torch.nn.Parameter(_r(N, K, seed=1) / K ** 0.5)                   # master: (c, p)-ordered input features
    b = torch.nn.Parameter(_r(N, seed=2))
    chw = (C, PP) if PP > 1 else None
    y = LinearAct.apply(x, w, b, relu, out_fp32, chw)
    assert y.dtype == (torch.float32 if out_fp32 else torch.bfloat16)
    dy = _r(rows, N, seed=3)
    dy = dy if out_fp32 else dy.bfloat16()
    y.backward(dy)
    xr = x.detach().float().view(rows, PP, C).permute(0, 2, 1).reshape(rows, K).requires_grad_(True)
    wr = w.detach().bfloat16().float().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True)
    yl = F.linear(xr, wr, br)
    yr = F.relu(yl) if relu else yl
    # backward under the product's ReLU mask (see test_conv_real_shapes_vs_torch_fp32)
    mask = (y.detach() > 0) if relu else torch.ones_like(yl, dtype=torch.bool)
    if relu:
        assert ((yr > 0) != mask).float().mean().item() < 1e-4
    yl.backward(dy.float() * mask)
    tol = lambda ref: 1.2e-2 * ref.abs().max().item() + 1e-3
    assert (y.float() - yr).abs().max().item() <= tol(yr)
    gx = xr.grad.view(rows, C, PP).permute(0, 2, 1).reshape(rows, K)
    assert (x.grad.float() - gx).abs().max().item() <= tol(gx)
    # dz is rounded to bf16 before the weight-gradient GEMM when dy arrives in fp32
    assert _rel(w.grad, wr.grad) <= (1e-2 if out_fp32 else 2e-3), _rel(w.grad, wr.grad)
    assert _rel(b.grad, br.grad) <= (1e-2 if out_fp32 else 2e-3)
    # second pass: w.grad / b.grad exist now (like the trainer's flat gradient arena) -> accumulated in place by the kernels
    y2 = LinearAct.apply(x.detach(), w, b, relu, out_fp32, chw)
    y2.backward(dy)
    assert _rel(w.grad, 2 * wr.grad) <= (1e-2 if out_fp32 else 2e-3)
    assert _rel(b.grad, 2 * br.grad) <= (1e-2 if out_fp32 else 2e-3)

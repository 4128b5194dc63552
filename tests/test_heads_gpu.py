"""GPU tests of the fused head kernels (head_loss_ops.cu, row-block linear variants, BatchNorm mask recomputation) against
the product's torch formulations of the same quantities — which in turn are pinned to the oracle by the loss-parity tests in
test_model_gpu.py / test_parity_r2_gpu.py (SURVEY 8a-9, 8a-10, 8a-11)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _r(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _roi_heads(K=50):
    from omni3d_b200.cubercnn.roi_heads import ROIHeads3D
    rh = ROIHeads3D.__new__(ROIHeads3D)
    torch.nn.Module.__init__(rh)
    rh.num_classes, rh.box_weights, rh.stats = K, (10.0, 10.0, 5.0, 5.0), {}
    return rh


def test_box_loss_kernel_vs_torch_formulation():
    from omni3d_b200.nnfunc import BoxLoss
    K, R = 50, 1536
    rh = _roi_heads(K)
    g = torch.Generator(device="cuda").manual_seed(3)
    pred = (_r(R, 256, seed=1) * 0.5).requires_grad_(True)
    classes = torch.randint(-1, K + 1, (R,), device="cuda", generator=g)
    valid = torch.rand(R, device="cuda", generator=g) > 0.2
    classes = torch.where(valid, classes, torch.full_like(classes, -1))
    xy = torch.rand(R, 2, device="cuda", generator=g) * 300
    wh = torch.rand(R, 2, device="cuda", generator=g) * 100 + 10
    boxes = torch.cat([xy, xy + wh], 1)
    gt = boxes + (torch.rand(R, 4, device="cuda", generator=g) - 0.5) * 10
    smp = {"classes": classes[None], "valid": valid[None], "boxes": boxes[None], "gt_boxes": gt[None]}
    # torch formulation (ROIHeads3D.box_losses) on the sliced outputs
    p2 = pred.detach().clone().requires_grad_(True)
    ref = rh.box_losses(p2[:, :K + 1], p2[:, K + 1:5 * K + 1], smp)
    ref_stats = dict(rh.stats)
    (ref["BoxHead/loss_cls"] * 1.3 + ref["BoxHead/loss_box_reg"] * 0.7).backward()
    o = BoxLoss.apply(pred, classes, valid, boxes, gt, K, rh.box_weights)
    (o[0] * 1.3 + o[1] * 0.7).backward()
    assert abs(float(o[0]) - float(ref["BoxHead/loss_cls"])) <= 2e-5 * abs(float(ref["BoxHead/loss_cls"]))
    assert abs(float(o[1]) - float(ref["BoxHead/loss_box_reg"])) <= 2e-5 * abs(float(ref["BoxHead/loss_box_reg"]))
    for i, k in ((2, "fast_rcnn/cls_accuracy"), (3, "fast_rcnn/fg_cls_accuracy"), (4, "fast_rcnn/false_negative")):
        assert abs(float(o[i]) - float(ref_stats[k])) < 1e-6, k
    assert _rel(pred.grad, p2.grad) < 1e-5
    assert (pred.grad[:, 5 * K + 1:] == 0).all()


def test_cube_head_loss_kernel_vs_fused_formulation():
    """CubeHeadLoss (gather + decode/loss + masked finite means straight from the fused predictor rows) == the existing
    path (torch gathers + CubeLossRows + finite_mean), values and gradient w.r.t. the predictor output."""
    from omni3d_b200.cubercnn import geometry as G
    from omni3d_b200.nnfunc import CubeHeadLoss
    K, B, Fc = 50, 4, 32
    n = B * Fc
    rh = _roi_heads(K)
    rh.w = dict(w3d=1.0, xy=1.0, z=1.0, dims=1.0, pose=1.0, joint=1.0, conf=1.0)
    rh.virtual_focal = 512.0
    rh.priors_dims_per_cat = torch.nn.Parameter(torch.rand(1, K, 2, 3, device="cuda") + 0.5)
    g = torch.Generator(device="cuda").manual_seed(5)
    pred = (_r(n, 768, seed=2) * 0.3)
    pred[:, 12 * K:13 * K] += 1.0
    classes = torch.randint(0, K, (n,), device="cuda", generator=g)
    valid = torch.rand(n, device="cuda", generator=g) > 0.25
    classes = torch.where(valid, classes, torch.full_like(classes, -1))
    xy = torch.rand(n, 2, device="cuda", generator=g) * 400 + 20
    wh = torch.rand(n, 2, device="cuda", generator=g) * 120 + 16
    boxes = torch.cat([xy, xy + wh], 1)
    f = torch.rand(B, device="cuda", generator=g) * 400 + 400
    Ks = torch.zeros(B, 3, 3, device="cuda"); Ks[:, 0, 0] = f; Ks[:, 1, 1] = f; Ks[:, 0, 2] = 320; Ks[:, 1, 2] = 240; Ks[:, 2, 2] = 1
    ratios = torch.tensor([1.0, 1.25, 0.8, 1.0], device="cuda")
    hw = torch.tensor([[480.0, 640.0]] * B, device="cuda")
    meta = torch.cat([hw, ratios[:, None], Ks.reshape(B, 9)], 1)
    gt3 = torch.cat([xy + wh / 2, torch.rand(n, 1, device="cuda", generator=g) * 30 + 2,
                     torch.rand(n, 3, device="cuda", generator=g) * 2 + 0.3, torch.zeros(n, 3, device="cuda")], 1)
    q, _ = torch.linalg.qr(_r(n, 3, 3, seed=7))
    gtR = q * torch.sign(torch.linalg.det(q))[:, None, None]
    # existing formulation
    p2 = pred.clone().requires_grad_(True)
    c = classes.clamp(0, K - 1)
    pick = lambda o, m: torch.gather(o.reshape(n, K, m), 1, c[:, None, None].expand(-1, 1, m)).squeeze(1)
    ur = pick(p2[:, 12 * K:13 * K], 1).squeeze(1)
    raw = dict(deltas=pick(p2[:, :2 * K], 2), dims=pick(p2[:, 2 * K:5 * K], 3), pose6=pick(p2[:, 5 * K:11 * K], 6),
               z=pick(p2[:, 11 * K:12 * K], 1).squeeze(1), uncert=ur.clip(0.01), uncert_raw=ur)
    Kb, v2r, _ = rh.per_box_camera(Ks, ratios, hw[:, 0], Fc, B, "cuda")
    ref = rh.cube_losses_fused(raw, boxes, classes, valid, gt3, gtR, Kb, v2r)
    ref_stats = dict(rh.stats)
    wts = [0.9, 1.1, 1.2, 0.8, 1.3, 0.7]
    keys = ["Cube/uncert", "Cube/loss_dims", "Cube/loss_xy", "Cube/loss_z", "Cube/loss_pose", "Cube/loss_joint"]
    sum(w * ref[k] for w, k in zip(wts, keys)).backward()
    p1 = pred.clone().requires_grad_(True)
    got = rh.cube_losses_kernel(p1, boxes, classes, valid, gt3, gtR, meta, Fc)
    sum(w * got[k] for w, k in zip(wts, keys)).backward()
    for k in keys:
        assert abs(float(got[k]) - float(ref[k])) <= 1e-5 * abs(float(ref[k])) + 1e-7, k
    for k in ("Cube/z_error", "Cube/dims_error", "Cube/xy_error", "Cube/z_close", "Cube/conf"):
        assert abs(float(rh.stats[k]) - float(ref_stats[k])) <= 1e-5 * abs(float(ref_stats[k])) + 1e-7, k
    assert _rel(p1.grad, p2.grad) < 1e-5


def test_two_head_fc1_vs_separate_linear_layers():
    from omni3d_b200.nnfunc import LinearAct, TwoHeadFC1
    B, S, Fc, C, PP, N = 4, 64, 16, 64, 4, 256
    D = C * PP
    x = _r(B * S, D).bfloat16()
    mk = lambda seed: torch.nn.Parameter(_r(N, D, seed=seed) / D ** 0.5)
    wb, wc = mk(1), mk(2)
    bb, bc = torch.nn.Parameter(_r(N, seed=3)), torch.nn.Parameter(_r(N, seed=4))
    gb, gc = _r(B * S, N, seed=5).bfloat16(), _r(B * Fc, N, seed=6).bfloat16()
    x1 = x.clone().requires_grad_(True)
    hb, hc = TwoHeadFC1.apply(x1, wb, bb, wc, bc, B, S, Fc, (C, PP))
    torch.autograd.backward([hb, hc], [gb, gc])
    got = [x1.grad.clone(), wb.grad.clone(), bb.grad.clone(), wc.grad.clone(), bc.grad.clone()]
    for p in (wb, bb, wc, bc):
        p.grad = None
    x2 = x.clone().requires_grad_(True)
    rb = LinearAct.apply(x2, wb, bb, True, False, (C, PP))
    xc = x2.view(B, S, D)[:, :Fc].reshape(B * Fc, D)
    rc = LinearAct.apply(xc, wc, bc, True, False, (C, PP))
    torch.autograd.backward([rb, rc], [gb, gc])
    assert torch.equal(hb, rb) and torch.equal(hc, rc)
    ref = [x2.grad, wb.grad, bb.grad, wc.grad, bc.grad]
    # dx: the cube head's rows are accumulated in the conv epilogue (bf16 + fp32 -> bf16) instead of bf16 + bf16
    assert _rel(got[0].float(), ref[0].float()) < 4e-3
    rows = torch.zeros(B, S, dtype=torch.bool, device="cuda"); rows[:, :Fc] = True
    assert torch.equal(got[0].view(B, S, D)[~rows], ref[0].view(B, S, D)[~rows])
    for a, b in zip(got[1:], ref[1:]):
        assert _rel(a, b) < 1e-5


@pytest.mark.parametrize("C,frozen", [(64, False), (256, True)])
def test_bn_backward_mask_recomputed_from_y_equals_mask_from_out(C, frozen):
    """ReLU BatchNorm layers without a residual no longer read `out` in the backward: the sign of
    fma(y - mean, rstd*gamma, beta) is recomputed exactly as the forward produced it => identical dy / dgamma / dbeta."""
    from omni3d_b200 import kernels as Kx
    P = 5000
    y = _r(P, C, seed=1).bfloat16()
    mean, rstd = _r(C, seed=2) * 0.1, torch.rand(C, device="cuda") + 0.5
    gamma, beta = torch.rand(C, device="cuda") + 0.5, _r(C, seed=3) * 0.3
    out = Kx.bn_apply(y, mean, rstd, gamma, beta, None, True)
    dout = _r(P, C, seed=4).bfloat16()
    res = []
    for use_out in (True, False):
        dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        dy, _ = Kx.bn_bwd(dout, out if use_out else None, y, mean, rstd, gamma, True, dg, db, False, frozen=frozen,
                          beta=None if use_out else beta)
        res.append((dy, dg, db))
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a, b)


def _ref_conv_packs(w, phases):
    """torch formulation of the bf16 conv-weight packs: forward (Cout,KH,KW,Cin), data gradient (Cin,KH,KW,Cout) rotated by
    180 degrees, and the stride-2 phase sub-kernels {(a, b): (Cin,KH',KW',Cout)} with parity 0 -> tap [1], parity 1 -> taps
    [2, 0]; "merged": the four phases as 2x2 row blocks of one zero-initialised (4*Cin,2,2,Cout) weight."""
    w = w.detach()
    O, I = w.shape[:2]
    ref = {"fwd": w.permute(0, 2, 3, 1).bfloat16(), "dgrad": w.flip(2, 3).permute(1, 2, 3, 0).bfloat16()}
    if phases is None:
        return ref
    taps = {0: [1], 1: [2, 0]}
    mg = torch.zeros((4 * I, 2, 2, O), device=w.device, dtype=torch.bfloat16)
    for a in (0, 1):
        for b in (0, 1):
            sub = w[:, :, taps[a]][:, :, :, taps[b]].permute(1, 2, 3, 0).bfloat16()
            if phases == "merged":
                blk = mg[(2 * a + b) * I:(2 * a + b + 1) * I]
                blk[:, :sub.shape[1], :sub.shape[2]] = sub
                sub = blk
            ref[(a, b)] = sub
    if phases == "merged":
        ref["merged"] = mg
    return ref


def _check_conv_packs(packs, w, phases):
    f, g, ph = packs
    ref = _ref_conv_packs(w, phases)
    assert torch.equal(f, ref.pop("fwd")) and torch.equal(g, ref.pop("dgrad"))
    if phases is None:
        assert ph is None
        return
    assert ph.keys() == ref.keys()
    for k in ref:
        assert torch.equal(ph[k], ref[k]), k


def test_conv_weight_packs_equal_torch_reference():
    """c3d_pack_conv_weights_batched (one launch for every conv weight of a model) and c3d_pack_conv_weight (one weight)
    == the torch formulation of the forward, data-gradient and stride-2 phase packs, for OIHW and channels-last (trainer
    arena) masters, merged and separate phase layouts; a parameter update invalidates the cached packs."""
    from omni3d_b200 import conv as K
    from omni3d_b200 import nnfunc

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a = torch.nn.Conv2d(16, 32, 3, stride=2, padding=1, bias=False)      # merged phases
            self.b = torch.nn.Conv2d(32, 64, 3, padding=1, bias=False)
            self.c = torch.nn.Conv2d(64, 16, 1, bias=False)
            self.d = torch.nn.Conv2d(32, 272, 3, stride=2, padding=1, bias=False)     # Cout > 256: separate phases
            self.skip = torch.nn.Conv2d(3, 16, 7, padding=3, bias=False)         # Cin 3: not packed here
    net = Net().cuda()
    with torch.no_grad():                          # channels-last storage like the trainer's arena
        for m in (net.b, net.d):
            m.weight.data = m.weight.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    layers = {net.a: "merged", net.b: None, net.c: None, net.d: "separate"}
    assert nnfunc._phase_layout(net.a.weight) == "merged" and nnfunc._phase_layout(net.d.weight) == "separate"
    nnfunc.invalidate_packed()
    assert nnfunc.prepack_model(net) == 4
    for m, phases in layers.items():
        _check_conv_packs(nnfunc._packed(m.weight), m.weight, phases)                    # seeded by prepack_model
        for layout in ("merged", "separate", None) if m.kernel_size == (3, 3) else (None,):         # one weight, one launch
            _check_conv_packs(K.pack_conv_weight(m.weight, phases=layout), m.weight, layout)
    f, _, _ = K.pack_conv_weight(net.b.weight, want_dgrad=False)
    assert torch.equal(f, _ref_conv_packs(net.b.weight, None)["fwd"])
    # a parameter update (version bump) invalidates the seeded entries; the repack of a cached entry without phases adds them
    with torch.no_grad():
        net.c.weight.add_(1.0)
        net.a.weight.mul_(-0.5)
    _check_conv_packs(nnfunc._packed(net.c.weight), net.c.weight, None)
    _check_conv_packs(nnfunc._packed(net.a.weight), net.a.weight, None)
    _check_conv_packs(nnfunc._packed(net.a.weight, phases=True), net.a.weight, "merged")
    nnfunc.invalidate_packed()

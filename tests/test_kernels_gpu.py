"""GPU unit tests of the sm_90a helper kernels against plain PyTorch fp32 references of the same op
(tolerances: bf16 storage => 2^-8 relative on outputs; fp32 accumulations 1e-5)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _r(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s,p", [(2, 32, 32, 64, 64, 3, 1, 1), (1, 20, 20, 256, 128, 3, 1, 1),
                                                  (2, 32, 32, 64, 128, 3, 2, 1), (2, 16, 16, 128, 256, 1, 1, 0),
                                                  (1, 64, 64, 16, 32, 3, 2, 1), (2, 24, 40, 32, 64, 1, 1, 0)])
def test_conv_fwd_dgrad_wgrad_vs_torch(N, H, W, Cin, Cout, k, s, p):
    from omni3d_b200.nnfunc import ConvBias
    torch.backends.cudnn.allow_tf32 = False
    x = _r(N, H, W, Cin).bfloat16().requires_grad_(True)
    w = (_r(Cout, Cin, k, k, seed=1) / (k * k * Cin) ** 0.5).requires_grad_(True)
    b = _r(Cout, seed=2).requires_grad_(True)
    y = ConvBias.apply(x, w, b, None, s, p, True, False)
    dy = _r(*y.shape, seed=3).bfloat16()
    y.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.detach().bfloat16().float().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True)
    yr = F.relu(F.conv2d(xr, wr, br, s, p))
    yr.backward(dy.float().permute(0, 3, 1, 2))
    tol = lambda ref: 1.2e-2 * ref.abs().max().item() + 1e-3
    assert (y.float() - yr.permute(0, 2, 3, 1)).abs().max().item() <= tol(yr)
    assert (x.grad.float() - xr.grad.permute(0, 2, 3, 1)).abs().max().item() <= tol(xr.grad)
    assert (w.grad - wr.grad).abs().max().item() <= 2e-2 * wr.grad.abs().max().item() + 1e-3
    assert (b.grad - br.grad).abs().max().item() <= 1e-2 * br.grad.abs().max().item() + 1e-3


@pytest.mark.parametrize("N,H,W,Cin,Cout,k", [(2, 40, 256, 16, 16, 3), (1, 33, 200, 8, 16, 7), (2, 70, 128, 32, 32, 3),
                                             (1, 9, 384, 16, 32, 5), (3, 35, 130, 32, 16, 3)])
def test_halo_conv_fwd_dgrad_wgrad_vs_torch(N, H, W, Cin, Cout, k):
    """thin-channel stride-1 layers (DLA stem / level0) run on conv_halo_* (rolling input rows in smem, no-swizzle
    UMMA descriptors): ragged strips (W % 128 != 0), chunk boundaries (H > 32) and both K-chunk modes."""
    from omni3d_b200 import conv as K
    from omni3d_b200.nnfunc import ConvBias
    p = k // 2
    x = _r(N, H, W, Cin).bfloat16().requires_grad_(Cin != 8)
    w = (_r(Cout, Cin, k, k, seed=1) / (k * k * Cin) ** 0.5).requires_grad_(True)
    b = _r(Cout, seed=2).requires_grad_(True)
    y = ConvBias.apply(x, w, b, None, 1, p, True, False)
    dy = _r(*y.shape, seed=3).bfloat16()
    y.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.detach().bfloat16().float().requires_grad_(True)
    br = b.detach().clone().requires_grad_(True)
    yr = F.relu(F.conv2d(xr, wr, br, 1, p))
    yr.backward(dy.float().permute(0, 3, 1, 2))
    tol = lambda ref: 1.2e-2 * ref.abs().max().item() + 1e-3
    assert (y.float() - yr.permute(0, 2, 3, 1)).abs().max().item() <= tol(yr)
    if Cin != 8:                      # the 8-channel stem has no data gradient in the model (dgrad needs Cout in {16,32})
        assert (x.grad.float() - xr.grad.permute(0, 2, 3, 1)).abs().max().item() <= tol(xr.grad)
    assert (w.grad - wr.grad).abs().max().item() <= 2e-2 * wr.grad.abs().max().item() + 1e-3
    # per-CTA BatchNorm partial statistics and the OHWI gradient layout
    wp = w.detach().permute(0, 2, 3, 1).contiguous().bfloat16()
    y2, stats = K.conv2d_fwd(x.detach(), wp, stride=1, pad=p, want_stats=True)
    ref = F.conv2d(xr.detach(), wr.detach(), None, 1, p).permute(0, 2, 3, 1)
    tot = stats.double().sum(0)
    assert (tot[0] - ref.double().sum((0, 1, 2))).abs().max().item() <= 2e-3 * ref.abs().sum((0, 1, 2)).max().item() + 1e-2
    assert (tot[1] - (ref.double() ** 2).sum((0, 1, 2))).abs().max().item() <= 2e-3 * (ref.double() ** 2).sum((0, 1, 2)).max().item()
    dz = dy.float() * (yr.permute(0, 2, 3, 1) > 0)
    g2 = K.conv2d_wgrad(x.detach(), dz.bfloat16().contiguous(), k, k, 1, p, oihw=False)
    assert (g2.permute(0, 3, 1, 2) - wr.grad).abs().max().item() <= 2e-2 * wr.grad.abs().max().item() + 1e-3


@pytest.mark.parametrize("C,relu,res", [(64, True, True), (128, True, False), (16, False, False), (512, True, True)])
def test_conv_bn_act_train_vs_torch(C, relu, res):
    from omni3d_b200.nnfunc import ConvBNAct
    N, H, W, Cin = 3, 24, 24, 64
    x = _r(N, H, W, Cin).bfloat16().requires_grad_(True)
    w = (_r(C, Cin, 3, 3, seed=1) / (9 * Cin) ** 0.5).requires_grad_(True)
    gamma = (1 + 0.1 * _r(C, seed=2)).requires_grad_(True)
    beta = (0.1 * _r(C, seed=3)).requires_grad_(True)
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    r = _r(N, H, W, C, seed=4).bfloat16().requires_grad_(True) if res else None
    out = ConvBNAct.apply(x, w, gamma, beta, rm, rv, r, 1, 1, relu, True, 1e-5, 0.1)
    dy = _r(*out.shape, seed=5).bfloat16()
    out.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.detach().bfloat16().float().requires_grad_(True)
    gr, br = gamma.detach().clone().requires_grad_(True), beta.detach().clone().requires_grad_(True)
    rmr, rvr = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    yr = F.batch_norm(F.conv2d(xr, wr, None, 1, 1), rmr, rvr, gr, br, True, 0.1, 1e-5)
    rr = None
    if res:
        rr = r.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
        yr = yr + rr
    if relu:
        yr = F.relu(yr)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    tol = lambda ref, f=2e-2: f * ref.abs().max().item() + 2e-3
    # gradients: relative Frobenius error (a ReLU mask that flips on a near-zero pre-activation moves single
    # elements by a whole dout, so max-abs is not a meaningful bound for the bf16 path)
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    assert (out.float() - yr.permute(0, 2, 3, 1)).abs().max().item() <= tol(yr)
    assert (rm - rmr).abs().max().item() < 1e-3 and (rv - rvr).abs().max().item() < 1e-3
    assert rel(gamma.grad, gr.grad) < 4e-2 and rel(beta.grad, br.grad) < 4e-2
    assert rel(x.grad.float(), xr.grad.permute(0, 2, 3, 1)) < 4e-2
    assert rel(w.grad, wr.grad) < 4e-2
    if res:
        assert rel(r.grad.float(), rr.grad.permute(0, 2, 3, 1)) < 4e-2


def test_maxpool2_fwd_bwd():
    from omni3d_b200.nnfunc import MaxPool2
    x = _r(2, 16, 24, 64).bfloat16().requires_grad_(True)
    y = MaxPool2.apply(x)
    dy = _r(*y.shape, seed=1).bfloat16()
    y.backward(dy)
    xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.max_pool2d(xr, 2, 2)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert torch.equal(y.float(), yr.permute(0, 2, 3, 1))
    assert torch.equal(x.grad.float(), xr.grad.permute(0, 2, 3, 1))


def test_preprocess_matches_reference_formula():
    from omni3d_b200 import kernels as Kx
    imgs = [torch.randint(0, 256, (3, 50, 70), device="cuda").float(), torch.randint(0, 256, (3, 64, 40), device="cuda").float()]
    mean, std = [103.53, 116.28, 123.675], [57.375, 57.12, 58.395]
    m, s = torch.tensor(mean, device="cuda").view(3, 1, 1), torch.tensor(std, device="cuda").view(3, 1, 1)
    mixed = [imgs[0].to(torch.uint8), imgs[1], torch.randint(0, 256, (3, 33, 90), device="cuda", dtype=torch.uint8)]
    for batch, shape in ((imgs, (2, 64, 128, 16)), (mixed, (3, 64, 128, 16))):      # one dtype, then uint8 and fp32 mixed
        out = Kx.preprocess_images(batch, mean, std, 64, 16)
        assert tuple(out.shape) == shape
        for i, im in enumerate(batch):
            ref = ((im.float() - m) / s).bfloat16().float()
            got = out[i, :im.shape[1], :im.shape[2], :3].float().permute(2, 0, 1)
            assert torch.equal(got, ref)
            assert out[i, im.shape[1]:].abs().sum() == 0 and out[i, :, im.shape[2]:].abs().sum() == 0
            assert out[i, ..., 3:].abs().sum() == 0


def test_roi_align_fwd_bwd_vs_torchvision():
    from torchvision.ops import roi_align
    from omni3d_b200.cubercnn.roi_heads import assign_levels
    from omni3d_b200.nnfunc import ROIAlign
    strides = (4, 8, 16, 32, 64)
    N, C = 2, 256
    feats = [(_r(N, 128 // (s // 4), 160 // (s // 4), C, seed=s) * 1.0).bfloat16().requires_grad_(True) for s in strides]
    g = torch.Generator(device="cuda").manual_seed(5)
    R = 300
    xy = torch.rand(R, 2, device="cuda", generator=g) * torch.tensor([560.0, 440.0], device="cuda")
    wh = torch.rand(R, 2, device="cuda", generator=g) ** 2 * 400 + 2
    boxes = torch.cat([xy, xy + wh], 1)
    bi = torch.randint(0, N, (R,), device="cuda", generator=g).float()
    lv = assign_levels(boxes)
    rois = torch.cat([bi[:, None], lv[:, None], boxes], 1).contiguous()
    out = ROIAlign.apply(rois, strides, 7, *feats)
    dy = _r(*out.shape, seed=9).bfloat16()
    out.backward(dy)
    fr = [f.detach().float().permute(0, 3, 1, 2).requires_grad_(True) for f in feats]
    ref = torch.zeros(R, C, 7, 7, device="cuda")
    for l, s in enumerate(strides):
        idx = (lv == l).nonzero().squeeze(1)
        if len(idx):
            ref[idx] = roi_align(fr[l], torch.cat([bi[idx, None], boxes[idx]], 1), (7, 7), 1.0 / s, 0, aligned=True)
    ref.backward(dy.float().permute(0, 3, 1, 2))
    assert (out.float() - ref.permute(0, 2, 3, 1)).abs().max().item() <= 2e-2 * ref.abs().max().item()
    for f, r in zip(feats, fr):
        if r.grad is None:
            continue
        assert (f.grad.float() - r.grad.permute(0, 2, 3, 1)).abs().max().item() <= 2e-2 * r.grad.abs().max().item() + 1e-3


@pytest.mark.parametrize("n,trick", [(900, 4000), (6000, 4000), (3000, 20000)])
def test_nms_batched_exact_vs_torchvision(n, trick):
    from torchvision.ops import batched_nms
    from omni3d_b200 import kernels as Kx
    B = 3
    g = torch.Generator().manual_seed(n)
    xy = torch.rand(B, n, 2, generator=g) * 500
    wh = torch.rand(B, n, 2, generator=g) * 120 + 4
    boxes = torch.cat([xy, xy + wh], 2)
    scores = torch.randn(B, n, generator=g)
    cats = torch.randint(0, 5, (B, n), generator=g).float()
    nvalid = torch.tensor([n, n - 37, n // 2], dtype=torch.int32)
    s_sorted, order = scores.sort(1, descending=True)
    b_sorted = torch.gather(boxes, 1, order[:, :, None].expand(-1, -1, 4))
    c_sorted = torch.gather(cats, 1, order)
    maxc = torch.stack([b_sorted[i, :nvalid[i]].max() for i in range(B)])
    import torchvision
    for grouped in (0, 5):                  # single sorted list vs per-category kernels: both == torchvision
        keep, cnt = Kx.nms_batched(b_sorted.cuda(), nvalid.cuda(), 0.7, 1000, cats=c_sorted.cuda().contiguous(),
                                   maxc=maxc.cuda(), trick_max_numel=trick, ncat=grouped, max_per_cat=n // 8)
        for i in range(B):
            nv = int(nvalid[i])
            bb, ss, cc = b_sorted[i, :nv], s_sorted[i, :nv], c_sorted[i, :nv].long()
            if bb.numel() > trick:      # torchvision's per-category path
                ref = torchvision.ops.boxes._batched_nms_vanilla(bb, ss, cc, 0.7)
            else:
                ref = torchvision.ops.boxes._batched_nms_coordinate_trick(bb, ss, cc, 0.7)
            ref = ref[:1000]
            got = keep[i, :int(cnt[i])].cpu().long()
            assert torch.equal(got, ref), (grouped, i, len(got), len(ref))

def test_sgd_and_finite_flag():
    from omni3d_b200 import kernels as Kx
    n = 100003
    p, g, m = _r(n, seed=1), _r(n, seed=2), torch.zeros(n, device="cuda")
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.SGD([pr], lr=0.02, momentum=0.9, weight_decay=1e-4)
    for _ in range(3):
        pr.grad = g.clone(); opt.step()
        Kx.sgd_momentum(p, g, m, 0.02, 0.9, 1e-4)
    assert (p - pr.detach()).abs().max().item() < 1e-6
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    Kx.grad_finite(g, flag); assert int(flag) == 0
    g[777] = float("inf"); Kx.grad_finite(g, flag); assert int(flag) == 1
    before = p.clone(); Kx.sgd_momentum(p, g, m, 0.02, 0.9, 1e-4, skip_flag=flag); assert torch.equal(p, before)


def test_fused_cube_loss_matches_torch_formulation():
    """c3d_cube_loss_fwd/bwd vs the batched torch fp32 formulation (ROIHeads3D.cube_losses + autograd)."""
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.cubercnn import geometry as G
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "MODEL.DEVICE", "cuda"])
    torch.manual_seed(0)
    heads = pc.ROI_HEADS_REGISTRY.get("ROIHeads3D")(cfg, 256, {"p2": 4, "p3": 8, "p4": 16, "p5": 32, "p6": 64}).cuda()
    heads.priors_dims_per_cat.data.uniform_(0.5, 2.0)
    n = 600
    g = torch.Generator(device="cuda").manual_seed(3)
    R = lambda *s: torch.randn(*s, device="cuda", generator=g)
    U = lambda lo, hi, *s: torch.rand(*s, device="cuda", generator=g) * (hi - lo) + lo
    xy = U(0, 400, n, 2); wh = U(20, 200, n, 2)
    boxes = torch.cat([xy, xy + wh], 1)
    classes = torch.randint(0, 50, (n,), device="cuda", generator=g)
    valid = torch.rand(n, device="cuda", generator=g) > 0.2
    f = U(400, 800, n)
    Kb = torch.zeros(n, 3, 3, device="cuda"); Kb[:, 0, 0] = f; Kb[:, 1, 1] = f; Kb[:, 0, 2] = 320; Kb[:, 1, 2] = 240; Kb[:, 2, 2] = 1
    v2r = U(0.5, 2.0, n)
    gt3 = torch.cat([xy + 0.5 * wh + R(n, 2) * 5, U(2, 40, n, 1), U(0.3, 3, n, 3), R(n, 3)], 1)
    q, _ = torch.linalg.qr(R(n, 3, 3)); gtR = q
    base = dict(deltas=R(n, 2) * 0.1, dims=R(n, 3) * 0.3, pose6=R(n, 6) * 0.5, z=U(1, 30, n), ur=U(-0.2, 5.0, n))
    out = {}
    for mode in ("torch", "fused"):
        leaves = {k: v.clone().requires_grad_(True) for k, v in base.items()}
        raw = dict(deltas=leaves["deltas"], dims=leaves["dims"], pose6=leaves["pose6"], z=leaves["z"],
                   uncert=leaves["ur"].clip(0.01), uncert_raw=leaves["ur"])
        fn = heads.cube_losses if mode == "torch" else heads.cube_losses_fused
        losses = fn(raw, boxes, classes, valid, gt3, gtR, Kb, v2r)
        sum(v * (i + 1) for i, v in enumerate(losses.values())).backward()
        out[mode] = ({k: float(v) for k, v in losses.items()}, {k: v.grad.clone() for k, v in leaves.items()},
                     {k: float(v) for k, v in heads.stats.items() if k.startswith("Cube/")})
    for k, v in out["torch"][0].items():
        assert abs(out["fused"][0][k] - v) <= 1e-4 * abs(v) + 1e-6, (k, out["fused"][0][k], v)
    for k, gref in out["torch"][1].items():
        gf = out["fused"][1][k]
        assert ((gf - gref).norm() / (gref.norm() + 1e-12)).item() < 2e-3, k    # chamfer argmin ties aside
    for k in ("Cube/z_error", "Cube/dims_error", "Cube/xy_error", "Cube/conf"):
        assert abs(out["fused"][2][k] - out["torch"][2][k]) <= 1e-4 * abs(out["torch"][2][k]) + 1e-6, k


@pytest.mark.parametrize("B,G,thr", [(3, 6, 0.7), (2, 1, 0.3), (4, 37, 0.05)])
def test_anchor_match_kernel_equals_torch_formulation(B, G, thr):
    """c3d_anchor_match (2 launches) == the (B,G,A) torch passes it replaces, bit for bit: matched GT, IoU, labels with
    low-quality matches, per-GT arg-max anchors, ignore-region IoA; incl. padded / ignore GTs and an image without GT."""
    from omni3d_b200.cubercnn import rpn as prpn
    ag = prpn.AnchorGenerator([[32], [64], [128], [256], [512]], [[0.5, 1.0, 2.0]], [4, 8, 16, 32, 64])
    anchors = torch.cat(ag([(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)], torch.device("cuda")))
    g = torch.Generator(device="cuda").manual_seed(B * 100 + G)
    xy = torch.rand(B, G, 2, device="cuda", generator=g) * torch.tensor([200.0, 140.0], device="cuda")
    wh = torch.rand(B, G, 2, device="cuda", generator=g) * 120 + 4
    boxes = torch.cat([xy, xy + wh], -1)
    boxes[0, 0] = anchors[777]                                 # an exact hit (IoU == 1) and a duplicate GT (ties)
    if G > 1:
        boxes[0, 1] = boxes[0, 0]
    present = torch.rand(B, G, device="cuda", generator=g) > 0.2
    ignore = torch.rand(B, G, device="cuda", generator=g) > 0.7
    present[-1] = False                                        # image without any GT
    valid, ign = present & ~ignore, present & ignore
    head = prpn.RPNWithIgnore.__new__(prpn.RPNWithIgnore)
    head.iou_thresholds = [thr, thr]
    got = prpn.RPNWithIgnore.match_anchors(head, anchors, boxes, valid, ign)
    ref = prpn.RPNWithIgnore.match_anchors(head, anchors.cpu(), boxes.cpu(), valid.cpu(), ign.cpu())
    names = ["matched_idx", "matched_iou", "labels", "best", "max_ioa"]
    for n, a, b in zip(names, got, ref):
        if n == "matched_idx":       # ties between duplicate GT boxes: both resolve to the first one
            assert torch.equal(boxes.cpu()[torch.arange(B)[:, None], a.cpu()], boxes.cpu()[torch.arange(B)[:, None], b]), n
            assert torch.equal(a.cpu(), b), n
        else:
            assert torch.equal(a.cpu(), b), n


def test_fused_rpn_loss_matches_torch_formulation():
    """c3d_rpn_loss_fwd/bwd == RPNWithIgnore.losses() written with torch ops (values, statistics and both gradients)."""
    from omni3d_b200.cubercnn import rpn as prpn
    ag = prpn.AnchorGenerator([[32], [64], [128], [256], [512]], [[0.5, 1.0, 2.0]], [4, 8, 16, 32, 64])
    anchors = torch.cat(ag([(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)], torch.device("cuda")))
    A, B, G = anchors.shape[0], 3, 5
    g = torch.Generator(device="cuda").manual_seed(7)
    xy = torch.rand(B, G, 2, device="cuda", generator=g) * torch.tensor([160.0, 110.0], device="cuda")
    boxes = torch.cat([xy, xy + torch.rand(B, G, 2, device="cuda", generator=g) * 100 + 8], -1)
    head = prpn.RPNWithIgnore.__new__(prpn.RPNWithIgnore)
    head.iou_thresholds, head.weights, head.batch_size_per_image = [0.3, 0.3], (1.0, 1.0, 1.0, 1.0), 256
    valid = torch.ones(B, G, dtype=torch.bool, device="cuda")
    idx, _, lab, _, _ = head.match_anchors(anchors, boxes, valid)
    lab = torch.where(torch.rand(B, A, device="cuda", generator=g) < 0.1, torch.full_like(lab, -1), lab)   # some ignored
    out = {}
    for fused in (False, True):
        head.fused_loss = fused
        logits = torch.randn(B, A, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)).requires_grad_(True)
        deltas = (0.5 * torch.randn(B, A, 4, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))).requires_grad_(True)
        losses = head.losses(anchors, logits, deltas, lab, idx, boxes)
        (losses["rpn/cls"] * 1.7 + losses["rpn/loc"] * 0.6).backward()
        out[fused] = (losses, dict(head.stats), logits.grad, deltas.grad)
    for k in ("rpn/cls", "rpn/loc"):
        a, b = float(out[True][0][k]), float(out[False][0][k])
        assert abs(a - b) <= 1e-4 * abs(b) + 1e-6, (k, a, b)
    for k, v in out[False][1].items():
        assert abs(float(out[True][1][k]) - float(v)) <= 1e-4 * abs(float(v)) + 1e-5, k
    for i in (2, 3):
        ref = out[False][i]
        assert (out[True][i] - ref).abs().max().item() <= 1e-5 * ref.abs().max().item() + 1e-9


def test_fused_proposal_decode_matches_torch_formulation():
    """RPNWithIgnore.predict_proposals with c3d_rpn_decode_level + grouped NMS == the torch-op formulation + single-list
    NMS: identical proposal boxes, scores and counts (bit for bit), incl. non-finite deltas and tiny boxes."""
    from omni3d_b200 import cubercnn as pc
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none"])
    torch.manual_seed(0)
    rpn = pc.build_model(cfg).proposal_generator.train()
    shapes = [(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)]
    anchors_l = rpn.anchor_generator(shapes, torch.device("cuda"))
    B = 3
    g = torch.Generator(device="cuda").manual_seed(5)
    logits = [torch.randn(B, a.shape[0], device="cuda", generator=g) for a in anchors_l]
    deltas = [0.7 * torch.randn(B, a.shape[0], 4, device="cuda", generator=g) for a in anchors_l]
    deltas[0][0, :50, 2] = float("nan"); deltas[1][1, :20, 0] = float("inf"); deltas[2][2, :10, 2:] = -20.0
    sizes = [(160, 224), (150, 200), (160, 224)]
    out = {}
    for fused in (False, True):
        rpn.fused_decode = fused
        out[fused] = rpn.predict_proposals(anchors_l, logits, deltas, sizes)
    rpn.fused_decode = True
    for a, b, name in zip(out[True], out[False], ("boxes", "scores", "count")):
        assert torch.equal(a, b), name
    assert int(out[True][2].min()) > 100


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s", [(2, 23, 37, 64, 128, 3, 1), (3, 24, 36, 128, 64, 3, 1), (2, 46, 30, 64, 128, 3, 2),
                                                (1, 80, 80, 192, 128, 1, 1), (2, 9, 11, 64, 64, 3, 1)])
@pytest.mark.parametrize("mode", ["stats", "relu_add", "up2", "fp32"])
def test_conv_swapped_kernel_epilogue_modes(N, H, W, Cin, Cout, k, s, mode):
    """Layers with 64 / 128 output channels (formerly a separate Cout-as-M kernel, now the general persistent kernel):
    every epilogue mode on ragged maps (partial tiles in both directions) vs fp32 torch."""
    from omni3d_b200 import conv as K
    torch.backends.cudnn.allow_tf32 = False
    p = k // 2
    x = _r(N, H, W, Cin).bfloat16()
    w = (_r(Cout, k, k, Cin, seed=1) / (k * k * Cin) ** 0.5).bfloat16()
    b = _r(Cout, seed=2)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), None, s, p)      # NCHW fp32
    Ho, Wo = ref.shape[2], ref.shape[3]
    tol = 1.2e-2 * ref.abs().max().item() + 1e-3
    if mode == "stats":
        y, stats = K.conv2d_fwd(x, w, None, stride=s, pad=p, want_stats=True)
        tot = stats.double().sum(0)
        s1, s2 = ref.double().sum((0, 2, 3)), (ref.double() ** 2).sum((0, 2, 3))
        assert (tot[0] - s1).abs().max().item() <= 1e-3 * ref.abs().sum((0, 2, 3)).max().item()
        assert (tot[1] - s2).abs().max().item() <= 1e-3 * s2.max().item()
        assert (y.float() - ref.permute(0, 2, 3, 1)).abs().max().item() <= tol
    elif mode == "relu_add":
        add = _r(N, Ho, Wo, Cout, seed=4).bfloat16()
        y = K.conv2d_fwd(x, w, b, stride=s, pad=p, relu=True, addend=add)
        want = F.relu(ref.permute(0, 2, 3, 1) + b + add.float())
        assert (y.float() - want).abs().max().item() <= tol + 1.2e-2 * add.float().abs().max().item()
    elif mode == "up2":
        if Ho % 2 or Wo % 2:
            # an odd output has no nearest-x2 source map: the entry point refuses it (C3D_EINVAL) before anything is launched
            from omni3d_b200 import _lib
            add = _r(N, (Ho + 1) // 2, (Wo + 1) // 2, Cout, seed=4).bfloat16()
            with pytest.raises(_lib.C3DError, match="even output"):
                K.conv2d_fwd(x, w, b, stride=s, pad=p, addend=add, up2=True)
            return
        add = _r(N, Ho // 2, Wo // 2, Cout, seed=4).bfloat16()
        y = K.conv2d_fwd(x, w, b, stride=s, pad=p, addend=add, up2=True)
        up = add.float().repeat_interleave(2, 1).repeat_interleave(2, 2)
        want = ref.permute(0, 2, 3, 1) + b + up
        assert (y.float() - want).abs().max().item() <= tol + 1.2e-2 * add.float().abs().max().item()
    else:
        y = K.conv2d_fwd(x, w, b, stride=s, pad=p, out_fp32=True)
        assert y.dtype == torch.float32
        assert (y - (ref.permute(0, 2, 3, 1) + b)).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-4


def test_reductions_are_run_to_run_deterministic():
    """the same inputs give bit-identical results on every call: split-K / per-CTA weight-gradient partials are summed in
    a fixed order, ROIAlign backward accumulates order-independently, and the top-k keeps the lowest indices of the
    values tied at its threshold (not the first to arrive)"""
    from omni3d_b200 import conv as K
    from omni3d_b200 import kernels as Kx
    # weight gradients: one many-split GEMM layer and one thin-channel (halo) layer
    for (N, H, W, Cin, Cout) in [(8, 64, 64, 64, 64), (4, 128, 128, 16, 16)]:
        x = _r(N, H, W, Cin, seed=1).bfloat16()
        dy = _r(N, H, W, Cout, seed=2).bfloat16()
        a = K.conv2d_wgrad(x, dy, 3, 3, 1, 1)
        b = K.conv2d_wgrad(x, dy, 3, 3, 1, 1)
        assert torch.equal(a, b), (Cin, Cout)
    # ROIAlign backward: many overlapping RoIs on one map
    feats = [_r(2, 64, 64, 64, seed=3).bfloat16()]
    g = torch.Generator(device="cuda").manual_seed(4)
    xy = torch.rand(400, 2, device="cuda", generator=g) * 40
    wh = torch.rand(400, 2, device="cuda", generator=g) * 40 + 8
    rois = torch.cat([(torch.arange(400, device="cuda") % 2).float()[:, None], torch.zeros(400, 1, device="cuda"),
                      xy, xy + wh], 1).contiguous()
    dout = _r(400, 7, 7, 64, seed=5).bfloat16()
    ga = Kx.roi_align_bwd(feats, [1.0], rois, dout)
    gb = Kx.roi_align_bwd(feats, [1.0], rois, dout)
    assert torch.equal(ga[0], gb[0])
    # top-k with a run of ties at the threshold: the lowest tied indices are kept
    v = torch.zeros(1, 5000, device="cuda")
    v[0, 4000:] = 1.0                                    # 1000 values above the tie
    vals, idx = Kx.topk_segments([(v, 1500)])
    kept = idx[0, 1000:].long().sort().values
    assert torch.equal(kept, torch.arange(500, device="cuda"))

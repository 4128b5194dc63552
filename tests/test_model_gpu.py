"""GPU parity of the accelerated Cube R-CNN path against the CPU fp32 oracle (oracle/cubercnn_oracle).
bf16 tensor-core convs => stated tolerances on activations / losses; RNG-dependent sampling decisions are
injected from the oracle run (SURVEY.md section 7 sampling protocol)."""
import pytest
import torch

from omni3d_b200 import synth

pytestmark = pytest.mark.gpu

H, W = 128, 192


@pytest.fixture(scope="module")
def pair():
    from omni3d_b200 import cubercnn as pc
    from oracle import cubercnn_oracle as co
    torch.manual_seed(0)
    orc = co.build_model(co.load_cfg("cubercnn_DLA34_FPN.yaml"))
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none"])
    torch.manual_seed(0)
    prod = pc.build_model(cfg)
    sd = orc.state_dict()
    for k, v in prod.state_dict().items():          # same-seed init is bit-identical to the oracle/reference
        assert torch.equal(v.cpu(), sd[k]), k
    return prod, orc


def _sync_state(prod, orc):
    """start every test from the oracle's exact parameters AND BatchNorm running statistics (earlier
    train-mode tests moved each model's running stats along its own fp32 / bf16 trajectory)."""
    for m in orc.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
    prod.load_state_dict(orc.state_dict())


def _freeze_bn(m, frozen=True):
    """cubercnn/solver/build.py:71-76 freeze_bn: BatchNorm layers use their running statistics."""
    m.train()
    if frozen:
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.eval()


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def test_backbone_fpn_features_frozen_bn(pair):
    """With BatchNorm on running statistics the bf16 tensor-core path tracks the fp32 oracle closely."""
    prod, orc = pair
    from oracle import model_io
    items = synth.make_batch(2, H, W, with_gt=False, seed=7)
    _sync_state(prod, orc)
    _freeze_bn(prod); _freeze_bn(orc)
    with torch.no_grad():
        x, _ = prod.preprocess_image(items)
        feats = prod.backbone(x)
        ref = orc.backbone(orc.preprocess_image(model_io.to_d2_inputs(items)).tensor)
    for k in ref:
        assert _rel(feats[k].float().cpu().permute(0, 3, 1, 2), ref[k]) < 3e-2, k


def test_backbone_train_bn_matches_bf16_library_baseline(pair):
    """Train-mode BatchNorm on a randomly initialised DLA34 amplifies ANY bf16 rounding (stock PyTorch bf16
    autocast / cuDNN drifts 17-27% from fp32 on these inputs): the stated tolerance for this regime is
    'not further from the fp32 oracle than the stock bf16 library path', layer group by layer group."""
    import copy
    prod, orc = pair
    from oracle import model_io
    items = synth.make_batch(2, H, W, with_gt=False, seed=7)
    prod.train(); orc.train()
    with torch.no_grad():
        xr = orc.preprocess_image(model_io.to_d2_inputs(items)).tensor
        ref = orc.backbone(xr)
        lib = copy.deepcopy(orc.backbone).cuda().train()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            f16 = lib(xr.cuda())
        x, _ = prod.preprocess_image(items)
        mine = prod.backbone(x)
    for k in ref:
        e_lib = _rel(f16[k].float().cpu(), ref[k])
        e_mine = _rel(mine[k].float().cpu().permute(0, 3, 1, 2), ref[k])
        assert e_mine <= 1.3 * e_lib + 0.02, (k, e_mine, e_lib)


def test_backbone_stages_teacher_forced(pair):
    """Every DLA stage fed the ORACLE's (bf16-rounded) input: per-stage error of the fused conv+BN(train)
    kernels without the cross-stage amplification."""
    prod, orc = pair
    from oracle import model_io
    from omni3d_b200.cubercnn.backbone import conv_bn
    items = synth.make_batch(2, H, W, with_gt=False, seed=9)
    prod.train(); orc.train()
    bu, ob = prod.backbone.bottom_up, orc.backbone.bottom_up
    with torch.no_grad():
        b = orc.preprocess_image(model_io.to_d2_inputs(items)).tensor
        x0, _ = prod.preprocess_image(items)
        for name in ("base_layer", "level0", "level1", "level2", "level3", "level4", "level5"):
            bq = b.bfloat16().float()
            a_in = x0 if name == "base_layer" else bq.permute(0, 2, 3, 1).contiguous().cuda().bfloat16()
            if name in ("base_layer", "level0", "level1"):
                seq = getattr(bu, name)
                a = conv_bn(a_in, seq[0], seq[1])
            else:
                a = getattr(bu, name)(a_in)
            b = getattr(ob, name)(bq)
            assert _rel(a.float().cpu().permute(0, 3, 1, 2), b) < 4e-2, name


def test_train_losses_with_injected_sampling(pair):
    prod, orc = pair
    from oracle_capture import run_oracle_train, to_injection
    items = synth.make_batch(2, H, W, num_gt=4, seed=1)
    ref_losses, _, cap = run_oracle_train(orc, items)
    prod.train(); prod.zero_grad()
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    assert set(losses) == set(ref_losses)
    for k, v in ref_losses.items():
        got, ref = float(losses[k].detach()), float(v.detach())
        assert abs(got - ref) <= 5e-2 * abs(ref) + 2e-3, (k, got, ref)       # fp32 oracle vs bf16 path


def test_train_losses_and_grads_frozen_bn(pair):
    """Full model, BatchNorm frozen (MODEL.USE_BN False semantics): losses AND parameter gradients of the
    CUDA path (wgmma dgrad/wgrad, BN/ROIAlign backward kernels) against the fp32 oracle."""
    prod, orc = pair
    from oracle_capture import run_oracle_train, to_injection
    items = synth.make_batch(2, H, W, num_gt=4, seed=2)
    _sync_state(prod, orc)
    _freeze_bn(orc)
    orc_train = orc.train
    orc.train = lambda *a, **k: orc            # keep BN frozen inside run_oracle_train
    try:
        ref_losses, _, cap = run_oracle_train(orc, items)
    finally:
        orc.train = orc_train
    _freeze_bn(prod); prod.zero_grad()
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    for k, v in ref_losses.items():
        got, ref = float(losses[k].detach()), float(v.detach())
        # the chamfer-based terms take an argmin over corner pairs per RoI on a handful of foreground RoIs: a bf16
        # rounding flip moves them by whole percents (seen: 3.4 % after a change of fp32 summation order only)
        rtol = 6e-2 if k in ("Cube/loss_joint", "Cube/loss_pose") else 3e-2
        assert abs(got - ref) <= rtol * abs(ref) + 2e-3, (k, got, ref)
    sum(losses.values()).backward()
    ref_g = {n: p.grad for n, p in orc.named_parameters() if p.grad is not None}
    got_g = {n: p.grad for n, p in prod.named_parameters() if p.grad is not None}
    assert set(ref_g) == set(got_g)
    errs = sorted((_rel(got_g[n].float().cpu(), g), n) for n, g in ref_g.items() if g.norm() > 1e-7)
    med = errs[len(errs) // 2][0]
    p95 = errs[int(0.95 * len(errs))][0]
    # bf16 activations/gradients through ~35 conv layers + ReLU-mask flips (the per-kernel backward tests in
    # test_kernels_gpu.py hold 4e-2); bound it at 0.12 / 0.30
    assert med < 0.12 and p95 < 0.30, (med, p95, errs[-5:])


def test_proposals_exact_given_oracle_head_outputs(pair):
    """'bit-exact proposal indexing': same fp32 logits/deltas in => identical top-k / NMS keep lists out."""
    prod, orc = pair
    from oracle import model_io
    items = synth.make_batch(2, H, W, with_gt=False, seed=11)
    orc.eval(); prod.eval()
    d2 = model_io.to_d2_inputs(items)
    with torch.no_grad():
        images = orc.preprocess_image(d2)
        f = orc.backbone(images.tensor)
        pg = orc.proposal_generator
        feats = [f[k] for k in pg.in_features]
        anchors = pg.anchor_generator(feats)
        lg, dl = pg.rpn_head(feats)
        lg = [s.permute(0, 2, 3, 1).flatten(1) for s in lg]
        dl = [x.view(x.shape[0], -1, 4, x.shape[-2], x.shape[-1]).permute(0, 3, 4, 1, 2).flatten(1, -2) for x in dl]
        ref = pg.predict_proposals(anchors, lg, dl, images.image_sizes)
        mine = prod.proposal_generator
        mine.nms_trick_max_numel = 4000          # the CPU oracle runs torchvision's CPU threshold
        boxes, scores, cnt = mine.predict_proposals([a.tensor.cuda() for a in anchors], [t.cuda() for t in lg],
                                                    [t.cuda() for t in dl], images.image_sizes)
    for i, r in enumerate(ref):
        n = int(cnt[i])
        assert n == len(r)
        # identical selection and order (logits are copied bit-for-bit); box coordinates agree to the last
        # ulps only (exp() differs between the CPU and CUDA math libraries)
        assert torch.equal(scores[i, :n].cpu(), r.objectness_logits)
        assert torch.allclose(boxes[i, :n].cpu(), r.proposal_boxes.tensor, atol=1e-3, rtol=1e-5)


def test_inference_runs_and_matches_loosely(pair):
    prod, orc = pair
    from oracle import model_io
    items = synth.make_batch(2, H, W, with_gt=False, seed=3)
    prod.eval(); orc.eval()
    with torch.no_grad():
        got = prod(items)
        ref = orc(model_io.to_d2_inputs(items))
    for g, r in zip(got, ref):
        gi, ri = g["instances"], r["instances"]
        assert set(gi.get_fields()) == set(ri.get_fields())
        assert len(gi) > 0 and tuple(gi.pred_bbox3D.shape[1:]) == (8, 3)
        assert abs(float(gi.scores.mean()) - float(ri.scores.mean())) < 0.05


def test_cuda_graph_step_matches_eager_step():
    """FlatSGDTrainer replays the recorded step body (CUDA graph) after two eager steps.  With lr = 0 the parameters
    stay put, so an eager trainer and the graph-replaying one see the same model: their losses on the same batches
    agree up to the random anchor / proposal sampling (different philox offsets), new inputs really reach the static
    buffers (different batches -> different losses), and the status read-back / launch accounting keep working."""
    from omni3d_b200 import _lib
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200.train import FlatSGDTrainer
    cfg = pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none", "SOLVER.BASE_LR", 0.0,
                                                  "SOLVER.IMS_PER_BATCH", 2])
    batches = [synth.make_batch(2, H, W, num_gt=4, seed=20 + j, image_dtype=torch.uint8 if j else torch.uint8) for j in range(3)]
    tot = {}
    for mode in (False, True):
        torch.manual_seed(0)
        model = pc.build_model(cfg)
        model.train()
        tr = FlatSGDTrainer(cfg, model, use_graph=mode)
        p0 = tr.flat_p.clone()
        vals = []
        for i in range(6):
            n0 = _lib.LAUNCHES["n"]
            tr.step(batches[i % 3])
            st = tr.status(wait=True)
            assert st is not None and all(v == v for v in st["losses"].values())
            vals.append(st["total_loss"])
            assert _lib.LAUNCHES["n"] - n0 > 100
        assert (tr.graph is not None) == mode
        assert torch.equal(tr.flat_p, p0)                     # lr = 0
        assert st["iterations_success"] + st["iterations_explode"] == 6
        tot[mode] = vals
    for a, b in zip(tot[False], tot[True]):
        assert abs(a - b) <= 0.12 * abs(a), (tot[False], tot[True])
    # steps 3..5 replay the graph on three different batches
    assert len({round(v, 4) for v in tot[True][3:]}) == 3, tot[True]


def test_inference_stages_vs_oracle(pair):
    """Inference parity stage by stage (the discrete post-processing is compared bit-exactly on identical inputs in
    test_select_gpu.py): with the ORACLE's proposals, (1) the dense box-head outputs — softmax scores and per-class decoded
    boxes of every proposal — and, with the ORACLE's detections, (2) the cube head's 3D outputs (centre, dimensions, pose,
    corners, confidence) agree with the fp32 oracle within the bf16 tolerance.  Eval-mode BatchNorm (running statistics)."""
    prod, orc = pair
    from oracle import model_io
    _sync_state(prod, orc)
    items = synth.make_batch(2, H, W, with_gt=False, seed=3)
    prod.eval(); orc.eval()
    d2 = model_io.to_d2_inputs(items)
    with torch.no_grad():
        images = orc.preprocess_image(d2)
        f = orc.backbone(images.tensor)
        props, _ = orc.proposal_generator(images, f, None)
        rh = orc.roi_heads
        feats_o = [f[k] for k in rh.box_in_features]
        pred = rh.box_predictor(rh.box_head(rh.box_pooler(feats_o, [p.proposal_boxes for p in props])))
        o_probs = rh.box_predictor.predict_probs(pred, props)
        o_boxes = rh.box_predictor.predict_boxes(pred, props)
        ref = orc(d2)
        # product, teacher-forced with the oracle's proposals
        x, sizes = prod.preprocess_image(items)
        feats = prod.backbone(x)
        pr = prod.roi_heads
        fl = [feats[k] for k in pr.in_features]
        P = max(len(p) for p in props)
        pb = torch.zeros(len(props), P, 4); pc = torch.zeros(len(props), dtype=torch.int32)
        for i, p in enumerate(props):
            pb[i, :len(p)], pc[i] = p.proposal_boxes.tensor, len(p)
        probs, pboxes = pr.box_dense(fl, pb.cuda(), pc.cuda())
    K = pr.num_classes
    for i, p in enumerate(props):
        n = len(p)
        # random-init FPN features are large, so the class logits span several units and the softmax is peaked: compare the
        # (centred) logits, where the bf16 error is a few percent, not the saturating probabilities
        lp, lo = torch.log(probs[i, :n].cpu().clamp(min=1e-30)), torch.log(o_probs[i].clamp(min=1e-30))
        assert _rel(lp - lp.mean(-1, keepdim=True), lo - lo.mean(-1, keepdim=True)) < 6e-2
        assert (probs[i, :n].cpu().argmax(-1) == o_probs[i].argmax(-1)).float().mean().item() > 0.9
        ob = o_boxes[i].view(n, K, 4)
        size = (ob[..., 2:] - ob[..., :2]).abs().amax(-1, keepdim=True)
        assert ((pboxes[i, :n].cpu() - ob).abs() <= 0.03 * size + 0.5).all()
    # (2) cube head on the oracle's own detections
    D = max(len(r["instances"]) for r in ref)
    if D == 0:
        pytest.skip("oracle produced no detections")
    db = torch.zeros(len(ref), D, 4); dc = torch.zeros(len(ref), D, dtype=torch.long); dv = torch.zeros(len(ref), D, dtype=torch.bool)
    Ks = torch.tensor([it["K"] for it in items]).cuda()
    ratios = torch.tensor([it["height"] / s[0] for it, s in zip(items, sizes)]).cuda()
    for i, r in enumerate(ref):
        inst = r["instances"]
        n = len(inst)
        # the oracle's boxes are post-processed to the original resolution (= the input resolution here: ratio 1)
        db[i, :n], dc[i, :n], dv[i, :n] = inst.pred_boxes.tensor, inst.pred_classes, True
    with torch.no_grad():
        c3 = pr.cube_decode(fl, db.cuda(), dc.cuda(), dv.cuda(), sizes, Ks, ratios)
    for i, r in enumerate(ref):
        inst = r["instances"]
        n = len(inst)
        sl = slice(i * D, i * D + n)
        assert _rel(c3["dims"][sl].cpu(), inst.pred_dimensions) < 3e-2
        assert _rel(c3["cam"][sl].cpu(), inst.pred_center_cam) < 3e-2
        # the pose comes from Gram-Schmidt on 6 outputs of ~1e-2 magnitude at random init: bf16 noise is amplified
        assert _rel(c3["pose"][sl].cpu(), inst.pred_pose) < 8e-2
        assert _rel(c3["corners"][sl].cpu(), inst.pred_bbox3D) < 4e-2
        assert _rel(c3["c2d"][sl].cpu(), inst.pred_center_2D) < 2e-2


def test_bn_folding_matches_unfolded_eval_and_oracle(pair):
    """SURVEY 8f-4: eval-mode BatchNorm folded into the convolution (one kernel, bias + residual + ReLU epilogue) gives the
    unfolded path's features up to bf16 rounding, and the oracle's within the frozen-BN tolerance."""
    prod, orc = pair
    from omni3d_b200 import checkpoint as ck
    from oracle import model_io
    _sync_state(prod, orc)
    saved = {k: v.clone() for k, v in orc.state_dict().items()}
    with torch.no_grad():                       # non-trivial running statistics / affine parameters
        for m in orc.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.uniform_(0.8, 1.2); m.bias.normal_(0, 0.1)
    prod.load_state_dict(orc.state_dict())
    items = synth.make_batch(2, H, W, with_gt=False, seed=13)
    prod.eval(); orc.eval()
    with torch.no_grad():
        x, _ = prod.preprocess_image(items)
        plain = prod.backbone(x)
        ck.fold_batchnorm(prod, True)
        folded = prod.backbone(x)
        ck.fold_batchnorm(prod, False)
        ref = orc.backbone(orc.preprocess_image(model_io.to_d2_inputs(items)).tensor)
    for k in ref:
        assert _rel(folded[k].float(), plain[k].float()) < 2e-2, k
        assert _rel(folded[k].float().cpu().permute(0, 3, 1, 2), ref[k]) < 3e-2, k
    orc.load_state_dict(saved)
    _sync_state(prod, orc)

"""GPU parity of the Bottleneck backbones (torchvision ResNet-50 / 101, DLA-46-C, DLA-60, DLA-102, DLA-169) on the
accelerated path against the CPU fp32 oracle (tests/bottleneck_oracle.py), with the tolerances of the DLA-34 / ResNet-34
tests (test_model_gpu.py, test_parity_r2_gpu.py); the oracle's sampling decisions are injected.  Plus, for one DLA type
with root residuals and 3-level trees (DLA-102) and for ResNet-50: graph-replayed trainer steps equal eager ones bit for
bit, and eval with BatchNorm folded into the convolutions matches unfolded eval."""
import os

import pytest
import torch

import bottleneck_oracle as bo
from omni3d_b200 import synth

pytestmark = pytest.mark.gpu

H, W = 128, 192
TYPES = list(bo.CASES)
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bottleneck_golden.pt"),
                  weights_only=False)


def _product_cfg(name, *opts):
    from omni3d_b200 import cubercnn as pc
    cfg_file, type_opts, _ = bo.CASES[name]
    return pc.load_cfg(cfg_file, ["MODEL.WEIGHTS_PRETRAIN", "none"] + list(type_opts) + list(opts))


def _pair(name):
    from omni3d_b200 import cubercnn as pc
    torch.manual_seed(0)
    orc = bo.build_model(bo.load_cfg(name))
    torch.manual_seed(0)
    prod = pc.build_model(_product_cfg(name))
    sd = orc.state_dict()
    assert set(sd) == set(prod.state_dict())
    for k, v in prod.state_dict().items():          # same-seed init is bit-identical to the oracle / reference
        assert torch.equal(v.cpu(), sd[k]), k
    return prod, orc


# Frozen BatchNorm at its initial statistics (mean 0, variance 1) leaves a random-init network unnormalised: DLA-169's
# features reach 1e13 and its depth loss 4e10, where bf16 rounding moved p2 by 3.8 % and Cube/loss_z by 5.2 %.  Statistics
# calibrated on one batch are no better (channels of near-zero variance amplify any rounding; at 2 x 640x640 DLA-169's
# BoxHead/loss_box_reg moved by 10 %), so DLA-169 is checked through its gradients only.
PARITY_TYPES = [t for t in TYPES if t != "dla169"]


@pytest.fixture(scope="module", params=PARITY_TYPES)
def rpair(request):
    prod, orc = _pair(request.param)
    yield request.param, prod, orc
    del prod, orc
    torch.cuda.empty_cache()


def _freeze_bn(m):
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eval()


def _rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))


def _sync_state(prod, orc):
    for m in orc.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.reset_running_stats()
    prod.load_state_dict(orc.state_dict())


def _calibrate_bn(prod, orc):
    """the oracle's BatchNorm running statistics set to the batch statistics of one calibration batch, then every parameter
    and buffer copied to the product"""
    from oracle import model_io
    bns = [m for m in orc.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    for m in bns:
        m.reset_running_stats()
        m.momentum = None                       # cumulative average: one batch sets the statistics to its own
    orc.train()
    with torch.no_grad():
        items = synth.make_batch(2, H, W, with_gt=False, seed=21)
        orc.backbone(orc.preprocess_image(model_io.to_d2_inputs(items)).tensor)
    for m in bns:
        m.momentum = 0.1
    prod.load_state_dict(orc.state_dict())


def _check_losses(losses, ref_losses):
    assert set(losses) == set(ref_losses)
    for k, v in ref_losses.items():
        got, ref = float(losses[k].detach()), float(v.detach())
        # the chamfer-based terms take an argmin over corner pairs on a handful of foreground RoIs: one bf16-induced flip
        # moves them by whole percents (cf. test_parity_r2_gpu.py::test_dla34_losses_640x640_vs_oracle)
        rtol = 8e-2 if k in ("Cube/loss_joint", "Cube/loss_pose") else 5e-2
        assert abs(got - ref) <= rtol * abs(ref) + 1e-5, (k, got, ref)


def test_fpn_features_frozen_bn(rpair):
    """bottom-up + FPN features with BatchNorm on running statistics vs the fp32 oracle"""
    name, prod, orc = rpair
    from oracle import model_io
    _sync_state(prod, orc)
    items = synth.make_batch(2, H, W, with_gt=False, seed=7)
    _freeze_bn(prod); _freeze_bn(orc)
    with torch.no_grad():
        x, _ = prod.preprocess_image(items)
        feats = prod.backbone(x)
        ref = orc.backbone(orc.preprocess_image(model_io.to_d2_inputs(items)).tensor)
    assert set(feats) <= set(ref)
    for k in feats:
        assert _rel(feats[k].float().cpu().permute(0, 3, 1, 2), ref[k]) < 3e-2, (name, k)


def test_train_losses_with_injected_sampling(rpair):
    """all 10 losses of a train forward vs the oracle, BatchNorm on running statistics (freeze_bn,
    cubercnn/solver/build.py:71-76): with batch statistics a randomly initialised 50-layer network amplifies the bf16
    rounding of every layer (DESIGN §6); on ResNet-50 that moved Cube/loss_pose by 11 % at this size."""
    name, prod, orc = rpair
    from oracle_capture import run_oracle_train, to_injection
    _sync_state(prod, orc)
    items = synth.make_batch(2, H, W, num_gt=4, seed=1)
    _freeze_bn(orc)
    orc_train = orc.train
    orc.train = lambda *a, **k: orc            # keep BN frozen inside run_oracle_train
    try:
        ref_losses, _, cap = run_oracle_train(orc, items)
    finally:
        orc.train = orc_train
    _freeze_bn(prod); prod.zero_grad(set_to_none=True)
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    _check_losses(losses, ref_losses)


@pytest.mark.parametrize("name", TYPES)
def test_gradients_finite_and_reach_exactly_the_used_parameters(name):
    """a train step's backward: every gradient finite, and exactly the parameters outside the reference's no-gradient set
    (tests/golden/bottleneck_golden.pt) receive one"""
    from omni3d_b200 import cubercnn as pc
    torch.manual_seed(0)
    prod = pc.build_model(_product_cfg(name)).train()
    prod.zero_grad(set_to_none=True)
    losses = prod(synth.make_batch(2, H, W, num_gt=4, seed=1))
    sum(losses.values()).backward()
    with_grad = {n for n, p in prod.named_parameters() if p.grad is not None}
    assert with_grad == {n for n, _ in prod.named_parameters()} - set(GOLD[name]["no_grad"])
    bad = [n for n, p in prod.named_parameters() if p.grad is not None and not torch.isfinite(p.grad).all()]
    assert not bad, bad


@pytest.mark.parametrize("name", ["resnet50", "dla60"])
def test_losses_640x640_vs_oracle(name):
    """2 x 640x640, the benchmark's image size: all 10 losses vs the fp32 CPU oracle, relative tolerance only.  BatchNorm on
    calibrated running statistics, as above: in train mode DLA-60's Cube/loss_pose moved by 8.7 %."""
    from oracle_capture import run_oracle_train, to_injection
    prod, orc = _pair(name)
    _calibrate_bn(prod, orc)
    items = synth.make_batch(2, 640, 640, num_gt=8, seed=5)
    _freeze_bn(orc)
    orc_train = orc.train
    orc.train = lambda *a, **k: orc
    try:
        ref_losses, _, cap = run_oracle_train(orc, items)
    finally:
        orc.train = orc_train
    _freeze_bn(prod)
    losses = prod(items, _inject=to_injection(cap, "cuda"))
    _check_losses(losses, ref_losses)
    sum(losses.values()).backward()
    assert all(torch.isfinite(p.grad).all() for p in prod.parameters() if p.grad is not None)


def _trainer_run(name, use_graph, steps=5):
    from omni3d_b200 import cubercnn as pc
    from omni3d_b200 import kernels as Kx
    from omni3d_b200.train import FlatSGDTrainer
    cfg = _product_cfg(name, "SOLVER.BASE_LR", 0.004, "SOLVER.WARMUP_ITERS", 0, "SOLVER.IMS_PER_BATCH", 2)
    torch.manual_seed(0)
    model = pc.build_model(cfg).train()
    Kx.rng_state(torch.device("cuda", torch.cuda.current_device()), seed=1234)     # same sampling stream in every run
    tr = FlatSGDTrainer(cfg, model, use_graph=use_graph)
    batches = [synth.make_batch(2, H, W, num_gt=4, seed=30 + j, image_dtype=torch.uint8) for j in range(2)]
    losses = []
    for i in range(steps):
        tr.step(batches[i % 2])
        losses.append(tr.status(wait=True)["losses"])
    assert (tr.graph is not None) == use_graph
    out = (tr.flat_p.clone(), {k: v.clone() for k, v in model.named_buffers()}, losses)
    del tr, model
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("name", ["dla102", "resnet50"])
def test_graph_replayed_steps_equal_eager_steps_bitwise(name):
    """2 eager warm-up steps, the captured step and 2 replays: parameters and BatchNorm statistics equal those of 5 eager
    steps bit for bit, and a second graph run reproduces the first one.  The logged loss values are sums of per-RoI terms
    added with atomics (head_loss_ops.cu; no gradient reads them), so they agree to fp32 rounding only."""
    p_e, b_e, l_e = _trainer_run(name, False)
    p_g, b_g, l_g = _trainer_run(name, True)
    p_g2, b_g2, l_g2 = _trainer_run(name, True)
    assert torch.equal(p_e, p_g)
    assert torch.equal(p_g, p_g2)
    for k in b_e:
        assert torch.equal(b_e[k], b_g[k]), k
        assert torch.equal(b_g[k], b_g2[k]), k
    for la, lb, lc in zip(l_e, l_g, l_g2):
        for k in la:
            assert abs(la[k] - lb[k]) <= 1e-5 * abs(la[k]) + 1e-7 and abs(lb[k] - lc[k]) <= 1e-5 * abs(lb[k]) + 1e-7, k


@pytest.mark.parametrize("name", ["dla102", "resnet50"])
def test_bn_folding_matches_unfolded_eval_and_oracle(name):
    """eval-mode BatchNorm folded into the convolution gives the unfolded path's features up to bf16 rounding, and the
    oracle's within the frozen-BN tolerance (test_model_gpu.py::test_bn_folding_matches_unfolded_eval_and_oracle)"""
    from omni3d_b200 import checkpoint as ck
    from oracle import model_io
    prod, orc = _pair(name)
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
    for k in plain:
        assert _rel(folded[k].float(), plain[k].float()) < 2e-2, k
        assert _rel(folded[k].float().cpu().permute(0, 3, 1, 2), ref[k]) < 3e-2, k

"""Gradient chaining (omni3d_b200.nnfunc.fork): consumers of a multiply-used activation add their gradient
contributions into ONE buffer inside the producing kernels instead of autograd running an add pass per consumer.
The sums are the same; only the rounding differs (fp32 add before the single bf16 rounding instead of a bf16
round per partial sum) — parameter gradients with and without chaining must agree to bf16 accuracy."""
import pytest
import torch

from omni3d_b200 import nnfunc, synth

pytestmark = pytest.mark.gpu


def _grads(name, chain, frozen_bn):
    from omni3d_b200 import cubercnn as pc
    nnfunc.GRAD_CHAIN = chain
    try:
        torch.manual_seed(0)
        cfg = pc.load_cfg(name, ["MODEL.WEIGHTS_PRETRAIN", "none"])
        model = pc.build_model(cfg)
        model.train()
        if frozen_bn:
            for m in model.modules():
                if isinstance(m, torch.nn.BatchNorm2d):
                    m.eval()
        items = synth.make_batch(2, 128, 192, with_gt=False, seed=3)
        x, _ = model.preprocess_image(items)
        feats = model.backbone(x)
        g = torch.Generator(device="cuda").manual_seed(5)
        loss = 0.0
        for k in sorted(feats):
            w = torch.randn(feats[k].shape, device="cuda", generator=g)
            loss = loss + (feats[k].float() * w).sum()
        loss.backward()
        return {n: p.grad.detach().clone() for n, p in model.backbone.named_parameters() if p.grad is not None}
    finally:
        nnfunc.GRAD_CHAIN = True


@pytest.mark.parametrize("name", ["cubercnn_DLA34_FPN.yaml", "cubercnn_ResNet34_FPN.yaml"])
def test_chained_gradients_equal_autograd_sums(name):
    # frozen BatchNorm: no batch-statistics amplification, the comparison isolates the gradient sums themselves
    ref = _grads(name, False, True)
    got = _grads(name, True, True)
    assert ref.keys() == got.keys() and len(ref) > 100
    rels = []
    for k in ref:
        r, g = ref[k].float(), got[k].float()
        assert torch.isfinite(g).all(), k
        rel = float((g - r).norm() / (r.norm() + 1e-20))
        rels.append(rel)
        # bf16 rounding of the partial sums (eps 2^-8) propagated through <= 40 layers; a dropped or doubled contribution
        # would show up as an O(1) error.
        assert rel < 5e-2, (k, rel)
    rels.sort()
    assert rels[len(rels) // 2] < 2e-2, rels[len(rels) // 2]


def test_chaining_removes_the_add_passes():
    """with chaining the backbone's backward issues no ATen add kernels for activation gradients"""
    from omni3d_b200 import cubercnn as pc
    from torch.profiler import profile, ProfilerActivity
    counts = {}
    for chain in (False, True):
        nnfunc.GRAD_CHAIN = chain
        try:
            torch.manual_seed(0)
            model = pc.build_model(pc.load_cfg("cubercnn_DLA34_FPN.yaml", ["MODEL.WEIGHTS_PRETRAIN", "none"]))
            model.train()
            items = synth.make_batch(2, 128, 192, with_gt=False, seed=3)
            x, _ = model.preprocess_image(items)
            feats = model.backbone(x)
            loss = sum(f.float().sum() for f in feats.values())
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                loss.backward()
                torch.cuda.synchronize()
            counts[chain] = sum(e.count for e in prof.key_averages() if "CUDAFunctor_add" in e.key)
        finally:
            nnfunc.GRAD_CHAIN = True
    assert counts[True] <= counts[False] - 20, counts


# ---- the accumulating kernel variants behind the protocol, one by one ------------------------------------------------
def _r(*shape, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g)


def test_bn_bwd_accumulating_dres_dense_and_slice():
    """c3d_bn_bwd flag bit 1: dres += masked dout (fp32 add) into a dense buffer and into a channel slice of a wider one"""
    from omni3d_b200 import kernels as Kx
    P, C = 4096, 64
    y = _r(2, 32, 64, C, seed=1).bfloat16()
    res = _r(2, 32, 64, C, seed=7).bfloat16()
    mean, rstd = _r(C, seed=2) * 0.1, torch.rand(C, device="cuda") + 0.5
    gamma, beta = torch.rand(C, device="cuda") + 0.5, _r(C, seed=3) * 0.3
    out = Kx.bn_apply(y, mean, rstd, gamma, beta, res, True)
    dout = _r(2, 32, 64, C, seed=4).bfloat16()
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    dy0, dres0 = Kx.bn_bwd(dout, out, y, mean, rstd, gamma, True, dg, db, True)
    prior = _r(2, 32, 64, C, seed=9).bfloat16()
    want = (prior.float() + dres0.float()).bfloat16()
    for wide in (False, True):
        if wide:
            buf = torch.zeros(2, 32, 64, 3 * C, device="cuda", dtype=torch.bfloat16)
            into = buf[..., C:2 * C]
            into.copy_(prior)
        else:
            into = prior.clone()
        dg2, db2 = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        dy1, _ = Kx.bn_bwd(dout, out, y, mean, rstd, gamma, True, dg2, db2, True, dres_into=into)
        assert torch.equal(dy1, dy0) and torch.equal(dg2, dg) and torch.equal(db2, db)
        assert torch.equal(into, want)
        if wide:
            assert float(buf[..., :C].abs().max()) == 0.0 and float(buf[..., 2 * C:].abs().max()) == 0.0


def test_maxpool2_bwd_accumulate():
    from omni3d_b200 import kernels as Kx
    x = _r(2, 16, 24, 32, seed=1).bfloat16()
    dy = _r(2, 8, 12, 32, seed=2).bfloat16()
    dx = Kx.maxpool2_bwd(x, dy)
    prior = _r(2, 16, 24, 32, seed=3).bfloat16()
    into = prior.clone()
    Kx.maxpool2_bwd(x, dy, into=into)
    assert torch.equal(into, (prior.float() + dx.float()).bfloat16())


@pytest.mark.parametrize("Cin,Cout,k,stride", [(64, 64, 3, 1), (128, 128, 3, 1), (256, 256, 3, 1), (64, 128, 3, 2), (16, 32, 3, 2),
                                               (256, 128, 1, 1)])
def test_conv_dgrad_accumulates_into_existing_gradient(Cin, Cout, k, stride):
    """_dgrad(..., into=buf): buf += dgrad in the conv epilogue (add_mode 3) on every kernel variant — the GEMM kernel
    at several tile widths, the merged stride-2 form with split channel placement — for a dense buffer and a channel slice."""
    from omni3d_b200 import nnfunc
    N, H, W = 2, 32, 48
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    w = torch.nn.Parameter(_r(Cout, Cin, k, k, seed=1) / (k * k * Cin) ** 0.5)
    dy = _r(N, Ho, Wo, Cout, seed=2).bfloat16()
    ref = nnfunc._dgrad(dy, w, stride, pad, (H, W)).float()
    prior = _r(N, H, W, Cin, seed=3).bfloat16()
    for wide in (False, True):
        if wide:
            buf = torch.zeros(N, H, W, Cin + 32, device="cuda", dtype=torch.bfloat16)
            into = buf[..., 16:16 + Cin]
            into.copy_(prior)
        else:
            into = prior.clone()
        nnfunc._dgrad(dy, w, stride, pad, (H, W), into=into)
        got, want = into.float(), prior.float() + ref
        # `ref` was rounded to bf16 once before the add, the fused path adds in fp32: one bf16 ulp of the sum
        assert float((got - want).abs().max()) <= 2.0 ** -7 * float(want.abs().max()) + 1e-3
        if wide:
            assert float(buf[..., :16].abs().max()) == 0.0 and float(buf[..., 16 + Cin:].abs().max()) == 0.0

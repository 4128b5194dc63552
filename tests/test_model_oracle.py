"""CPU tests: pin oracle/cubercnn_oracle against the fixture produced by running the reference's own
cubercnn code (tests/golden/make_model_golden.py): same-seed init, losses, logged scalars, gradient
norms, unused parameters and inference detections."""
import os

import pytest
import torch

from omni3d_b200 import synth
from oracle import cubercnn_oracle as co
from oracle import model_io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests/golden/model_golden.pt"), weights_only=False)
CASES = {"dla34": ("cubercnn_DLA34_FPN.yaml", (128, 160)), "resnet34": ("cubercnn_ResNet34_FPN.yaml", (128, 128))}


@pytest.mark.parametrize("name", ["dla34", "resnet34"])
def test_oracle_matches_reference_run(name):
    from detectron2.utils.events import EventStorage
    cfg_file, (H, W) = CASES[name]
    g = GOLD[name]
    cfg = co.load_cfg(cfg_file)
    torch.manual_seed(0)
    model = co.build_model(cfg)
    sd = model.state_dict()
    assert set(sd) == set(g["init_sum"]), "state_dict key names differ from the reference"
    assert sum(p.numel() for p in model.parameters()) == g["n_params"]
    for k, v in sd.items():   # same-seed init is bit-identical; only the float64 reduction order of the checksum may
        # differ between CPUs (vector width), by far less than one changed float32 element would move it
        assert float(v.double().sum()) == pytest.approx(g["init_sum"][k], rel=1e-13, abs=1e-15), k
        assert float(v.double().abs().sum()) == pytest.approx(g["init_abs"][k], rel=1e-13, abs=1e-15), k
    model.train()
    torch.manual_seed(123)
    with EventStorage(0) as st:
        losses = model(model_io.to_d2_inputs(synth.make_batch(2, H, W, num_gt=4, seed=1)))
        sum(losses.values()).backward()
        scalars = st.latest()
    # the fixture was recorded on one CPU; another vector width rounds the fp32 reductions differently in the last bits
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


@pytest.mark.parametrize("src", ["repo", "reference"])
def test_config_surface(src):
    """the flattened repo configs and the reference's own YAML chain load to the same values (the reference chain as
    stored in tests/golden/reference_cfg_DLA34_FPN.yaml: the CfgNode.dump() of its configs/cubercnn_DLA34_FPN.yaml
    loaded through the oracle's config system)"""
    path = "cubercnn_DLA34_FPN.yaml"
    if src == "reference":
        path = os.path.join(ROOT, "tests/golden/reference_cfg_DLA34_FPN.yaml")
    cfg = co.load_cfg(path)
    assert cfg.MODEL.META_ARCHITECTURE == "RCNN3D" and cfg.MODEL.ROI_HEADS.NUM_CLASSES == 50
    assert cfg.MODEL.BACKBONE.NAME == "build_dla_from_vision_fpn_backbone"
    assert cfg.MODEL.RPN.IOU_THRESHOLDS == [0.05, 0.05] and cfg.MODEL.ROI_CUBE_HEAD.VIRTUAL_FOCAL == 512.0
    assert cfg.SOLVER.IMS_PER_BATCH == 192 and cfg.SOLVER.STEPS == (69600, 92800)

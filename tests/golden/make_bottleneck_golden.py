"""Generates tests/golden/bottleneck_golden.pt by running the REFERENCE'S OWN cubercnn modeling code
(/root/reference, unmodified) on oracle/d2lite (see oracle/ref_runner.py) on seeded synthetic inputs, for the
Bottleneck backbones: torchvision ResNet-50 / 101 and DLA-46-C, DLA-60, DLA-102, DLA-169.

Same recipe and record as make_model_golden.py.  Pins tests/bottleneck_oracle.py (tests/test_bottleneck_cpu.py) and,
through it, the CUDA path.
Run here only:   python tests/golden/make_bottleneck_golden.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import model_io, ref_runner  # noqa: E402
from omni3d_b200 import synth  # noqa: E402

# name -> (reference config, overrides, (H, W)); the same table as tests/bottleneck_oracle.py:CASES
CASES = {
    "resnet50": ("configs/cubercnn_ResNet34_FPN.yaml", ["MODEL.RESNETS.DEPTH", 50], (128, 128)),
    "resnet101": ("configs/cubercnn_ResNet34_FPN.yaml", ["MODEL.RESNETS.DEPTH", 101], (128, 128)),
    "dla46_c": ("configs/cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla46_c"], (128, 160)),
    "dla60": ("configs/cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla60"], (128, 160)),
    "dla102": ("configs/cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla102"], (128, 160)),
    "dla169": ("configs/cubercnn_DLA34_FPN.yaml", ["MODEL.DLA.TYPE", "dla169"], (128, 160)),
}


def main():
    out = {}
    for name, (cfg_file, opts, (H, W)) in CASES.items():
        cfg = ref_runner.reference_cfg(cfg_file, opts)
        torch.manual_seed(0)
        model = ref_runner.build_reference_model(cfg)
        from detectron2.utils.events import EventStorage
        sd = model.state_dict()
        rec = {"init_sum": {k: float(v.double().sum()) for k, v in sd.items()},
               "init_abs": {k: float(v.double().abs().sum()) for k, v in sd.items()},
               "n_params": sum(p.numel() for p in model.parameters())}
        model.train()
        items = synth.make_batch(2, H, W, num_gt=4, seed=1)
        torch.manual_seed(123)
        with EventStorage(0) as st:
            losses = model(model_io.to_d2_inputs(items))
            sum(losses.values()).backward()
            rec["scalars"] = st.latest()
        rec["losses"] = {k: v.detach().clone() for k, v in losses.items()}
        rec["grad_norm"] = {n: float(p.grad.double().norm()) for n, p in model.named_parameters() if p.grad is not None}
        rec["no_grad"] = sorted(n for n, p in model.named_parameters() if p.grad is None)
        model.eval()
        with torch.no_grad():
            res = model(model_io.to_d2_inputs(synth.make_batch(2, H, W, with_gt=False, seed=3)))
        rec["detections"] = [{k: (v.tensor if hasattr(v, "tensor") else v).clone()
                              for k, v in r["instances"].get_fields().items()} for r in res]
        out[name] = rec
        print(name, rec["n_params"], len(rec["no_grad"]), {k: round(float(v), 6) for k, v in rec["losses"].items()},
              [len(d["scores"]) for d in rec["detections"]])
    torch.save(out, os.path.join(ROOT, "tests/golden/bottleneck_golden.pt"))
    print("wrote tests/golden/bottleneck_golden.pt")


if __name__ == "__main__":
    main()

"""Writes tests/golden/reference_cfg_DLA34_FPN.yaml: the reference's own configs/cubercnn_DLA34_FPN.yaml (with its _BASE_
chain) loaded through the oracle's config system and dumped with CfgNode.dump().  tests/test_model_oracle.py checks the
repo's flattened config against it.

Run only where the reference checkout is available:   python tests/golden/make_config_golden.py REFERENCE_ROOT"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import cubercnn_oracle as co  # noqa: E402


def main(ref_root):
    cfg = co.load_cfg(os.path.join(os.path.abspath(ref_root), "configs", "cubercnn_DLA34_FPN.yaml"))
    out = os.path.join(ROOT, "tests", "golden", "reference_cfg_DLA34_FPN.yaml")
    with open(out, "w") as f:
        f.write(cfg.dump())
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1])

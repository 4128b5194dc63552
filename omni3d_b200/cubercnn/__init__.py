"""Host-side mirror of the reference's `cubercnn` interface for the accelerated path.

Same registry names / config keys / state_dict names / call signatures as
cubercnn/modeling/{meta_arch,backbone,proposal_generator,roi_heads} (SURVEY.md section 8b), with the
arithmetic running on libc3d.so (sm_90a kernels) — see DESIGN.md for the boundary.
"""
from .config import CfgNode, get_cfg, get_cfg_defaults, load_cfg  # noqa: F401
from .registry import (BACKBONE_REGISTRY, META_ARCH_REGISTRY, PROPOSAL_GENERATOR_REGISTRY,  # noqa: F401
                       ROI_CUBE_HEAD_REGISTRY, ROI_HEADS_REGISTRY)
from .structures import Boxes, Instances  # noqa: F401
from .model import RCNN3D, build_model  # noqa: F401

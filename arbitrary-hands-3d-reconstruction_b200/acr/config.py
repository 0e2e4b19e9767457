"""Configuration shim compatible with the reference's ``acr.config`` (acr/config.py:19-270).

The reference parses ``sys.argv`` and ``configs/demo.yml`` *at import time* into a class-level
singleton read everywhere through ``args()`` (:225-270).  Here ``args()`` returns the same kind
of namespace with the hot-path-relevant defaults (values and source lines below), nothing is
parsed at import, and ``parse_args(list)`` / ``ConfigContext`` accept overrides explicitly.
"""
from __future__ import annotations

import argparse
import os
from typing import Optional, Sequence

project_dir = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

_DEFAULTS = dict(
    tab="ACR_hrnet_internet", backbone="hrnet",          # config.py:95 ("resnet50 or hrnet"; only a log tag there, SURVEY F1):
                                                          # values starting with "resnet" select the ResNet-50 trunk
                                                          # (backbone_kind), every other value the HRNet trunk
    model_precision="bf16",                               # reference: fp32|fp16 (config.py:96); here bf16|fp16 = tensor-core
                                                          # plans, fp32 = the (slow, reference-accurate) validation plan,
                                                          # tf32 = fp32 storage with tf32 tensor-core convs (what the
                                                          # reference's fp32 runs as on Ampere / Hopper with cuDNN's TF32)
    hrnet_width=32,                                        # 32 = the reference's HRNet-W32 (the only trunk it contains); 48 = the
                                                          # HRNet-W48 trunk of BASELINE configs[4] (no reference: parity unpinned)
    input_size=512,                                        # config.py:61
    centermap_size=64, centermap_conf_thresh=0.35,         # config.py:130-131
    kernel_sizes=[5], max_hand=4,                          # config.py:185,161 (max_hand is the reference's training-time
                                                          # value; it does not switch multi-hand parsing on)
    max_hands_per_side=1,                                  # hands kept per image and side, 1..16; 1 = the reference's
                                                          # inference parse, > 1 = multi-hand parsing (DESIGN.md)
    Rot_type="6D", rot_dim=6, cam_dim=3, align_idx=9,      # config.py:167-170
    mano_theta_num=16, head_block_num=2,                   # config.py:172,98
    inter_prior=True, prior_mode="cross",                  # config.py:88-89
    offset_mode="concat", attention_mode="pred-part",      # config.py:84-85
    merge_mano_camera_head=False, dataset="internet",      # config.py:159
    perspective_proj=False, model_version=1,               # config.py:47-48
    focal_length=1265.0, FOV=22.5,                         # configs/demo.yml:13-14
    mano_mesh_root_align=True,                             # configs/demo.yml:11
    val_batch_size=1, GPUS="0",                            # configs/demo.yml:3,8
    temporal_optimization=False, smooth_coeff=4.0,         # config.py:29-30
    track_hands=False, track_gate=8, track_max_missed=15,  # multi-hand tracking in process_results (DESIGN.md): track ids,
                                                          # and with temporal_optimization one filter bank per track;
                                                          # gate in centre-map cells, max_missed in frames
    track_streams=1,                                       # streams one batch may hold (batch_forward's stream_ids)
    model_path=os.path.join(project_dir, "checkpoints", "wild.pkl"),
    mano_root=os.path.join(project_dir, "mano"),           # acr/mano_wrapper.py:22 uses 'mano/'
    cam_trans_mode="lstsq",                                # 'lstsq' (device least squares, SURVEY 8f-1) | 'pnp' (device
                                                          # RANSAC-EPnP, the reference's cv2.solvePnPRansac) | 'none'
    return_maps=True,                                      # materialise NCHW fp32 maps lazily on access
    return_part_labels=False,                              # outputs['part_labels']: per-image uint8 part labels at the
                                                          # frame's resolution (acr_b200.ops.part_labels, DESIGN.md)
    demo_mode="image", inputs=None, output_dir=None, save_dict_results=False,
)


def parse_args(input_args: Optional[Sequence[str]] = None) -> argparse.Namespace:
    """Subset of the reference's flags that matter on the hot path; unknown flags are ignored."""
    p = argparse.ArgumentParser(description="ACR hot path (H100)")
    for k, v in _DEFAULTS.items():
        if isinstance(v, bool):
            p.add_argument(f"--{k}", type=lambda s: str(s).lower() == "true", default=v)
        elif isinstance(v, list) or v is None:
            p.add_argument(f"--{k}", default=v)
        else:
            p.add_argument(f"--{k}", type=type(v), default=v)
    ns, _ = p.parse_known_args(list(input_args) if input_args is not None else [])
    return ns


class ConfigContext(object):
    """Same role as the reference's ConfigContext (:225-267) minus the yaml dump side effects."""
    parsed_args = parse_args([])

    def __init__(self, parsed_args=None):
        if parsed_args is not None:
            ConfigContext.parsed_args = parsed_args

    def __enter__(self):
        return ConfigContext.parsed_args

    def __exit__(self, exc_type, exc, tb):
        return False


def args() -> argparse.Namespace:
    return ConfigContext.parsed_args


def backbone_kind(ns: Optional[argparse.Namespace] = None) -> str:
    """The trunk a configuration selects: "resnet50" for ``backbone`` values starting with "resnet" (the reference
    documents "resnet50 or hrnet", configs/demo.yml carries 'resnet'), "hrnet" for every other value."""
    ns = ns if ns is not None else args()
    return "resnet50" if str(getattr(ns, "backbone", "hrnet")).lower().startswith("resnet") else "hrnet"

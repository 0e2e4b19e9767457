"""Seeded synthetic assets: network weights and MANO hand models.

The reference ships neither its checkpoint (``checkpoints/wild.pkl``) nor the
licence-gated ``MANO_LEFT/RIGHT.pkl`` (/root/reference/README.md:40-41), so
parity tests and the benchmark use seeded synthetic tensors with the
reference's exact shapes and state-dict keys (SURVEY.md F4, section 8c-4/6).
Everything here is generated with explicit ``torch.Generator`` / ``numpy``
generators on the CPU, so the same seed gives bit-identical assets in this
container and on the GPU box.
"""
from __future__ import annotations

import math
import os
from collections import OrderedDict
from typing import Dict, Optional

import numpy as np
import torch

from .netspec import NetSpec, build_acr_spec

# MANO kinematic tree (kintree_table[0]); mano/manolayer.py:100-102 reads it, the
# forward pass hard-codes the three finger levels (mano/manolayer.py:191-193).
MANO_PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 0, 10, 11, 0, 13, 14]


def synth_state_dict(seed: int = 0, spec: Optional[NetSpec] = None,
                     bn_stats: Optional[Dict[str, np.ndarray]] = None,
                     center_bias: float = 1.0) -> "OrderedDict[str, torch.Tensor]":
    """Random-init weights with the reference's 2067 state-dict keys (or those of ``spec``: any trunk).

    * conv / linear weights: N(0, gain^2 * 2/fan_in); the last BN of each residual
      block and the fuse-layer BNs get a small gamma so activations stay O(1)
      through ~40 residual blocks.
    * BN gamma/beta random, running stats either from ``bn_stats`` (calibrated by
      ``tests/golden/make_golden.py`` with the reference in train mode) or (0, 1).
    * centre-head biases are pushed to ``center_bias`` so both hands clear the 0.35
      detection threshold (/root/reference/acr/result_parser.py:203,240).
    """
    spec = spec or build_acr_spec()
    g = torch.Generator().manual_seed(seed)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for key, (shape, kind) in spec.params.items():
        if kind == "conv_w":
            fan_in = shape[1] * shape[2] * shape[3]
            w = torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in)
        elif kind == "deconv_w":   # ConvTranspose2d (cin, cout, 4, 4), k4 s2: every output pixel sees cin x 2 x 2 live taps
            w = torch.randn(shape, generator=g) * math.sqrt(2.0 / (shape[0] * 4))
        elif kind == "lin_w":
            w = torch.randn(shape, generator=g) * math.sqrt(1.0 / shape[1])
        elif kind == "lc_w":
            w = torch.randn(shape, generator=g) * math.sqrt(1.0 / shape[2])
        elif kind in ("conv_b", "lin_b"):
            w = torch.randn(shape, generator=g) * 0.05
        elif kind == "bn_w":
            small = key.endswith(("bn2.weight", "bn3.weight")) and "backbone.bn2" not in key
            small = small or ".fuse_layers." in key or ".downsample." in key
            lo, hi = (0.2, 0.5) if small else (0.6, 1.4)
            w = torch.rand(shape, generator=g) * (hi - lo) + lo
        elif kind == "bn_b":
            w = torch.randn(shape, generator=g) * 0.1
        elif kind == "bn_mean":
            w = torch.zeros(shape)
        elif kind == "bn_var":
            w = torch.ones(shape)
        elif kind == "bn_nbt":
            w = torch.zeros(shape, dtype=torch.long)
        else:
            raise KeyError(kind)
        sd[key] = w
    if bn_stats is not None:
        for k, v in bn_stats.items():
            assert k in sd and tuple(v.shape) == tuple(sd[k].shape), k
            sd[k] = torch.from_numpy(np.asarray(v)).to(sd[k].dtype).clone()
    for side in ("l", "r"):
        sd[f"{side}_final_layers.2.2.bias"].fill_(center_bias)
        # keep the heads' outputs in a sane range (params ~ O(1))
        for idx in (1, 3, 4):
            sd[f"{side}_final_layers.{idx}.2.weight"].mul_(0.5)
    return sd


def load_bn_calibration(seed: int = 0) -> Optional[Dict[str, np.ndarray]]:
    """BN running statistics measured once with the reference (tests/golden)."""
    here = os.path.dirname(os.path.abspath(__file__))
    path = os.path.join(here, "..", "..", "tests", "golden", f"bn_calib_seed{seed}.npz")
    if not os.path.exists(path):
        return None
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def make_synthetic_mano(side: str = "right", seed: Optional[int] = None) -> Dict[str, np.ndarray]:
    """A MANO-shaped hand model with seeded contents.

    Keys / shapes follow what ``ready_arguments`` returns for the real pickle
    (/root/reference/mano/manolayer.py:350-394, shapes verified in SURVEY.md 8b):
    hands_components (45,45), hands_mean (45,), betas (10,), shapedirs (778,3,10),
    posedirs (778,3,135), v_template (778,3), J_regressor (16,778) dense here,
    weights (778,16) row-stochastic, f (1538,3), kintree_table (2,16).
    Magnitudes mimic the real model: a ~0.2 m hand, mm-scale blend shapes.
    """
    if seed is None:
        seed = 0 if side == "right" else 1
    rng = np.random.default_rng(1000 + seed)
    nv = 778
    # template: an elongated blob around the origin
    v_template = (rng.standard_normal((nv, 3)) * np.array([0.04, 0.02, 0.01])).astype(np.float32)
    shapedirs = (rng.standard_normal((nv, 3, 10)) * 0.004).astype(np.float32)
    posedirs = (rng.standard_normal((nv, 3, 135)) * 0.0015).astype(np.float32)
    # joint regressor: each joint a convex combination of ~12 vertices
    J = np.zeros((16, nv), np.float32)
    for j in range(16):
        idx = rng.choice(nv, 12, replace=False)
        w = rng.random(12).astype(np.float32)
        J[j, idx] = w / w.sum()
    # skinning weights: <=4 bones per vertex, rows sum to 1
    W = np.zeros((nv, 16), np.float32)
    for v in range(nv):
        idx = rng.choice(16, 4, replace=False)
        w = rng.random(4).astype(np.float32) ** 2
        W[v, idx] = w / w.sum()
    faces = rng.integers(0, nv, (1538, 3)).astype(np.int64)
    kintree = np.stack([np.array(MANO_PARENTS, np.int64), np.arange(16, dtype=np.int64)])
    kintree[0, 0] = 4294967295  # the real pickle stores uint32(-1) for the root
    comps = rng.standard_normal((45, 45)).astype(np.float32) * 0.3
    mean = (rng.standard_normal(45) * 0.25).astype(np.float32)
    return dict(hands_components=comps, hands_mean=mean, betas=np.zeros(10, np.float32),
                shapedirs=shapedirs, posedirs=posedirs, v_template=v_template,
                J_regressor=J, weights=W, f=faces, kintree_table=kintree, side=side)

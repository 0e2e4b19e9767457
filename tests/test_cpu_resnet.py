"""CPU: the ResNet-50 trunk's spec, parameter registry, FLOP count, weight packing, records and kernel instances (no GPU)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as Fn

from acr_b200 import lib as L
from acr_b200.netspec import build_acr_spec, conv_flops_per_image, op_flops
from tests import resnet_ref

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _trunk_key(k):
    return k.startswith("backbone.") and not k.startswith("backbone.hand_segm.")


@pytest.fixture(scope="module")
def spec():
    return build_acr_spec(512, backbone="resnet50")


def test_spec_keys_load_strictly_into_the_oracle_trunk(spec):
    """The registry's trunk keys and shapes are exactly those of an nn.Module ResNet-50 + deconv trunk, in its order."""
    from acr_b200.synth import synth_state_dict
    sd = synth_state_dict(0, spec=spec)
    trunk = resnet_ref.ResNet50Trunk()
    trunk.load_state_dict(resnet_ref.trunk_state(sd), strict=True)
    assert list(resnet_ref.trunk_state(sd)) == list(trunk.state_dict())
    assert spec.params["backbone.conv1.weight"][0] == (64, 3, 7, 7)
    assert spec.params["backbone.deconv_layers.0.weight"][0] == (2048, 256, 4, 4)
    assert spec.params["backbone.layer4.0.downsample.0.weight"][0] == (2048, 1024, 1, 1)


def test_non_trunk_keys_equal_the_w32_model(spec):
    """Heads, SegmNet, part branch and the dead-but-present parameters: the W32 model's names, shapes and order."""
    w32 = build_acr_spec(512)
    a = [(k, v) for k, v in spec.params.items() if not _trunk_key(k)]
    b = [(k, v) for k, v in w32.params.items() if not _trunk_key(k)]
    assert a == b and len(a) > 100


def test_conv_flops_equal_a_hook_count_on_the_oracle(spec):
    """conv_flops_per_image: the trunk part equals a forward-hook count on the oracle modules (deconvs by live taps:
    2x2 of the 16 per output pixel), the rest equals the W32 model's heads."""
    trunk = resnet_ref.ResNet50Trunk().to("meta")
    total = [0.0]

    def hook(m, inp, out):
        x = inp[0]
        if isinstance(m, nn.ConvTranspose2d):
            total[0] += 2.0 * out[0].numel() * x.shape[1] * 4
        else:
            total[0] += 2.0 * out[0].numel() * x.shape[1] * m.kernel_size[0] * m.kernel_size[1] // m.groups
    for m in trunk.modules():
        if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            m.register_forward_hook(hook)
    out = trunk(torch.zeros(1, 512, 512, 3, device="meta"))
    assert tuple(out.shape) == (1, 32, 128, 128)
    cut = lambda s: next(i for i, op in enumerate(s.ops) if op.kind == "coordcat")
    trunk_fl = sum(op_flops(op) for op in spec.ops[:cut(spec)])
    assert trunk_fl == total[0]
    w32 = build_acr_spec(512)
    heads = conv_flops_per_image(w32) - sum(op_flops(op) for op in w32.ops[:cut(w32)])
    assert conv_flops_per_image(spec) == pytest.approx(trunk_fl + heads, rel=1e-12)
    assert 68e9 < conv_flops_per_image(spec) < 70e9


def test_deconv_packing_puts_each_weight_at_its_parity_and_tap():
    """engine.deconv_parity_weights: the four 2x2 convs (parity p = py*2+px, tap (ty,tx) reading input offset
    (py+ty-1, px+tx-1)) that the transposed-conv kernel multiplies ARE ConvTranspose2d(k4, s2, p1)."""
    from acr_b200.engine import deconv_parity_weights
    g = torch.Generator().manual_seed(0)
    cin, cout, H = 5, 3, 6
    w = torch.randn(cin, cout, 4, 4, generator=g)
    x = torch.randn(1, cin, H, H, generator=g)
    par = torch.from_numpy(deconv_parity_weights(w.numpy()))
    assert tuple(par.shape) == (4, cout, cin, 2, 2)
    xp = Fn.pad(x, (1, 1, 1, 1))
    y = torch.zeros(1, cout, 2 * H, 2 * H)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    # input offset (py+ty-1, px+tx-1) = padded window start (py+ty, px+tx)
                    win = xp[:, :, py + ty: py + ty + H, px + tx: px + tx + H]
                    y[:, :, py::2, px::2] += torch.einsum("bchw,oc->bohw", win, par[py * 2 + px, :, :, ty, tx])
    exp = Fn.conv_transpose2d(x, w, None, 2, 1)
    assert torch.allclose(y, exp, atol=1e-5, rtol=1e-5)
    # and one weight element by hand: w[ci, co, ky, kx] with ky = 3 - py - 2 ty
    assert par[1 * 2 + 0, 2, 4, 0, 1] == w[4, 2, 2, 1]


def test_records_and_1x1_stride2_packing():
    """Engine(dry_run=True, backbone='resnet50'): 7x7 stem, one max-pool, 52 trunk convs incl. four downsamples (three
    of them 1x1 stride 2), three transposed convs (the last one writing the coord-concat buffer), then the W32 heads; the 1x1
    stride-2 weights pack as [cout_pad][1][cin_pad]."""
    from acr_b200.engine import Engine
    eng = Engine(None, 2, "cpu", torch.bfloat16, dry_run=True, backbone="resnet50")
    kinds = [r["kind"] for r in eng.recs]
    assert kinds[:2] == [L.OP_STEM_TC, L.OP_MAXPOOL] and kinds.count(L.OP_MAXPOOL) == 1
    cut = kinds.index(L.OP_COORD)
    trunk = eng.recs[2:cut]
    dec = [r for r in trunk if r.get("attrs", {}).get("deconv")]
    s2_1x1 = [r for r in trunk if r["attrs"]["k"] == 1 and r["attrs"]["s"] == 2]
    assert len(trunk) == 55 and len(dec) == 3 and len(s2_1x1) == 3
    assert [r["attrs"]["w"] for r in s2_1x1] == [f"backbone.layer{i}.0.downsample.0" for i in (2, 3, 4)]
    assert dec[-1]["out"].name == "feat32" and dec[-1]["out"].base.C == 34
    w32 = Engine(None, 2, "cpu", torch.bfloat16, dry_run=True)
    assert [r["kind"] for r in eng.recs[cut:]] == [r["kind"] for r in w32.recs[[r["kind"] for r in w32.recs].index(L.OP_COORD):]]
    from tests.helpers import pack_conv_host
    w = np.random.default_rng(0).standard_normal((48, 40, 1, 1)).astype(np.float32)
    wp, _ = pack_conv_host(w, None, None, 48, 48, L.DT_BF16)
    got = torch.from_numpy(wp.view(np.int16).copy()).view(torch.bfloat16).float()
    assert tuple(wp.shape) == (48, 1, 48)
    assert torch.equal(got[:, 0, :40], torch.from_numpy(w[:, :, 0, 0]).to(torch.bfloat16).float())
    assert float(got[:, 0, 40:].abs().max()) == 0.0


@pytest.mark.parametrize("kw", [dict(act_dtype=torch.float32), dict(act_dtype=torch.bfloat16, debug_ref_conv=True)])
def test_fp32_and_debug_ref_conv_raise(kw):
    from acr_b200.engine import Engine
    with pytest.raises(L.AcrB200Error, match="tensor cores only"):
        Engine(None, 1, "cpu", dry_run=True, backbone="resnet50", **kw)


def test_input_size_must_be_a_multiple_of_512():
    with pytest.raises(ValueError, match="multiple of 512"):
        build_acr_spec(384, backbone="resnet50")
    assert build_acr_spec(1024, backbone="resnet50").tensors["feat32"].H == 256


def test_config_shim_maps_backbone_values():
    from acr.config import backbone_kind, parse_args
    for v, want in [("resnet", "resnet50"), ("resnet50", "resnet50"), ("ResNet", "resnet50"), ("hrnet", "hrnet"),
                    ("hrnetv4", "hrnet"), ("anything", "hrnet")]:
        assert backbone_kind(parse_args(["--backbone", v])) == want, v
    assert backbone_kind(parse_args([])) == "hrnet"


def test_model_registers_resnet_keys_and_round_trips(spec):
    """acr.model.ACR with backbone='resnet': the state dict has the spec's keys and shapes, the trunk in construction
    order, and a strict load_state_dict of it round-trips."""
    from acr.config import args
    from acr.model import ACR
    old = args().backbone
    args().backbone = "resnet"
    try:
        m = ACR()
    finally:
        args().backbone = old
    sd = m.state_dict()
    assert set(sd) == set(spec.params)
    assert [k for k in sd if _trunk_key(k)] == [k for k in spec.params if _trunk_key(k)]
    assert all(tuple(sd[k].shape) == spec.params[k][0] for k in sd)
    m.load_state_dict({k: v.clone() for k, v in sd.items()}, strict=True)


def test_new_kernel_instances_pass_the_sass_checks():
    """The transposed-conv conv_tc instances and the 7x7 stem: no local memory, and the wgmma + TMA + mbarrier
    pipeline (the stem builds its operand itself: no TMA loads) with the producer / consumer register split."""
    lib = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
    if not (os.path.exists(lib) and os.path.exists("/usr/local/cuda/bin/cuobjdump")):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(lib)
    finally:
        sys.path.pop(0)
    deconv = {n: r for n, r in rows.items() if n.startswith("conv_tc_kernel<64,") and n.split(",")[2].strip() == "64"}
    stem7 = {n: r for n, r in rows.items() if n.startswith("stem_tc_kernel<") and n.endswith(", 7>")}
    pool = {n: r for n, r in rows.items() if n.startswith("maxpool3s2_kernel<")}
    assert len(deconv) == 4 and len(stem7) == 2 and len(pool) == 2
    for n, r in {**deconv, **stem7, **pool}.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
    for n, r in {**deconv, **stem7}.items():
        assert r["HGMMA"] > 0 and r["SYNCS"] > 0, n
    for n, r in deconv.items():
        assert r["UTMALDG"] > 0 and r["USETMAXREG"] == 2, n

"""GPU: the fused Bottleneck launch (csrc/conv_bottleneck.cuh) is bit-identical to the block's three conv launches
(ACR_B200_FUSE_BLOCKS=0): block 0 (64-channel input, downsample output as the residual) and a 256-channel block, both
16-bit types, a one-tile image (every border at once), tile counts that are not a multiple of the grid, batch 1, 3 and
SMs + 5 with distinct frames, the whole HRNet-W32 Engine and a ResNet-50 plan."""
import ctypes as C

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import ctensor, pack_conv_host, rup

pytestmark = pytest.mark.gpu


def _conv_weights(cout, cin, k, dt, g):
    w = (torch.randn(cout, cin, k, k, generator=g) * (2 / (k * k * cin)) ** 0.5).numpy()
    bn = [(torch.rand(cout, generator=g) + 0.5).numpy(), (torch.randn(cout, generator=g) * 0.1).numpy(),
          (torch.randn(cout, generator=g) * 0.1).numpy(), (torch.rand(cout, generator=g) + 0.5).numpy()]
    wp, b = pack_conv_host(w, None, bn, cin, cout, dt)
    return wp.view(np.uint8).reshape(-1), b


def _run_bottleneck(cin, dt, B, H, W, fuse, monkeypatch, seed=0):
    """One Bottleneck as a three-op plan (cin = 64: the residual is a separate 256-channel tensor, as a downsample's
    output; cin = 256: the block input) -> the 256-channel output (B, H, W, 256)."""
    monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", "1" if fuse else "0")
    g = torch.Generator().manual_seed(seed)
    tdt = torch.bfloat16 if dt == L.DT_BF16 else torch.float16
    x = torch.randn(B, H, W, cin, generator=g).to(tdt)
    res = x if cin == 256 else torch.randn(B, H, W, 256, generator=g).to(tdt)
    ws = [_conv_weights(64, cin, 1, dt, g), _conv_weights(64, 64, 3, dt, g), _conv_weights(256, 64, 1, dt, g)]
    offs, blob = [], []
    top = 0
    for w, b in ws:
        for a in (w, b.view(np.uint8)):
            offs.append(top)
            blob.append((top, a))
            top = rup(top + a.nbytes, 1024)
    wblob = np.zeros(top, np.uint8)
    for o, a in blob:
        wblob[o:o + a.nbytes] = a
    npx = B * H * W
    off_x = 0
    off_r = rup(npx * cin * 2, 1024)
    off_y1 = off_r + (rup(npx * 256 * 2, 1024) if cin == 64 else 0)
    off_y2 = off_y1 + rup(npx * 64 * 2, 1024)
    off_o = off_y2 + rup(npx * 64 * 2, 1024)
    arena = torch.zeros(off_o + rup(npx * 256 * 2, 1024), dtype=torch.uint8)
    arena[off_x:off_x + npx * cin * 2] = x.view(torch.uint8).flatten()
    if cin == 64:
        arena[off_r:off_r + npx * 256 * 2] = res.view(torch.uint8).flatten()
    else:
        off_r = off_x
    d_arena, d_blob = arena.cuda(), torch.from_numpy(wblob).cuda()
    t_x, t_r = ctensor(off_x, cin, H, W, cin, dt), ctensor(off_r, 256, H, W, 256, dt)
    t_y1, t_y2 = ctensor(off_y1, 64, H, W, 64, dt), ctensor(off_y2, 64, H, W, 64, dt)
    t_o = ctensor(off_o, 256, H, W, 256, dt)
    ops = (L.Op * 3)()
    geo = [(1, cin, 64, t_x, t_y1), (3, 64, 64, t_y1, t_y2), (1, 64, 256, t_y2, t_o)]
    for i, (o, (k, ci, co, tin, tout)) in enumerate(zip(ops, geo)):
        o.kind, o.k, o.stride, o.relu, o.cin_pad, o.cout_pad = L.OP_CONV, k, 1, 1, ci, co
        o.w_offset[0], o.w_offset[1] = offs[2 * i], offs[2 * i + 1]
        o.n_in, o.in_[0], o.out = 1, tin, tout
    ops[0].shift[0] = L.CONV_BOTTLENECK
    ops[2].n_in, ops[2].has_residual, ops[2].in_[1] = 2, 1, t_r
    lib = L.load()
    plan = C.c_void_p()
    L.check(lib.acr_b200_plan_create(ops, 3, B, d_arena.data_ptr(), d_arena.numel(), d_blob.data_ptr(), d_blob.numel(),
                                     dt, C.byref(plan)), "plan_create")
    try:
        assert lib.acr_b200_plan_num_launches(plan) == (1 if fuse else 3)
        L.check(lib.acr_b200_plan_run(plan, None, torch.cuda.current_stream().cuda_stream), "plan_run")
        torch.cuda.synchronize()
    finally:
        lib.acr_b200_plan_destroy(plan)
    return d_arena[off_o:off_o + npx * 256 * 2].view(tdt).view(B, H, W, 256).cpu()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (B, H, W): one tile; tile counts that are not a multiple of the grid; the layer1 grid at batch 1 and 3; past one
# tile per SM
SHAPES = [(1, 16, 16), (5, 48, 80), (1, 128, 128), (3, 128, 128), ("sms+5", 16, 16)]


@pytest.mark.parametrize("dt", [L.DT_BF16, L.DT_F16])
@pytest.mark.parametrize("cin", [64, 256])
@pytest.mark.parametrize("shape", SHAPES)
def test_fused_bottleneck_equals_three_launches(cin, dt, shape, monkeypatch):
    B, H, W = shape
    B = _sms() + 5 if B == "sms+5" else B
    ref = _run_bottleneck(cin, dt, B, H, W, False, monkeypatch)
    out = _run_bottleneck(cin, dt, B, H, W, True, monkeypatch)
    assert torch.equal(out, ref)
    assert out.float().abs().sum() > 0
    if B > 1:   # distinct frames give distinct outputs (no image is computed from another one's tiles)
        assert not torch.equal(out[0], out[B - 1])


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


def _engine_outputs(make, image, names_of, monkeypatch):
    res = {}
    for fuse in ("1", "0"):
        monkeypatch.setenv("ACR_B200_FUSE_BLOCKS", fuse)
        eng = make()
        eng.run(image)
        torch.cuda.synchronize()
        res[fuse] = ({n: eng.view(n).clone() for n in names_of(eng)}, eng.num_launches, list(eng.bottleneck_starts))
        del eng
    return res


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_engine_fused_bottlenecks_bit_identical(sd, dtype, monkeypatch):
    """HRNet-W32 at reuse_memory=True: every kept output and feat32, fused against unfused; 8 fewer launches."""
    from acr_b200.engine import Engine
    g = torch.Generator().manual_seed(5)
    image = torch.randint(0, 256, (3, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
    names = lambda e: ["segms", "l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps",
                       "r_prior_maps", "pooled", "feat32"]
    res = _engine_outputs(lambda: Engine(sd, 3, "cuda", dtype, keep_extra=("feat32",)), image, names, monkeypatch)
    assert len(res["1"][2]) == 4
    assert res["0"][1] - res["1"][1] == 4 * 2 + 80   # two launches saved per Bottleneck, one per BasicBlock
    for n, v in res["1"][0].items():
        assert torch.equal(v, res["0"][0][n]), n


def test_engine_resnet_fused_bottlenecks_bit_identical(monkeypatch):
    from acr_b200.engine import Engine
    from acr_b200.netspec import build_acr_spec
    from acr_b200.synth import synth_state_dict
    sdr = synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50"))
    g = torch.Generator().manual_seed(6)
    image = torch.randint(0, 256, (2, 512, 512, 3), generator=g, dtype=torch.uint8).cuda()
    names = lambda e: ["l_center_map", "r_center_map", "l_params_maps", "r_params_maps", "l_prior_maps", "r_prior_maps",
                       "pooled"]
    res = _engine_outputs(lambda: Engine(sdr, 2, "cuda", torch.bfloat16, backbone="resnet50"), image, names, monkeypatch)
    assert len(res["1"][2]) == 2
    for n, v in res["1"][0].items():
        assert torch.equal(v, res["0"][0][n]), n

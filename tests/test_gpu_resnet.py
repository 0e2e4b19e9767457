"""GPU: the ResNet-50 trunk (netspec.build_acr_spec(backbone="resnet50")) and the kernels it adds.

* op level, bf16 and fp16, against the CPU oracle (tests/resnet_ref.py, unrounded fp32 parameters) at the per-op bounds of
  the teacher-forced sweep (2^-7 / 2^-10): the transposed conv (MODE_DECONV of conv_tc), the 1x1 stride-2 conv, the
  2048-wide conv, the 7x7 tensor-core stem; the max-pool bit for bit against F.max_pool2d on the same 16-bit input;
* every launch of the whole ResNet plan, teacher forced;
* acr.main.ACR with backbone='resnet' from frames to MANO: finite, both hands found, the W32 run's schema, batch
  invariance, CUDA-graph replay == eager."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from acr_b200 import lib as L
from tests import resnet_ref
from tests.helpers import ctensor, pack_conv_host, rel_err, rup, run_conv_case, to_nhwc_padded

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}
DT = {torch.bfloat16: L.DT_BF16, torch.float16: L.DT_F16}
DTYPES = [torch.bfloat16, torch.float16]


def _bn_params(g, c):
    return [torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1, torch.randn(c, generator=g) * 0.1,
            torch.rand(c, generator=g) + 0.5]


def _bn_sd(key, bn):
    return {f"{key}.{n}": t for n, t in zip(("weight", "bias", "running_mean", "running_var"), bn)}


def _run_op(op, B, arena, blob, dt, external=None):
    L.check(L.load().acr_b200_run_op(C.byref(op), B, arena.data_ptr(), None if blob is None else blob.data_ptr(),
                                     None if external is None else external.data_ptr(), dt,
                                     torch.cuda.current_stream().cuda_stream), "run_op")
    torch.cuda.synchronize()


def _blob(*arrays):
    """uint8 CUDA blob of the arrays at 256-byte aligned offsets -> (blob, offsets)."""
    parts, offs, size = [], [], 0
    for a in arrays:
        pad = (-size) % 256
        parts.append(np.zeros(pad, np.uint8))
        size += pad
        offs.append(size)
        b = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        parts.append(b)
        size += b.size
    return torch.from_numpy(np.concatenate(parts)).cuda(), offs


# ------------------------------------------------------------------------------------------------------------ op level
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,cin,cout,out_stride", [
    (37, 16, 2048, 256, 256),    # deconv_layers.0: 2 N splits x 4 parities per 16x16 input tile
    (25, 32, 256, 128, 128),     # deconv_layers.3
    (5, 64, 128, 32, 48),        # deconv_layers.6 into channels [0, 32) of the 48-stride coord-concat buffer
])
def test_deconv_op(dtype, B, H, cin, cout, out_stride):
    """ConvTranspose2d(k4, s2, p1) + BN + ReLU as the conv_tc transposed-conv mode; the batch sizes give odd virtual tile
    counts per persistent CTA.  Channels past cout of a wider destination are never written."""
    from acr_b200.engine import deconv_parity_weights
    g = torch.Generator().manual_seed(cin + cout)
    dt = DT[dtype]
    x = torch.randn(B, cin, H, H, generator=g)
    w = torch.randn(cin, cout, 4, 4, generator=g) * (2.0 / (cin * 4)) ** 0.5
    bn = _bn_params(g, cout)
    cin_pad, cout_pad = rup(cin, 64), rup(cout, 16)
    par = deconv_parity_weights(w.numpy())
    wps, bias = [], None
    for p in range(4):
        wp, bias = pack_conv_host(par[p], None, [t.numpy() for t in bn], cin_pad, cout_pad, dt)
        wps.append(wp)
    blob, (w_off, b_off) = _blob(np.stack(wps), bias)
    xin = to_nhwc_padded(x, cin, dtype)
    off_o = rup(xin.numel() * 2, 1024)
    obytes = B * 4 * H * H * out_stride * 2
    arena = torch.zeros(off_o + obytes, dtype=torch.uint8, device="cuda")
    arena[:xin.numel() * 2] = xin.view(torch.uint8).flatten().cuda()
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 1
    op.in_[0] = ctensor(0, cin, H, H, cin, dt)
    op.out = ctensor(off_o, cout, 2 * H, 2 * H, out_stride, dt)
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    op.k, op.stride, op.relu, op.has_residual = 4, 2, 1, 0
    op.cin_pad, op.cout_pad = cin_pad, cout_pad
    op.shift[0] = L.CONV_DECONV
    _run_op(op, B, arena, blob, dt)
    out = arena[off_o:].view(dtype).view(B, 2 * H, 2 * H, out_stride).cpu()
    assert torch.equal(out[..., cout:], torch.zeros_like(out[..., cout:])), "channels past cout were written"
    got = out[..., :cout].float().permute(0, 3, 1, 2)
    sd = {"d.weight": w, **_bn_sd("b", bn)}
    torch.set_num_threads(min(32, os.cpu_count()))
    exp = resnet_ref.deconv_bn_relu(xin.float().permute(0, 3, 1, 2), sd, "d", "b")
    assert torch.isfinite(got).all()
    e = rel_err(got.numpy(), exp.numpy())
    assert e <= TOL[dtype], e


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,cin,cout", [(2, 128, 256, 512), (3, 64, 512, 1024), (3, 32, 1024, 2048)])
def test_1x1_stride2_op(dtype, B, H, cin, cout):
    """The downsample of the first block of layers 2-4: 1x1 stride 2, padding 0 (reads input pixel (2y, 2x)); the
    last one is 2048 wide (16 N splits of 128, K = 16 chunks of 64)."""
    got, exp, pad_ok = run_conv_case(L.OP_CONV, B, H, H, cin, cout, 1, 2, False, False, False, True, False, dt=DT[dtype])
    assert pad_ok
    e = rel_err(got.numpy(), exp.numpy())
    assert e <= TOL[dtype], e


@pytest.mark.parametrize("dtype", DTYPES)
def test_2048_wide_conv_with_residual(dtype):
    """layer4's conv3: 512 -> 2048 1x1 + BN + residual + ReLU at 16x16, 2048 output channels (cout_pad 2048)."""
    got, exp, pad_ok = run_conv_case(L.OP_CONV, 5, 16, 16, 512, 2048, 1, 1, True, True, False, True, False, dt=DT[dtype])
    assert pad_ok
    e = rel_err(got.numpy(), exp.numpy())
    assert e <= TOL[dtype], e


@pytest.mark.parametrize("dtype", DTYPES)
def test_stem7_op(dtype):
    """conv1 7x7 s2 p3 + bn1 + ReLU with the A operand built in shared memory from the uint8 frame (zeros in the padding,
    bias in spare K channels) against the oracle on the unrounded parameters."""
    g = torch.Generator().manual_seed(7)
    dt = DT[dtype]
    B, S = 3, 512
    img = torch.randint(0, 256, (B, S, S, 3), generator=g, dtype=torch.uint8)
    w = torch.randn(64, 3, 7, 7, generator=g) * (2.0 / 147) ** 0.5
    bn = _bn_params(g, 64)
    w1 = np.zeros((64, 160, 1, 1), np.float32)
    w1[:, :147, 0, 0] = w.permute(0, 2, 3, 1).reshape(64, 147).numpy()
    wp, bias = pack_conv_host(w1, None, [t.numpy() for t in bn], 160, 64, dt)
    blob, (w_off, b_off) = _blob(wp, bias)
    arena = torch.zeros(B * (S // 2) ** 2 * 64 * 2, dtype=torch.uint8, device="cuda")
    op = L.Op()
    op.kind, op.n_in, op.k = L.OP_STEM_TC, 1, 7
    op.in_[0] = ctensor(0, 3, S, S, 3, L.DT_U8, external=1)
    op.out = ctensor(0, 64, S // 2, S // 2, 64, dt)
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    d_img = img.cuda()
    _run_op(op, B, arena, blob, dt, external=d_img)
    got = arena.view(dtype).view(B, S // 2, S // 2, 64).float().permute(0, 3, 1, 2).cpu()
    torch.set_num_threads(min(32, os.cpu_count()))
    exp = resnet_ref.stem7(img, {"backbone.conv1.weight": w, **_bn_sd("backbone.bn1", bn)})
    e = rel_err(got.numpy(), exp.numpy())
    assert e <= TOL[dtype], e


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C_,stride", [(64, 64), (64, 80)])
def test_maxpool_op_bit_exact(dtype, C_, stride):
    """MaxPool 3x3 s2 p1 over the valid taps only: bit for bit F.max_pool2d on the same 16-bit input (negative values
    included, so a zero from the padding would show)."""
    g = torch.Generator().manual_seed(5)
    B, H = 3, 256
    x = torch.randn(B, H, H, stride, generator=g).to(dtype)
    arena = torch.zeros(x.numel() * 2 + B * (H // 2) ** 2 * stride * 2, dtype=torch.uint8, device="cuda")
    arena[:x.numel() * 2] = x.view(torch.uint8).flatten().cuda()
    dt = DT[dtype]
    op = L.Op()
    op.kind, op.n_in = L.OP_MAXPOOL, 1
    op.in_[0] = ctensor(0, C_, H, H, stride, dt)
    op.out = ctensor(x.numel() * 2, C_, H // 2, H // 2, stride, dt)
    _run_op(op, B, arena, None, dt)
    got = arena[x.numel() * 2:].view(dtype).view(B, H // 2, H // 2, stride)[..., :C_].cpu()
    exp = Fn.max_pool2d(x[..., :C_].cuda().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).cpu()
    assert torch.equal(got, exp)


# -------------------------------------------------------------------------------------------------- whole plan
@pytest.fixture(scope="module")
def sd_resnet():
    from acr_b200.netspec import build_acr_spec
    from acr_b200.synth import synth_state_dict
    return synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50"))


class _Without:
    """The engine seen without some launches (the existing sweep checks the rest)."""

    def __init__(self, eng, recs):
        self._eng, self.recs = eng, recs

    def __getattr__(self, name):
        return getattr(self._eng, name)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_op_of_the_resnet_plan_teacher_forced(sd_resnet, dtype):
    """Every launch of the ResNet plan against the oracle on the plan's own stored inputs: the ResNet kinds here, the rest
    (bottleneck convs incl. 1x1 stride 2, heads, SegmNet, pooling, part head) through tests/test_gpu_teacher_forced.sweep."""
    from acr_b200.engine import Engine
    from tests.pack_ref import check_bound, direction_counts, direction_ok
    from tests.test_gpu_teacher_forced import conv_bound, stem_bound, sweep
    torch.set_num_threads(min(32, os.cpu_count()))
    gi = torch.Generator().manual_seed(123)
    image = torch.randint(0, 256, (1, 512, 512, 3), generator=gi, dtype=torch.uint8)
    eng = Engine(sd_resnet, 1, "cuda", dtype, reuse_memory=False, backbone="resnet50")
    eng.run(image.cuda())
    torch.cuda.synchronize()
    sdf = {k: v.float() for k, v in sd_resnet.items() if v.dtype.is_floating_point}
    get = lambda t: eng.map_nchw(t).cpu()
    rows, rest = [], []
    for i, r in enumerate(eng.recs):
        a = r.get("attrs", {})
        if r["kind"] == L.OP_STEM_TC:
            rows.append((i, "stem 7x7", rel_err(get(r["out"]).numpy(), resnet_ref.stem7(image, sdf).numpy())))
            g, e64, acc, tdt = stem_bound(eng, i, {k: v.numpy() for k, v in sdf.items()}, eng.weights.cpu().numpy(), image)
            worst, nbad = check_bound(g, e64, acc, tdt)
            (tw, aw), (ta, aa) = direction_counts(g, e64, acc, tdt)
            print(f"stem 7x7: worst err/bound {worst:.3f}, off-RNE toward zero / away: decided {tw} / {aw}, all {ta} / {aa}")
            assert nbad == 0 and direction_ok(tw, aw), ("stem 7x7", worst, nbad, tw, aw)
        elif r["kind"] == L.OP_MAXPOOL:
            x = eng.view(r["ins"][0])[..., :64].permute(0, 3, 1, 2)
            exp = Fn.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1)
            assert torch.equal(eng.view(r["out"])[..., :64], exp), "max-pool"
            rows.append((i, "max-pool", 0.0))
        elif a.get("deconv"):
            exp = resnet_ref.deconv_bn_relu(get(r["ins"][0]), sdf, a["w"], a["bn"])
            rows.append((i, f"deconv {a['w']}", rel_err(get(r["out"]).numpy(), exp.numpy())))
            # per element: the live packed weights pinned to the restatement, the fp64 bound and the rounding direction
            g, e64, acc, tdt = conv_bound(eng, i, {k: v.numpy() for k, v in sdf.items()}, eng.weights.cpu().numpy(), get)
            worst, nbad = check_bound(g, e64, acc, tdt)
            (tw, aw), (ta, aa) = direction_counts(g, e64, acc, tdt)
            print(f"deconv {a['w']}: worst err/bound {worst:.3f}, off-RNE toward zero / away: decided {tw} / {aw}, all {ta} / {aa}")
            assert nbad == 0 and direction_ok(tw, aw), (a["w"], worst, nbad, tw, aw)
        else:
            rest.append(r)
    kinds = [r["kind"] for r in eng.recs]
    assert kinds.count(L.OP_MAXPOOL) == 1 and kinds.count(L.OP_STEM_TC) == 1 and len(rows) == 5
    rows += sweep(_Without(eng, rest), sd_resnet, image, TOL[dtype])
    print(f"resnet teacher-forced sweep {dtype}: {len(rows)} checks over {len(eng.recs)} launches; worst:",
          sorted(rows, key=lambda r: -r[2])[:5])
    assert len(rows) >= len(eng.recs) - 1
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[dtype]]
    assert not bad, f"{len(bad)} ops above {TOL[dtype]:.2e}: {bad[:8]}"


# ------------------------------------------------------------------------------------------------------ drop-in
@pytest.fixture
def resnet_args():
    from acr.config import args
    old = args().backbone
    args().backbone = "resnet"
    yield args()
    args().backbone = old


def _assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


def test_dropin_resnet_end_to_end(sd_resnet, resnet_args):
    """acr.main.ACR with backbone='resnet': frames -> trunk -> heads -> parse -> MANO.  Finite outputs, both hands detected
    (synthetic centre bias), the same output schema as the W32 run, and batch 4 == 4 x batch 1 bit for bit."""
    from acr.config import args
    from acr.main import ACR
    from acr_b200.synth import synth_state_dict
    gi = torch.Generator().manual_seed(11)
    frames = torch.randint(0, 256, (4, 512, 512, 3), generator=gi, dtype=torch.uint8)
    app = ACR(state_dict=sd_resnet, mano_assets=_assets())
    assert app.model._spec.backbone == "resnet50"
    out = app.batch_forward(frames)
    torch.cuda.synchronize()
    for k in ("verts", "j3d", "pj2d_org", "params_pred", "l_center_map", "segms"):
        assert torch.isfinite(out[k]).all(), k
    hand_type = out["output_hand_type"].cpu().numpy()
    assert set(hand_type.tolist()) == {0, 1} and len(hand_type) == 8, hand_type   # both hands in every frame
    per = []
    for b in range(4):
        o = app.batch_forward(frames[b:b + 1])
        per.append({k: o[k].clone() for k in ("verts", "params_pred", "l_center_map", "r_params_maps")})
    for k in ("l_center_map", "r_params_maps"):
        assert torch.equal(out[k], torch.cat([p[k] for p in per])), k
    by_img = out["reorganize_idx"].cpu().numpy()
    for b in range(4):
        rows = np.nonzero(by_img == b)[0]
        assert torch.equal(out["verts"][rows], per[b]["verts"]) and torch.equal(out["params_pred"][rows], per[b]["params_pred"])
    # same schema (keys, per-key dtype and trailing shape) as the HRNet-W32 run
    args().backbone = "hrnet"
    w32 = ACR(state_dict=synth_state_dict(0), mano_assets=_assets()).batch_forward(frames[:1])
    args().backbone = "resnet"
    assert set(out.keys()) == set(w32.keys())
    for k, v in w32.items():
        if torch.is_tensor(v):
            assert out[k].dtype == v.dtype and tuple(out[k].shape[1:]) == tuple(v.shape[1:]), k


def test_resnet_fused_forward_and_graph_replay(sd_resnet, resnet_args):
    """The sync-free pipeline (fused_forward) on the ResNet trunk, and its CUDA-graph capture == eager bit for bit."""
    from acr.main import ACR
    app = ACR(state_dict=sd_resnet, mano_assets=_assets())
    gi = torch.Generator().manual_seed(78)
    offs = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(2, 1).cuda()
    replay = app.capture_graph(2)
    for _ in range(2):
        frame = torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8).cuda()
        bufs, mano = app.fused_forward(frame, offs)
        torch.cuda.synchronize()
        n = int(bufs.counts[2])
        assert n == 4
        v_eager, p_eager = mano["verts"][:n].clone(), bufs.params_pred[:n].clone()
        bufs_g, mano_g = replay(frame, offs)
        torch.cuda.synchronize()
        assert int(bufs_g.counts[2]) == n
        assert torch.equal(mano_g["verts"][:n], v_eager) and torch.equal(bufs_g.params_pred[:n], p_eager)


def test_head_forward_on_resnet_model(sd_resnet, resnet_args):
    """ACR.head_forward (the heads-only plan) on a ResNet model: the heads are the reference's own, so the trunk's
    (B,32,128,128) feature of the full plan fed back through head_forward gives the full plan's maps."""
    from acr.model import ACR as Model
    from acr_b200.engine import Engine
    m = Model().cuda()
    m.load_state_dict(sd_resnet, strict=True)
    gi = torch.Generator().manual_seed(3)
    frames = torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8)
    full = Engine(sd_resnet, 2, "cuda", torch.bfloat16, backbone="resnet50", keep_extra=("feat32",))   # feat32 kept alive
    full.run(frames.cuda())
    maps = m.head_forward(full.map_nchw("feat32"))
    for k in ("l_center_map", "r_params_maps", "segms"):
        assert torch.equal(maps[k], full.map_nchw(k)), k

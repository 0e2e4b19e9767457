"""GPU: acr_b200_part_labels against the fp64 statement (tests/part_labels_ref.py).

* bf16 / fp16 / fp32 logit maps at the arena's 48-channel stride: smooth random fields (many part boundaries), planted
  near-ties within an ulp, constant maps; frames 1x1, 1x4032, 4032x1, 255x255, 720p, 1080p and 3024x4032.  A label may
  differ from the statement only where the fp64 margin between the two labels is within the kernel's fp32 bound
  (part_labels_ref.fp32_bound_scale); the number of such pixels is printed.  Two calls give the same bytes.
* invalid offsets rows and frames past the capacity are flagged and get no stores;
* through the network on the seeded weights: the eager path, fused_forward, frame-graph replays with changing sizes
  and a JPEG-graph replay give the statement's labels of outputs['segms'] (and the eager path's bytes); once each the
  TF32 plan, the fp32 plan, the ResNet trunk and K = 4 with a tracker.
"""
import numpy as np
import pytest
import torch

from acr_b200 import ops
from acr_b200.preprocess import offsets_vector, preprocess_frames
from tests import part_labels_ref as ref

pytestmark = pytest.mark.gpu

FRAMES = [(1, 1), (1, 4032), (4032, 1), (255, 255), (720, 1280), (1080, 1920), (3024, 4032)]
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _smooth_maps(n, seed, dtype, scale=4.0):
    """(n, 256, 256, 48) NHWC logits: 33 bilinearly upsampled 16 x 16 random fields, garbage in channels 33..47."""
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(n, 33, 16, 16, generator=g, dtype=torch.float64) * scale
    up = torch.nn.functional.interpolate(low, size=(256, 256), mode="bilinear", align_corners=False)
    m = torch.full((n, 256, 256, 48), 1e4, dtype=torch.float64)
    m[..., :33] = up.permute(0, 2, 3, 1)
    return m.to(dtype).cuda().contiguous()


def _run(segms, rows):
    rows = np.asarray(rows, np.float32)
    buf = ops.PartLabels(ops.part_label_layout(rows, 0)[2], len(rows))
    ops.part_labels(segms, torch.from_numpy(rows), buf)
    torch.cuda.synchronize()
    return buf


def _check(segms, rows, buf, what):
    """Every image's labels against the statement; returns the exempt pixel count."""
    exempt = 0
    for i, row in enumerate(rows):
        segm = segms[i, :, :, :33].float().cpu().numpy()
        bad, ex = ref.compare(segm, row, buf[i].cpu().numpy())
        assert bad == 0, f"{what} image {i} ({ref.frame_geometry(row)}): {bad} labels off the statement"
        exempt += ex
    return exempt


@pytest.mark.parametrize("dt", list(DTYPES))
def test_kernel_equals_the_statement_on_smooth_fields(dt):
    frames = FRAMES if dt == "bf16" else FRAMES[:-1]        # the 12 MP frame once: its fp64 statement is slow
    rows = [offsets_vector(*f) for f in frames]
    segms = _smooth_maps(len(rows), 1, DTYPES[dt])
    buf = _run(segms, rows)
    first = buf.data.clone()
    ops.part_labels(segms, torch.from_numpy(np.stack(rows)), buf)
    torch.cuda.synchronize()
    assert torch.equal(first, buf.data), "two calls gave different bytes"
    ex = _check(segms, rows, buf, dt)
    n = sum(h * w for h, w in frames)
    counts = np.bincount(buf.data.cpu().numpy(), minlength=33)
    print(f"\n{dt}: {n} pixels, {ex} within the fp32 bound of the statement, {int((counts > 0).sum())} labels used")
    assert (counts > 0).sum() >= 20, "the fields should cover most part labels"


def test_near_ties_and_constant_maps():
    n = 4
    segms = _smooth_maps(n, 2, torch.float32, scale=1.0)
    g = torch.Generator().manual_seed(3)
    cells = torch.randint(0, 256, (n, 400, 2), generator=g)
    for i in range(n):                              # channel pairs equal or one ulp apart at planted cells
        for k, (y, x) in enumerate(cells[i].tolist()):
            a, b = (k % 33), (k * 7 + 3) % 33
            v = segms[i, y, x, :33].max() + 0.5
            segms[i, y, x, a] = v
            segms[i, y, x, b] = v if k % 2 else torch.nextafter(v, v + 1)
    segms[3, :, :, :33] = 0.25                      # a constant map: every channel ties, label 0
    rows = [offsets_vector(720, 1280), offsets_vector(300, 257), offsets_vector(255, 255), offsets_vector(1080, 1920)]
    buf = _run(segms, rows)
    ex = _check(segms, rows, buf, "near ties")
    assert (buf[3] == 0).all()
    bf = _run(segms.to(torch.bfloat16), rows)
    ex += _check(segms.to(torch.bfloat16), rows, bf, "near ties bf16")
    print(f"\nnear ties: {ex} pixels within the fp32 bound of the statement")


def test_invalid_rows_and_capacity_get_flags_and_no_stores():
    segms = _smooth_maps(6, 4, torch.bfloat16)
    rows = np.stack([offsets_vector(40, 30),
                     np.array([10, 10, 0, 0, 0, 0, 0.5, 0, 0, 0], np.float32),   # non-integer
                     offsets_vector(20, 20),
                     np.array([10, 10, 0, 0, 0, 0, 6, 0, 4, 0], np.float32),     # pad_t + pad_b >= side
                     offsets_vector(50, 50),                                       # past the capacity
                     np.array([16385, 16385, 0, 0, 0, 0, 0, 0, 0, 0], np.float32)]).astype(np.float32)
    cap = 40 * 30 + 20 * 20 + 100
    buf = ops.PartLabels(cap + 64, 6)
    buf.capacity = cap                              # the bytes past `cap` must stay untouched too
    buf.data.fill_(0xAB)
    ops.part_labels(segms, torch.from_numpy(rows).cuda(), buf)      # device offsets: checked on the device
    torch.cuda.synchronize()
    start, H, W, flags = ref.packing(rows, cap)
    assert buf.flags.cpu().numpy().tolist() == flags.tolist() == [0, 1, 0, 1, 2, 1]
    assert np.array_equal(buf.frame_offset.cpu().numpy(), start)
    data = buf.data.cpu().numpy()
    assert (data[40 * 30 + 20 * 20:] == 0xAB).all()
    assert (data[:40 * 30 + 20 * 20] != 0xAB).all()
    for i in (1, 3, 4, 5):
        with pytest.raises(ValueError, match="no part labels"):
            buf[i]
    _check(segms[[0, 2]], rows[[0, 2]], _run(segms[[0, 2]], rows[[0, 2]]), "valid rows")
    assert torch.equal(buf[0], _run(segms[[0]], rows[[0]])[0])


# ------------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def app():
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    a = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
    yield a
    del a
    torch.cuda.empty_cache()


def _bgr(shapes, seed):
    rng = np.random.default_rng(seed)
    out = []
    for h, w in shapes:   # a smooth image with some texture: the seeded network gives varied maps
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 100 * np.sin(yy / 37.0 + seed) * np.cos(xx / 23.0))[..., None]
        out.append(np.clip(base + rng.integers(-40, 40, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def _eager(app, frames, **cfg):
    """batch_forward with return_part_labels (and any other args() overrides) -> (labels list on the CPU, segms)."""
    from acr.config import args
    old = {k: getattr(args(), k) for k in cfg}
    args().return_part_labels = True
    for k, v in cfg.items():
        setattr(args(), k, v)
        setattr(app, k, v)                          # acr.main.ACR copies args() at construction
    try:
        img, offs = preprocess_frames(frames)
        out = app.batch_forward(img, offs)
        segms = out["segms"].permute(0, 2, 3, 1).contiguous()
        labels = [t.cpu() for t in out["part_labels"]]
    finally:
        args().return_part_labels = False
        for k, v in old.items():
            setattr(args(), k, v)
            setattr(app, k, v)
    assert len(labels) == len(frames)
    for lab, f in zip(labels, frames):
        assert lab.shape == f.shape[:2] and lab.dtype == torch.uint8
    rows = offs.numpy()
    ex = 0
    for i, row in enumerate(rows):
        bad, e = ref.compare(segms[i].cpu().numpy(), row, labels[i].numpy())
        assert bad == 0, (cfg, i)
        ex += e
    print(f"\neager {cfg or 'bf16'}: {ex} pixels within the fp32 bound of the statement")
    return labels, segms, offs


SHAPES_A = [(720, 1280), (1080, 1920), (37, 1001)]
SHAPES_B = [(1, 1), (1920, 1080), (480, 640)]


def test_eager_fused_and_frame_graph_replays(app):
    frames_a, frames_b = _bgr(SHAPES_A, 0), _bgr(SHAPES_B, 1)
    exp_a, _, offs_a = _eager(app, frames_a)
    exp_b, _, _ = _eager(app, frames_b)
    # fused_forward into a caller's buffer
    img, offs = preprocess_frames(frames_a)
    buf = ops.PartLabels(sum(h * w for h, w in SHAPES_A), 3)
    _, mano = app.fused_forward(img, offs, part_labels=buf)
    assert mano["part_labels"] is buf
    for i in range(3):
        assert torch.equal(buf[i].cpu(), exp_a[i])
    with pytest.raises(ValueError, match="capacity"):
        app.fused_forward(img, offs, part_labels=ops.PartLabels(100, 3))
    # frame-graph replays with changing sizes
    replay = app.capture_frames_graph(3, max(sum(h * w * 3 for h, w in s) for s in (SHAPES_A, SHAPES_B)),
                                      part_labels=True)
    for frames, exp in ((frames_a, exp_a), (frames_b, exp_b), (frames_a, exp_a)):
        _, mano = replay(frames)
        labels = mano["part_labels"]
        assert labels is replay.part_labels and len(labels) == 3
        for i in range(3):
            assert torch.equal(labels[i].cpu(), exp[i])
    # capture_graph on device offsets: the views read the geometry back
    g = app.capture_graph(3, part_labels=sum(h * w for h, w in SHAPES_A))
    _, mano = g(img, offs.cuda())
    for i in range(3):
        assert torch.equal(mano["part_labels"][i].cpu(), exp_a[i])
    _, mano = g(img, offs)
    for i in range(3):
        assert torch.equal(mano["part_labels"][i].cpu(), exp_a[i])
    with pytest.raises(ValueError, match="capacity in pixels"):
        app.capture_graph(3, part_labels=True)


def test_jpeg_graph_replay(app):
    from acr_b200 import jpeg
    from tests import jpeg_cases as JC
    specs = [(720, 1280, 90, "420", 0, "smooth"), (17, 9, 100, "444", 1, "noisy"), (1080, 1920, 90, "422", 4, "smooth")]
    files = [JC.encode(*s) for s in specs]
    coded = sum(jpeg.parse(b).scan_len for b in files)
    frame_bytes = sum(jpeg.parse(b).H * jpeg.parse(b).W * 3 for b in files)
    exp, _, _ = _eager(app, [JC.cv2_decode(b) for b in files])
    replay = app.capture_jpeg_graph(3, coded, frame_bytes, part_labels=True)
    _, mano = replay(files)
    replay.jpeg.raise_on_status()
    for i in range(3):
        assert torch.equal(mano["part_labels"][i].cpu(), exp[i])


@pytest.mark.parametrize("cfg", [dict(model_precision="tf32"), dict(model_precision="fp32"),
                                 dict(max_hands_per_side=4, track_hands=True)], ids=["tf32", "fp32", "K4-tracker"])
def test_precisions_and_multi_hand(app, cfg):
    _eager(app, _bgr([(720, 1280), (300, 200)], 5), **cfg)


def test_resnet_trunk():
    from acr.config import args
    from acr.main import ACR
    from acr_b200.netspec import build_acr_spec
    from acr_b200.synth import make_synthetic_mano, synth_state_dict
    old = args().backbone
    args().backbone = "resnet"
    try:
        a = ACR(state_dict=synth_state_dict(0, spec=build_acr_spec(512, backbone="resnet50")),
                mano_assets={"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")})
        assert a.model._spec.backbone == "resnet50"
        _eager(a, _bgr([(720, 1280), (300, 200)], 6))
    finally:
        args().backbone = old

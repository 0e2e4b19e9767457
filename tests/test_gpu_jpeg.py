"""GPU: baseline JPEG decoding on the device (csrc/jpeg.cu, acr_b200.jpeg).

* every file of the test matrix (tests/jpeg_cases.py) decodes equal to cv2.imdecode, batched per size;
* a batch mixing every size and sampling gives each file the bytes it gets alone;
* decoded frames through preprocess_frames + batch_forward == the same path fed with cv2-decoded frames;
* capture_jpeg_graph replays == the eager path over several replays, with and without a tracker; over-cap batches
  raise before launch;
* host_fallback puts a progressive file into a mixed batch;
* a truncated file raises through the status word and decodes black; bit-flipped files give the right shape or
  JpegError;
* the device's quantised coefficients equal oracle/jpeg_ref.coefficients; data after the first EOI is ignored.
"""
import numpy as np
import pytest
import torch

from acr_b200 import jpeg
from tests import jpeg_cases as JC

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("size", JC.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_matrix_equals_cv2(size):
    cases = JC.matrix([size])
    bufs = [JC.encode(*c) for c in cases]
    bad = []
    for k in range(0, len(bufs), 30):
        out = jpeg.decode(bufs[k:k + 30])
        for c, b, o in zip(cases[k:k + 30], bufs[k:k + 30], out):
            if not np.array_equal(o.cpu().numpy(), JC.cv2_decode(b)):
                bad.append(c)
    assert not bad, f"{len(bad)} of {len(cases)} files differ from cv2, first {bad[:4]}"


def test_mixed_batch_equals_each_file_alone():
    cases = [(h, w, q, s, r, c) for (h, w) in JC.SIZES for s in JC.SAMPLINGS
             for q, r, c in ((90, 0, "smooth"), (50, 4, "noisy"))]
    bufs = [JC.encode(*c) for c in cases]
    order = np.random.default_rng(3).permutation(len(bufs))
    mixed = jpeg.decode([bufs[i] for i in order])
    for j, i in enumerate(order):
        alone = jpeg.decode([bufs[i]])[0]
        assert torch.equal(mixed[j], alone), cases[i]
        assert np.array_equal(alone.cpu().numpy(), JC.cv2_decode(bufs[i])), cases[i]


def test_host_fallback_puts_a_progressive_file_into_the_batch():
    prog = JC.encode(17, 9, 90, "420", 0, "smooth", progressive=True)
    bufs = [JC.encode(720, 1280, 90, "422", 0, "smooth"), prog, JC.encode(7, 13, 50, "grey", 1, "noisy")]
    with pytest.raises(jpeg.JpegUnsupported, match="progressive"):
        jpeg.decode(bufs)
    out = jpeg.decode(bufs, host_fallback=True)
    for o, b in zip(out, bufs):
        assert np.array_equal(o.cpu().numpy(), JC.cv2_decode(b))
    assert out[0].untyped_storage().data_ptr() == out[2].untyped_storage().data_ptr()   # one packed buffer


def test_coefficients_equal_the_oracle():
    from oracle import jpeg_ref
    bufs = [JC.encode(*c) for c in [(720, 1280, 90, "420", 0, "noisy"), (17, 9, 100, "444", 1, "noisy"),
                                    (7, 13, 50, "grey", 4, "smooth"), (720, 1280, 50, "422", 4, "smooth"),
                                    (17, 9, 90, "440", 0, "noisy"), (1, 1, 90, "420", 0, "smooth")]]
    lay, _ = jpeg.plan(bufs)
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks)
    jb.load(bufs, lay)
    jb.launch()
    jb.raise_on_status()
    for i, b in enumerate(bufs):
        exp = jpeg_ref.coefficients(b)
        got = jb.coefficients(i)
        assert len(got) == len(exp)
        for c, (g, e) in enumerate(zip(got, exp)):
            assert np.array_equal(g.cpu().numpy(), e), (i, c)


def test_data_after_the_first_eoi_is_ignored():
    first = JC.encode(720, 1280, 90, "420", 0, "smooth")
    f = first + JC.encode(17, 9, 90, "444", 4, "noisy")      # an appended preview / trailer
    out = jpeg.decode([JC.encode(7, 13, 90, "422", 0, "noisy"), f])
    assert np.array_equal(out[1].cpu().numpy(), JC.cv2_decode(f))


def test_truncated_file_raises_through_the_status_word():
    good = JC.encode(720, 1280, 90, "420", 0, "noisy")
    small = JC.encode(7, 13, 90, "444", 0, "smooth")
    info = jpeg.parse(good)
    for cut in (info.scan_offset + info.scan_len // 3, info.scan_offset + info.scan_len - 40):
        bad = good[:cut] + b"\xff\xd9"          # a file cut inside its scan, closed with an EOI
        with pytest.raises(jpeg.JpegError, match="file 1: corrupt"):
            jpeg.decode([small, bad])
        lay, _ = jpeg.plan([small, bad])        # the batch's other frame decodes; the corrupt one is black
        jb = jpeg.JpegBatch(2, lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks)
        jb.out.fill_(77)
        jb.load([small, bad], lay)
        jb.launch()
        fr = jb.frames()
        assert int(jb.status[1]) != 0 and int(jb.status[0]) == 0
        assert np.array_equal(fr[0].cpu().numpy(), JC.cv2_decode(small))
        assert int(fr[1].max()) == 0
    ok = jpeg.decode([good])[0]                 # the decoder still works after a failed batch
    assert np.array_equal(ok.cpu().numpy(), JC.cv2_decode(good))


def test_bit_flipped_files_give_an_image_or_the_error():
    rng = np.random.default_rng(11)
    base = [JC.encode(720, 1280, 90, "420", 4, "smooth"), JC.encode(17, 9, 100, "444", 0, "noisy"),
            JC.encode(1080, 1920, 50, "440", 0, "noisy")]
    n_img = n_err = 0
    for b in base:
        info = jpeg.parse(b)
        for _ in range(8):
            a = bytearray(b)
            for _ in range(int(rng.integers(1, 4))):
                p = info.scan_offset + int(rng.integers(0, info.scan_len))
                a[p] ^= 1 << int(rng.integers(0, 8))
            try:
                out = jpeg.decode([bytes(a)])[0]
                assert out.shape == (info.H, info.W, 3)
                n_img += 1
            except jpeg.JpegError:
                n_err += 1
    torch.cuda.synchronize()
    assert n_img + n_err == 24
    ok = jpeg.decode(base)                      # no fault: later batches still decode
    for o, b in zip(ok, base):
        assert np.array_equal(o.cpu().numpy(), JC.cv2_decode(b))


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


def _files(specs):
    return [JC.encode(*s) for s in specs]


MIX_A = [(720, 1280, 90, "420", 0, "smooth"), (17, 9, 100, "444", 1, "noisy"), (1080, 1920, 90, "422", 4, "smooth"),
         (7, 13, 50, "grey", 0, "smooth")]
MIX_B = [(1080, 1920, 50, "440", 0, "noisy"), (1, 1, 90, "420", 0, "smooth"), (720, 1280, 100, "grey", 4, "smooth"),
         (720, 1280, 90, "444", 0, "noisy")]


def test_jpeg_frames_through_batch_forward_equal_cv2_frames(app):
    from acr.utils import img_preprocess, img_preprocess_jpeg
    bufs = _files(MIX_A)
    paths = [f"/frames/{i:06d}.jpg" for i in range(len(bufs))]
    meta = img_preprocess_jpeg(bufs, paths)
    ref_meta = img_preprocess([JC.cv2_decode(b) for b in bufs], paths)
    assert meta["imgpath"] == paths and torch.equal(meta["image"], ref_meta["image"])
    assert torch.equal(meta["offsets"], ref_meta["offsets"])
    out = app.batch_forward(meta["image"], meta["offsets"])
    ref = app.batch_forward(ref_meta["image"], ref_meta["offsets"])
    torch.cuda.synchronize()
    for k in ("reorganize_idx", "detection_flag", "params_pred", "verts", "j3d", "pj2d", "pj2d_org", "cam_trans"):
        assert torch.equal(out[k], ref[k]), k


def _snapshot(bufs, mano):
    torch.cuda.synchronize()
    n = int(bufs.counts[2])
    snap = [bufs.counts.clone(), bufs.params_pred[:n].clone(), bufs.offsets_out[:n].clone(), mano["verts"][:n].clone(),
            mano["pj2d_org"][:n].clone()]
    if "track_id" in mano:
        snap.append(mano["track_id"][:n].clone())
    return snap


@pytest.mark.parametrize("tracked", [False, True], ids=["plain", "tracker"])
def test_jpeg_graph_replays_equal_eager(app, tracked):
    from acr_b200.ops import HandTracker
    from acr_b200.preprocess import preprocess_frames
    from acr.result_parser import ResultParser
    mixes = [_files(MIX_A), _files(MIX_B), _files(MIX_A[::-1])]
    coded = max(sum(jpeg.parse(b).scan_len for b in m) for m in mixes)
    frame_bytes = max(sum(jpeg.parse(b).H * jpeg.parse(b).W * 3 for b in m) for m in mixes)
    K = ResultParser.hands_per_side()
    t_graph = HandTracker("cuda", K) if tracked else None
    t_eager = HandTracker("cuda", K) if tracked else None
    replay = app.capture_jpeg_graph(4, coded, frame_bytes, tracker=t_graph)
    for mix in mixes:
        img, offs = preprocess_frames([torch.from_numpy(JC.cv2_decode(b)).cuda() for b in mix])
        exp = _snapshot(*app.fused_forward(img, offs.cuda(), tracker=t_eager))
        got = _snapshot(*replay(mix))
        replay.jpeg.raise_on_status()
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            assert torch.equal(g, e)
    big = _files([(1080, 1920, 100, "444", 0, "noisy")] * 4)
    with pytest.raises(ValueError, match="capacity"):
        replay(big)
    with pytest.raises(ValueError, match="exactly"):
        replay(mixes[0][:3])
    with pytest.raises(jpeg.JpegUnsupported, match="progressive"):
        replay(mixes[0][:3] + [JC.encode(17, 9, 90, "420", 0, "smooth", progressive=True)])

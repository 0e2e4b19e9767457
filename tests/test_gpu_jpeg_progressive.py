"""GPU: progressive and multi-scan sequential JPEG files on the device (acr_b200_jpeg_decode_scans, ``max_scans``).

* cv2 progressive files (every sampling, with and without RST, up to 1080p, and a 12 MP and a 24 MP file), Pillow
  progressive files, every script of the progressive writer and multi-scan sequential files decode equal to cv2.imdecode with status 0, and their
  coefficients equal the numpy statement (tests/jpeg_progressive_ref.py);
* a mixed batch (baseline, progressive, multi-scan sequential, host fallback) equals each file decoded alone, and a
  baseline-only batch gives the same bytes with and without scan capacity;
* a progressive file with a cut scan sets its status bits and decodes black; bit flips give status bits or an image;
* capture_jpeg_graph(max_scans=N) replays with different script mixes equal fused_forward on cv2 frames, with and
  without a tracker; a replay over a cap raises before it writes, and the next one is still right.
"""
import numpy as np
import pytest
import torch

from acr_b200 import jpeg
from tests import jpeg_cases as JC
from tests import jpeg_progressive_ref as PR
from tests import jpeg_progressive_writer as PW

pytestmark = pytest.mark.gpu
BIG = 4096     # scan capacity for planning: larger than any batch here needs


def _batch(bufs, max_scans=None):
    lay, fb = jpeg.plan(bufs, max_scans=BIG if max_scans is None else max_scans)
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks,
                        max_scans=len(lay.scans) if max_scans is None else max_scans)
    jb.load(bufs, lay)
    jb.launch()
    return jb


def _corpus():
    out = {}
    for (h, w) in ((1, 1), (7, 13), (17, 9), (37, 53), (720, 1280), (1080, 1920)):
        for s in JC.SAMPLINGS:
            for r in (0, 4):
                out[f"cv2-{h}x{w}-{s}-r{r}"] = PW.cv2_progressive(h, w, 90, s, r, "smooth" if h > 100 else "noisy")
    for sub in (0, 1, 2):
        out[f"pillow-{sub}"] = PW.pillow_progressive(45, 83, 80, sub)
    for s in ("444", "422", "420", "440"):
        b0 = JC.encode(37, 53, 90, s, 0, "noisy")
        out[f"multi-{s}-a"] = PW.multi_scan_sequential(b0, [[0], [1, 2]], (3, 0))
        out[f"multi-{s}-b"] = PW.multi_scan_sequential(b0, [[1], [0], [2]], (1, 5, 2))
    return out


def test_corpus_equals_cv2_and_the_statement():
    files = _corpus()
    names = list(files)
    bad = []
    for k in range(0, len(names), 16):
        group = names[k:k + 16]
        jb = _batch([files[n] for n in group])
        fr = jb.frames()
        st = jb.status[:len(group)].cpu().numpy()
        for i, n in enumerate(group):
            b = files[n]
            if st[i] != 0 or not np.array_equal(fr[i].cpu().numpy(), JC.cv2_decode(b)):
                bad.append((n, int(st[i])))
            elif jpeg.parse(b, BIG).H < 100:
                exp = PR.coefficients(b)
                for c, g in enumerate(jb.coefficients(i)):
                    if not np.array_equal(g.cpu().numpy(), exp[c]):
                        bad.append((n, f"coefficients {c}"))
    assert not bad, bad[:8]


def test_writer_scripts_equal_cv2_and_the_statement():
    """Every script of tests/jpeg_progressive_writer.py, every sampling, optimal and all-long tables, and the file
    with an EOB run of 32767 blocks: equal to cv2 with status 0, coefficients equal to the statement's."""
    from tests.test_cpu_jpeg_progressive import long_eob_file, writer_files
    files = {k: v[0] for k, v in writer_files().items()}
    files["long-eob"] = long_eob_file()[0]
    names = list(files)
    bad = []
    for k in range(0, len(names), 12):
        group = names[k:k + 12]
        jb = _batch([files[n] for n in group])
        fr = jb.frames()
        st = jb.status[:len(group)].cpu().numpy()
        for i, n in enumerate(group):
            b = files[n]
            if st[i] != 0 or not np.array_equal(fr[i].cpu().numpy(), JC.cv2_decode(b)):
                bad.append((n, int(st[i])))
                continue
            exp = PR.coefficients(b)
            for c, g in enumerate(jb.coefficients(i)):
                if not np.array_equal(g.cpu().numpy(), exp[c]):
                    bad.append((n, f"coefficients {c}"))
    assert not bad, bad[:8]


def test_large_progressive_files_equal_cv2():
    import cv2
    for h, w, s in ((3000, 4000, "420"), (4000, 6000, "422")):
        rng = np.random.default_rng(h)
        img = np.clip(JC.image(h, w, "smooth").astype(np.int16) + rng.integers(-6, 7, (h, w, 3), dtype=np.int16),
                      0, 255).astype(np.uint8)
        ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1,
                                             cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                             getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{s}")])
        b = buf.tobytes()
        out = jpeg.decode([b], max_scans=BIG)[0]
        assert np.array_equal(out.cpu().numpy(), JC.cv2_decode(b)), (h, w)


def test_mixed_batch_equals_each_file_alone():
    incomplete = PW.cv2_progressive(17, 9, 90, "420", 0)
    info = jpeg.parse(incomplete, BIG)
    last = info.scans[-1]
    sos = incomplete.rfind(b"\xff\xda", 0, last.offset)
    incomplete = incomplete[:sos] + b"\xff\xd9"                # no last refinement: the host decodes it
    bufs = [JC.encode(720, 1280, 90, "420", 0, "smooth"), PW.cv2_progressive(720, 1280, 90, "444", 4, "smooth"),
            PW.multi_scan_sequential(JC.encode(37, 53, 90, "420", 0, "noisy"), [[0], [1, 2]]), incomplete,
            PW.pillow_progressive(45, 83, 80, 2), JC.encode(7, 13, 50, "grey", 1, "noisy"),
            PW.cv2_progressive(17, 9, 50, "grey", 1)]
    order = np.random.default_rng(5).permutation(len(bufs))
    mixed = jpeg.decode([bufs[i] for i in order], host_fallback=True, max_scans=BIG)
    for j, i in enumerate(order):
        alone = jpeg.decode([bufs[i]], host_fallback=True, max_scans=BIG)[0]
        assert torch.equal(mixed[j], alone), i
        assert np.array_equal(alone.cpu().numpy(), JC.cv2_decode(bufs[i])), i


def test_baseline_batch_is_the_same_with_scan_capacity():
    bufs = [JC.encode(*c) for c in [(720, 1280, 90, "420", 4, "noisy"), (17, 9, 100, "444", 1, "noisy"),
                                    (7, 13, 50, "grey", 0, "smooth"), (1080, 1920, 90, "422", 0, "smooth")]]
    a = _batch(bufs, max_scans=0)
    b = _batch(bufs, max_scans=24)
    torch.cuda.synchronize()
    assert torch.equal(a.out, b.out) and torch.equal(a.status, b.status) and int(a.status.abs().sum()) == 0


def test_cut_and_flipped_progressive_files():
    good = PW.cv2_progressive(720, 1280, 90, "420", 4, "smooth")
    small = PW.cv2_progressive(17, 9, 90, "444", 0)
    info = jpeg.parse(good, BIG)
    for k in (1, 4, len(info.scans) - 1):                      # a scan cut short, the later scans kept
        s = info.scans[k]
        bad = good[:s.offset + s.length // 2] + good[s.offset + s.length:]
        jb = _batch([small, bad])
        jb.out.fill_(77)
        jb.load([small, bad], jb.layout)
        jb.launch()
        fr = jb.frames()
        assert int(jb.status[1]) != 0 and int(jb.status[0]) == 0, k
        assert np.array_equal(fr[0].cpu().numpy(), JC.cv2_decode(small))
        assert int(fr[1].max()) == 0
    rng = np.random.default_rng(7)
    n_img = n_bad = 0
    for _ in range(32):
        a = bytearray(good)
        s = info.scans[int(rng.integers(0, len(info.scans)))]
        p = s.offset + int(rng.integers(0, s.length))
        v = a[p] ^ (1 << int(rng.integers(0, 8)))
        if a[p] == 0xFF or v == 0xFF or (p > 0 and a[p - 1] == 0xFF):
            continue                                           # keep the marker structure
        a[p] = v
        try:
            jb = _batch([bytes(a)])
        except jpeg.JpegError:
            continue
        st = int(jb.status[0])
        fr = jb.frames()[0]
        if st:
            assert int(fr.max()) == 0
            n_bad += 1
        else:
            n_img += 1
    torch.cuda.synchronize()
    assert n_img + n_bad >= 16 and n_bad > 0, (n_img, n_bad)   # flips reached the device, and some set status bits
    ok = jpeg.decode([good], max_scans=BIG)[0]                 # later batches still decode
    assert np.array_equal(ok.cpu().numpy(), JC.cv2_decode(good))


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


def _snapshot(bufs, mano):
    torch.cuda.synchronize()
    n = int(bufs.counts[2])
    snap = [bufs.counts.clone(), bufs.params_pred[:n].clone(), bufs.offsets_out[:n].clone(), mano["verts"][:n].clone(),
            mano["pj2d_org"][:n].clone()]
    if "track_id" in mano:
        snap.append(mano["track_id"][:n].clone())
    return snap


@pytest.mark.parametrize("tracked", [False, True], ids=["plain", "tracker"])
def test_jpeg_graph_replays_with_scripts_equal_eager(app, tracked):
    from acr_b200.ops import HandTracker
    from acr_b200.preprocess import preprocess_frames
    from acr.result_parser import ResultParser
    A = [PW.cv2_progressive(720, 1280, 90, "420", 0, "smooth"), JC.encode(17, 9, 100, "444", 1, "noisy"),
         PW.cv2_progressive(1080, 1920, 90, "444", 4, "smooth"),
         PW.multi_scan_sequential(JC.encode(37, 53, 90, "420", 0, "noisy"), [[0], [1, 2]])]
    B = [JC.encode(1080, 1920, 50, "440", 0, "noisy"), JC.encode(1, 1, 90, "420", 0, "smooth"),
         JC.encode(720, 1280, 100, "grey", 4, "smooth"), JC.encode(720, 1280, 90, "444", 0, "noisy")]
    C = [PW.pillow_progressive(45, 83, 80, 2), PW.cv2_progressive(17, 9, 90, "grey", 1), A[2], B[0]]
    mixes = [A, B, C, A[::-1]]
    coded = max(sum(jpeg.parse(b, BIG).scan_len for b in m) for m in mixes)
    frame_bytes = max(sum(jpeg.parse(b, BIG).H * jpeg.parse(b, BIG).W * 3 for b in m) for m in mixes)
    scans = max(len(jpeg.plan(m, max_scans=BIG)[0].scans) for m in mixes)
    K = ResultParser.hands_per_side()
    t_graph = HandTracker("cuda", K) if tracked else None
    t_eager = HandTracker("cuda", K) if tracked else None
    replay = app.capture_jpeg_graph(4, coded, frame_bytes, tracker=t_graph, max_scans=scans)

    def check(mix):
        img, offs = preprocess_frames([torch.from_numpy(JC.cv2_decode(b)).cuda() for b in mix])
        exp = _snapshot(*app.fused_forward(img, offs.cuda(), tracker=t_eager))
        got = _snapshot(*replay(mix))
        replay.jpeg.raise_on_status()
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            assert torch.equal(g, e)

    for mix in mixes[:2]:
        check(mix)
    many = [PW.cv2_progressive(17, 9, 90, "420", 0)] * 3 + [PW.cv2_progressive(7, 13, 90, "444", 0)]
    if len(jpeg.plan(many, max_scans=BIG)[0].scans) > scans:
        with pytest.raises(ValueError, match="capacity"):
            replay(many)
    for mix in mixes[2:]:
        check(mix)

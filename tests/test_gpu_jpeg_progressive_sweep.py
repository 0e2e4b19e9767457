"""GPU: the progressive and multi-scan sequential sweep of tests/test_cpu_jpeg_progressive_sweep.py on the device
(acr_b200_jpeg_decode_scans).

* every file (cv2 progressive at every (h, w) in jpeg_cases.SWEEP^2, sampling and RST interval 0 / 1 / 3; every
  writer script and table kind at sizes from {1, 7, 8, 9, 16, 17, 33}^2 with restart layouts from each scan's
  geometry and 0xFF fill bytes; multi-scan sequential files with per-scan restarts and fill bytes; grey frames with
  2x2 / 1x2 / 2x1 SOF sampling; medium frames with scans of more than 256 blocks; a frame with EOB runs of every
  length class) decodes equal to cv2.imdecode with status 0, in shuffled batches that mix the kinds with baseline
  files;
* its coefficients equal the device's coefficients of its baseline source (the same quantised coefficients, coded
  once as a single sequential scan), and, under 100 px, the numpy statement's;
* one batch of every kind, baseline files and a host-fallback file equals each file decoded alone, with scan
  capacity exactly the batch's scans and with spare (unused) scan descriptors.
"""
import time

import numpy as np
import pytest
import torch

from acr_b200 import jpeg
from tests import jpeg_cases as JC
from tests import jpeg_progressive_ref as PR
from tests import test_cpu_jpeg_progressive_sweep as SW

pytestmark = pytest.mark.gpu
CAP = 65535           # planning capacity: any batch here fits
SCANS_PER_BATCH = 6000


@pytest.fixture(scope="module")
def clock():
    t = time.perf_counter()
    yield
    print(f"\ntest_gpu_jpeg_progressive_sweep: {time.perf_counter() - t:.1f} s wall")


def corpus():
    """label -> (file, baseline source with the same coefficients)."""
    out = {k: v for k, v in SW.cv2_sweep().items()}
    for files in (SW.writer_sweep(), SW.grey_sampling_files(), SW.medium_files()):
        out.update({k: (b, src) for k, (b, _, src) in files.items()})
    out.update(SW.multi_sweep())
    b, _, src = SW.eob_classes_file()
    out["eob-classes"] = (b, src)
    return out


def _batches(files, labels):
    """Groups of labels in order, each under SCANS_PER_BATCH scans and 48 files (their sources ride along)."""
    group, scans = [], 0
    for n in labels:
        k = len(jpeg.parse(files[n][0], CAP).scans)
        if group and (scans + k > SCANS_PER_BATCH or len(group) == 48):
            yield group
            group, scans = [], 0
        group.append(n)
        scans += k
    if group:
        yield group


def _decode(bufs, max_scans=None, host_fallback=False):
    lay, fb = jpeg.plan(bufs, host_fallback, CAP)
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks,
                        max_scans=len(lay.scans) if max_scans is None else max_scans)
    jb.load(bufs, lay)
    jb.launch()
    jb.put_host_frames(fb)
    return jb


def test_sweep_equals_cv2_the_baseline_source_and_the_statement(clock):
    files = corpus()
    labels = list(files)
    np.random.default_rng(11).shuffle(labels)       # mixed groups: every kind next to every other
    bad = []
    n_stmt = 0
    for group in _batches(files, labels):
        bufs = [files[n][0] for n in group] + [files[n][1] for n in group]
        jb = _decode(bufs)
        fr = jb.frames()
        st = jb.status[:len(bufs)].cpu().numpy()
        for i, n in enumerate(group):
            b, src = files[n]
            j = len(group) + i
            if st[i] != 0 or st[j] != 0:
                bad.append((n, int(st[i]), int(st[j])))
                continue
            if not np.array_equal(fr[i].cpu().numpy(), JC.cv2_decode(b)):
                bad.append((n, "pixels"))
                continue
            # the component's own blocks: a one-component scan codes no MCU padding, which a baseline file does
            info = jpeg.parse(b, CAP)
            own = [(-(-info.comp_size(c)[1] // 8), -(-info.comp_size(c)[0] // 8)) for c in range(info.ncomp)]
            got = [g[:h, :w] for g, (h, w) in zip(jb.coefficients(i), own)]
            base = [g[:h, :w] for g, (h, w) in zip(jb.coefficients(j), own)]
            if len(base) != info.ncomp or not all(torch.equal(g, e) for g, e in zip(got, base)):
                bad.append((n, "coefficients != the baseline source's"))
                continue
            if max(info.H, info.W) < 100:
                n_stmt += 1
                exp = PR.coefficients(b, info)        # whole planes: the padding the scans skip stays zero
                if not all(np.array_equal(g.cpu().numpy(), e) for g, e in zip(jb.coefficients(i), exp)):
                    bad.append((n, "coefficients != the statement's"))
    assert not bad, (len(bad), bad[:8])
    assert n_stmt > 0.9 * len(files)


def _incomplete():
    b = SW.PW.cv2_progressive(17, 9, 90, "420", 0)
    last = jpeg.parse(b, CAP).scans[-1]
    return b[:b.rfind(b"\xff\xda", 0, last.offset)] + b"\xff\xd9"   # no last refinement: decoded on the host


def test_mixed_batch_equals_each_file_alone(clock):
    files = corpus()
    pick = {}
    for prefix in ("cv2-17x33-420-r3", "cv2-9x16-422-r1", "cv2-33x1-grey-r0"):
        pick[prefix] = files[prefix][0]
    for prefix in ("w-420-", "w-444-", "w-grey-", "ms-440-", "ms-422-", "grey2x2-", "grey2x1-", "m-422-", "m-grey-"):
        ks = [k for k in files if k.startswith(prefix) and ("-f1" in k or "-v2" in k or prefix[0] in "gm")]
        pick[ks[0]] = files[ks[0]][0]
    pick["eob-classes"] = files["eob-classes"][0]
    pick["baseline-420-r4"] = JC.encode(45, 83, 90, "420", 4, "noisy")
    pick["baseline-grey"] = JC.encode(17, 9, 50, "grey", 0, "smooth")
    pick["host-fallback"] = _incomplete()
    labels = list(pick)
    np.random.default_rng(2).shuffle(labels)
    bufs = [pick[n] for n in labels]
    need = len(jpeg.plan(bufs, True, CAP)[0].scans)
    alone = {n: jpeg.decode([pick[n]], host_fallback=True, max_scans=CAP)[0].cpu().numpy() for n in labels}
    for cap in (need, need + 37):
        jb = _decode(bufs, max_scans=cap, host_fallback=True)
        fr = jb.frames()
        jb.raise_on_status()
        for i, n in enumerate(labels):
            got = fr[i].cpu().numpy()
            assert np.array_equal(got, alone[n]), (cap, n)
            assert np.array_equal(got, JC.cv2_decode(pick[n])), (cap, n)

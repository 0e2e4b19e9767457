"""GPU: the device JPEG decoder (csrc/jpeg.cu) on streams other encoders write, byte for byte against cv2.imdecode.

* every writer variant (tests/jpeg_writer.py: per-component Huffman and quantisation tables with ids 0-3, codes of
  10-16 bits, 16-bit DQT with SOF1, restart intervals up to 65535, fill bytes before markers, a trailing RST, header
  variants), cv2 files with optimised tables, the committed Pillow files, every size of the small sweep in all
  samplings with and without restarts, and a 12 MP and a 24 MP frame: status 0 and cv2's bytes;
* the device's quantised coefficients equal oracle/jpeg_ref.coefficients on the writer variants;
* one mixed batch of every writer variant gives each file the bytes it gets alone;
* Pillow's RGB file raises JpegUnsupported, and decodes to cv2's pixels with host_fallback.
"""
import numpy as np
import pytest
import torch

from acr_b200 import jpeg
from tests import jpeg_cases as JC

pytestmark = pytest.mark.gpu


def _batch(bufs):
    """Decode one batch -> (JpegBatch, status per file as numpy)."""
    lay, _ = jpeg.plan(bufs)
    jb = jpeg.JpegBatch(len(bufs), lay.coded_bytes, lay.out_bytes, lay.chunks, lay.blocks)
    jb.out.fill_(77)
    jb.load(bufs, lay)
    jb.launch()
    return jb, jb.status[:len(bufs)].cpu().numpy()


def _check(files, per_batch=300):
    """Every file decodes with status 0 to cv2's bytes -> list of failures."""
    names = list(files)
    bad = []
    for k in range(0, len(names), per_batch):
        part = names[k:k + per_batch]
        bufs = [files[n] for n in part]
        jb, st = _batch(bufs)
        for n, b, s, fr in zip(part, bufs, st, jb.frames()):
            if s != 0:
                bad.append(f"{n}: status {int(s)}")
            elif not np.array_equal(fr.cpu().numpy(), JC.cv2_decode(b)):
                bad.append(f"{n}: pixels differ")
    return bad


def test_writer_variants_equal_cv2():
    files = {k: b for k, (b, _) in JC.writer_files().items()}
    bad = _check(files)
    assert not bad, f"{len(bad)} of {len(files)}: {bad[:8]}"


def test_cv2_optimized_and_pillow_files_equal_cv2():
    files = dict(JC.cv2_optimized())
    files.update({k: b for k, b in JC.pillow_files().items() if "rgb" not in k})
    bad = _check(files)
    assert not bad, f"{len(bad)} of {len(files)}: {bad[:8]}"


def test_small_sweep_equals_cv2():
    cases = JC.small_sweep()
    files = {c: JC.encode(*c) for c in cases}
    bad = _check(files, per_batch=400)
    assert not bad, f"{len(bad)} of {len(files)}: {bad[:8]}"


def test_large_frames_equal_cv2():
    files = JC.large_files()
    assert max(jpeg.parse(b).n_chunks for b in files.values()) > 12000
    bad = _check(files)
    assert not bad, bad


def test_coefficients_equal_the_oracle_on_the_writer_variants():
    from oracle import jpeg_ref
    files = {k: b for k, (b, _) in JC.writer_files().items()}
    names = list(files)
    jb, st = _batch([files[n] for n in names])
    assert not st.any(), [names[i] for i in np.flatnonzero(st)][:8]
    bad = []
    for i, n in enumerate(names):
        exp = jpeg_ref.coefficients(files[n])
        got = jb.coefficients(i)
        if len(got) != len(exp) or not all(np.array_equal(g.cpu().numpy(), e) for g, e in zip(got, exp)):
            bad.append(n)
    assert not bad, f"{len(bad)} of {len(names)}: {bad[:8]}"


def test_mixed_batch_of_every_variant_equals_each_file_alone():
    files = {k: b for k, (b, _) in JC.writer_files().items()}
    files.update({k: b for k, b in JC.pillow_files().items() if "rgb" not in k})
    names = list(files)
    order = np.random.default_rng(7).permutation(len(names))
    mixed = jpeg.decode([files[names[i]] for i in order])
    for j, i in enumerate(order):
        alone = jpeg.decode([files[names[i]]])[0]
        assert torch.equal(mixed[j], alone), names[i]


def test_rgb_file_is_unsupported_and_falls_back_to_cv2():
    files = JC.pillow_files()
    rgb = files["pillow-rgb_keep_rgb"]
    other = files["pillow-sof1_q16_420"]
    with pytest.raises(jpeg.JpegUnsupported, match="RGB"):
        jpeg.decode([other, rgb])
    out = jpeg.decode([other, rgb], host_fallback=True)
    assert np.array_equal(out[0].cpu().numpy(), JC.cv2_decode(other))
    assert np.array_equal(out[1].cpu().numpy(), JC.cv2_decode(rgb))

"""Seeded JPEG test files for the device decoder (tests/test_cpu_jpeg.py, tests/test_gpu_jpeg.py): cv2.imencode of
smooth and noisy BGR arrays over qualities, samplings, restart intervals and sizes.  The conformance files
(tests/test_*_jpeg_conformance.py) add a small-size sweep, cv2 files with optimised tables, 12 and 24 MP frames,
the committed Pillow files and the writer variants of tests/jpeg_writer.py."""
import functools

import numpy as np

SIZES = [(1, 1), (7, 13), (17, 9), (720, 1280), (1080, 1920)]
QUALITIES = [50, 90, 100]
SAMPLINGS = ["444", "422", "420", "440", "grey"]
RESTARTS = [0, 1, 4]
CONTENTS = ["smooth", "noisy"]


def image(h, w, content, seed=0):
    if content == "noisy":
        return np.random.default_rng(seed + 7 * h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:h, :w].astype(np.float64)
    r = np.hypot(yy - h / 3, xx - w / 2)
    b = 128 + 100 * np.sin(xx / max(w, 1) * 6.0 + yy / max(h, 1) * 2.0)
    g = 128 + 90 * np.cos(r / max(h, w, 1) * 9.0)
    rr = (xx + 2 * yy) * 255.0 / max(w + 2 * h, 1)
    return np.clip(np.stack([b, g, rr], 2), 0, 255).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def encode(h, w, q, sampling, rst, content, progressive=False) -> bytes:
    import cv2
    img = image(h, w, content)
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if progressive:
        params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if sampling == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{sampling}")]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def matrix(sizes=SIZES):
    """Every (h, w, quality, sampling, restart, content) of the test matrix."""
    return [(h, w, q, s, r, c) for (h, w) in sizes for q in QUALITIES for s in SAMPLINGS for r in RESTARTS
            for c in CONTENTS]


def cv2_decode(buf: bytes):
    import cv2
    return cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)


# ---- conformance files (tests/test_cpu_jpeg_conformance.py, tests/test_gpu_jpeg_conformance.py) --------------------
SWEEP = list(range(1, 19)) + [31, 32, 33]     # every partial MCU, chroma planes 1..3 samples on both sides


def small_sweep():
    """Every (h, w) with h, w in SWEEP, every sampling, no restarts and RST interval 1, noisy content."""
    return [(h, w, 90, s, r, "noisy") for h in SWEEP for w in SWEEP for s in SAMPLINGS for r in (0, 1)]


@functools.lru_cache(maxsize=None)
def cv2_optimized():
    """cv2 with optimised Huffman tables and separate luma / chroma qualities, every sampling and a few sizes."""
    import cv2
    out = {}
    for h, w in ((1, 1), (5, 3), (23, 37), (121, 203)):
        for s in SAMPLINGS:
            for ql, qc in ((95, 40), (60, 90)):
                img = image(h, w, "noisy", seed=ql)
                params = [cv2.IMWRITE_JPEG_OPTIMIZE, 1, cv2.IMWRITE_JPEG_LUMA_QUALITY, ql,
                          cv2.IMWRITE_JPEG_CHROMA_QUALITY, qc]
                if s == "grey":
                    img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
                else:
                    params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{s}")]
                ok, buf = cv2.imencode(".jpg", img, params)
                assert ok
                out[f"cv2opt-{h}x{w}-{s}-l{ql}c{qc}"] = buf.tobytes()
    return out


def pillow_files():
    """name -> bytes of the committed Pillow files (tests/golden/make_jpeg_golden.py)."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_pillow_golden.npz"))
    return {f"pillow-{k}": z[k].tobytes() for k in z.files}


# writer sources: cv2 files whose coefficients the writer codes again
WRITER_SOURCES = {"420": (96, 160, 90, "420", 0, "noisy"), "422": (45, 83, 75, "422", 0, "noisy"),
                  "444": (40, 51, 90, "444", 0, "noisy"), "440": (37, 26, 95, "440", 0, "noisy"),
                  "grey": (35, 50, 90, "grey", 0, "noisy")}


def _lower_quant(q, c):
    """Component c's table scaled down (entries stay <= the source's, so no dequantised value exceeds an encoder's)
    and different for every component."""
    f = (0.8, 0.6, 0.45)[c]
    return np.maximum(1, np.floor(q.astype(np.float64) * f)).astype(np.uint16)


def writer_variants(name):
    """label -> jpeg_writer.write keyword arguments for the source WRITER_SOURCES[name]."""
    import tests.jpeg_writer as JW
    src = JW.source(encode(*WRITER_SOURCES[name]))
    nc = src.ncomp
    mx, my = src.mcus
    ids = lambda *v: list(v[:nc])
    out = {"source-tables": {}}
    for t in ("optimal", "long", "short", "skewed"):
        out[f"tables-{t}"] = dict(tables=t, dc_ids=ids(1, 2, 3), ac_ids=ids(2, 3, 0))
    q = np.stack([_lower_quant(src.quant[c], c) for c in range(nc)])
    out["quant8-per-comp"] = dict(quant=q, q_ids=ids(3, 2, 0))
    out["quant16-sof1"] = dict(quant=q, qprec=(1, 1, 1), q_ids=ids(2, 0, 1))
    out["quant16-luma-only"] = dict(quant=q, qprec=(1, 0, 0), q_ids=ids(0, 1, 3))
    rsts = sorted({1, 2, 3, 5, 7, mx, mx + 1, mx * my, 65535})
    for k, r in enumerate(rsts):
        out[f"dri{r}"] = dict(restart=r, tables=("optimal", "long", "source")[k % 3], dc_ids=ids(0, 1, 2),
                              ac_ids=ids(0, 1, 2))
        out[f"dri{r}-fill"] = dict(restart=r, fill=(1, 2, 3), tables=("skewed", "short", "optimal")[k % 3],
                                   dc_ids=ids(3, 1, 2), ac_ids=ids(1, 3, 2))
    out["dri0-explicit"] = dict(dri=[0])
    out["dri-twice"] = dict(restart=3, dri=[7, 3], fill=(2,))
    out["dri-twice-to-0"] = dict(restart=0, dri=[5, 0])
    out["trailing-rst"] = dict(restart=mx, trailing_rst=True)
    out["trailing-rst-fill"] = dict(restart=1, trailing_rst=True, fill=(3, 1), tables="long", dc_ids=ids(0, 1, 2),
                                    ac_ids=ids(0, 1, 2))
    out["fill-eoi-only"] = dict(fill=(2,))
    out["one-segment"] = dict(one_segment=True, tables="optimal", quant=q, dc_ids=ids(0, 1, 2), ac_ids=ids(0, 1, 2),
                              q_ids=ids(0, 1, 2))
    out["redefined"] = dict(redefine=True, tables="skewed", quant=q, dc_ids=ids(3, 2, 1), ac_ids=ids(3, 2, 1),
                            q_ids=ids(3, 2, 1))
    for cid in ((0, 1, 2), (7, 8, 9)):
        for app in ("jfif", "exif", "adobe", "none"):
            out[f"ids{''.join(map(str, cid))}-{app}"] = dict(comp_ids=cid, app=app)
    out["ids123-none-com-app2"] = dict(app="none", com=True, app2=True, restart=2)
    out["exif-com-app2"] = dict(app="exif", com=True, app2=True)
    if nc == 1:
        out["grey-2x2"] = dict(grey_hv=(2, 2))
        out["grey-2x2-rst"] = dict(grey_hv=(2, 2), restart=mx, fill=(1,))
    return src, out


@functools.lru_cache(maxsize=None)
def writer_files():
    """label -> (bytes, whether its quantisation tables differ from the source's) over every writer source."""
    import tests.jpeg_writer as JW
    out = {}
    for name in WRITER_SOURCES:
        src, variants = writer_variants(name)
        for label, kw in variants.items():
            out[f"writer-{name}-{label}"] = (JW.write(src, **kw), "quant" in kw)
    return out


def large_files():
    """A 12 MP camera layout (4:2:0 q95, EXIF APP1, one restart interval per MCU row) and a 24 MP 4:2:2 q90 file."""
    import cv2
    out = {}
    for h, w, s, q, exif in ((3000, 4000, "420", 95, True), (4000, 6000, "422", 90, False)):
        rng = np.random.default_rng(h)
        img = np.clip(image(h, w, "smooth").astype(np.int16) + rng.integers(-6, 7, (h, w, 3), dtype=np.int16),
                      0, 255).astype(np.uint8)
        fx = 2
        mcus_x = -(-w // (8 * fx))
        params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                  getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{s}")]
        if exif:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, mcus_x]
        ok, buf = cv2.imencode(".jpg", img, params)
        assert ok
        b = buf.tobytes()
        if exif:
            from tests.jpeg_writer import EXIF
            b = b[:2] + EXIF + b[2:]
        out[f"large-{h}x{w}-{s}-q{q}"] = b
    return out

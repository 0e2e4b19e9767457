"""Seeded JPEG test files for the device decoder (tests/test_cpu_jpeg.py, tests/test_gpu_jpeg.py): cv2.imencode of
smooth and noisy BGR arrays over qualities, samplings, restart intervals and sizes."""
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

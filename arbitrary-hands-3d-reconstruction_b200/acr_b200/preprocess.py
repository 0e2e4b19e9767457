"""Host side of the device pre-processing (csrc/preprocess.cu): padding geometry, offsets vector and the
fixed-point cubic tables, built exactly like the third-party code the reference calls.

* padding split: imgaug 0.4.0 ``compute_paddings_to_reach_aspect_ratio`` (absent from this image; restated
  from its published source): a landscape frame gets floor(diff/2) rows on top and ceil(diff/2) below, a
  portrait frame floor(diff/2) columns left and ceil(diff/2) right.
* offsets vector: ``[padded_h, padded_w, crop t,r,b,l (= 0), pad t,r,b,l]`` (acr/utils.py:1301,1311).
* cubic tables: opencv-python ``resize.cpp`` (INTER_CUBIC, 8-bit): ``fx = (d+0.5)*scale-0.5`` in float32,
  ``A = -0.75``, coefficients ``round(c*2048)`` as int16.
"""
from __future__ import annotations

from functools import lru_cache
from typing import Tuple

import numpy as np
import torch

from . import lib as L


def paddings_to_square(h: int, w: int) -> Tuple[int, int, int, int]:
    """(top, right, bottom, left) that make an (h, w) frame square."""
    top = right = bottom = left = 0
    if w > h:
        d = w - h
        top, bottom = d // 2, d - d // 2
    elif h > w:
        d = h - w
        left, right = d // 2, d - d // 2
    return top, right, bottom, left


def offsets_vector(h: int, w: int) -> np.ndarray:
    t, r, b, l = paddings_to_square(h, w)
    return np.array([h + t + b, w + l + r, 0, 0, 0, 0, t, r, b, l], np.float32)


@lru_cache(maxsize=32)
def cubic_tables(n_src: int, n_dst: int) -> Tuple[np.ndarray, np.ndarray]:
    """-> (coef (n_dst,4) int16, ofs (n_dst) int32): taps ofs-1 .. ofs+2 of the source axis."""
    scale = np.float64(n_src) / n_dst
    A = np.float32(-0.75)
    coef = np.zeros((n_dst, 4), np.int16)
    ofs = np.zeros(n_dst, np.int32)
    for d in range(n_dst):
        fx = np.float32((d + 0.5) * scale - 0.5)
        s = int(np.floor(fx))
        x = np.float32(fx - s)
        c = np.zeros(4, np.float32)
        c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A
        c[1] = ((A + 2) * x - (A + 3)) * x * x + 1
        c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1
        c[3] = np.float32(1.0) - c[0] - c[1] - c[2]
        ofs[d] = s
        coef[d] = np.rint(c * np.float32(2048)).astype(np.int16)
    return coef, ofs


_dev_tables = {}


def preprocess_frames(frames_bgr, input_size: int = 512):
    """(n,H,W,3) uint8 BGR CUDA tensor -> ((n,S,S,3) uint8 RGB CUDA tensor, (n,10) offsets).

    ``frames_bgr`` may also be a list of (H_i, W_i, 3) uint8 BGR frames of any sizes: numpy arrays or CPU tensors
    (one pinned staging buffer, one H2D copy, then the current CUDA device), or CUDA tensors of one device (packed
    with one ``torch.cat``).  They are resized in one launch (``RaggedFrames``); the result is the same as that of
    each frame on its own.  The offsets are a CPU tensor either way."""
    if isinstance(frames_bgr, (list, tuple)):
        desc, offsets, total = ragged_layout(frames_bgr)
        dev = next((f.device for f in frames_bgr if isinstance(f, torch.Tensor) and f.is_cuda), None)
        rf = RaggedFrames(len(frames_bgr), total, dev, input_size)
        rf.load(frames_bgr)
        out, _ = rf.launch(with_offsets=False)
        return out, torch.from_numpy(offsets)
    L.require_cuda(frames_bgr)
    assert frames_bgr.dtype == torch.uint8 and frames_bgr.dim() == 4 and frames_bgr.shape[-1] == 3
    frames_bgr = frames_bgr.contiguous()
    n, H, W, _ = frames_bgr.shape
    t, r, b, l = paddings_to_square(H, W)
    side = max(H, W)
    key = (side, input_size, str(frames_bgr.device))
    if key not in _dev_tables:
        coef, ofs = cubic_tables(side, input_size)
        _dev_tables[key] = (torch.from_numpy(coef).to(frames_bgr.device), torch.from_numpy(ofs).to(frames_bgr.device))
    coef, ofs = _dev_tables[key]
    out = torch.empty(n, input_size, input_size, 3, dtype=torch.uint8, device=frames_bgr.device)
    L.check(L.load().acr_b200_preprocess(L.ptr(frames_bgr), n, H, W, L.ptr(coef), L.ptr(ofs), L.ptr(coef), L.ptr(ofs),
                                         side, t, l, input_size, L.ptr(out), L.current_stream()), "preprocess")
    offsets = torch.from_numpy(np.tile(offsets_vector(H, W), (n, 1)))
    return out, offsets


# ---- ragged batches: frames of any sizes in one launch ------------------------------------------------------------
# acr_b200_frame (include/acr_b200.h): where a frame's bytes start in the packed buffer and its padded square
FRAME_DTYPE = np.dtype([("offset", "<i8"), ("H", "<i4"), ("W", "<i4"), ("side", "<i4"), ("pad_t", "<i4"),
                        ("pad_l", "<i4"), ("reserved", "<i4")])
assert FRAME_DTYPE.itemsize == 32


def _frame_hw(i: int, f) -> Tuple[int, int]:
    if isinstance(f, np.ndarray):
        is_u8 = f.dtype == np.uint8
    elif isinstance(f, torch.Tensor):
        is_u8 = f.dtype == torch.uint8
    else:
        raise TypeError(f"frame {i}: expected a numpy array or a torch tensor, got {type(f).__name__}")
    if not is_u8:
        raise TypeError(f"frame {i}: expected uint8 BGR, got {f.dtype}")
    if f.ndim != 3 or f.shape[2] != 3:
        raise ValueError(f"frame {i}: expected shape (H, W, 3), got {tuple(f.shape)}")
    if f.shape[0] < 1 or f.shape[1] < 1:
        raise ValueError(f"frame {i}: empty frame of shape {tuple(f.shape)}")
    return int(f.shape[0]), int(f.shape[1])


def shapes_layout(shapes) -> Tuple[np.ndarray, np.ndarray, int]:
    """``ragged_layout`` of frames given by their (H, W) only."""
    desc = np.zeros(len(shapes), FRAME_DTYPE)
    offsets = np.zeros((len(shapes), 10), np.float32)
    pos = 0
    for i, (H, W) in enumerate(shapes):
        t, r, b, l = paddings_to_square(H, W)
        desc[i] = (pos, H, W, max(H, W), t, l, 0)
        offsets[i] = offsets_vector(H, W)
        pos += H * W * 3
    return desc, offsets, pos


def ragged_layout(frames) -> Tuple[np.ndarray, np.ndarray, int]:
    """Layout of a list of (H_i, W_i, 3) uint8 frames packed back to back -> (descriptors (n,) FRAME_DTYPE,
    offsets vectors (n,10) float32, packed bytes).  Frame i starts at the sum of H_j * W_j * 3 over j < i.  Raises
    TypeError / ValueError for anything that is not such a frame, and for an empty list."""
    if len(frames) == 0:
        raise ValueError("a ragged batch needs at least one frame")
    desc = np.zeros(len(frames), FRAME_DTYPE)
    offsets = np.zeros((len(frames), 10), np.float32)
    pos = 0
    for i, f in enumerate(frames):
        H, W = _frame_hw(i, f)
        t, r, b, l = paddings_to_square(H, W)
        desc[i] = (pos, H, W, max(H, W), t, l, 0)
        offsets[i] = offsets_vector(H, W)
        pos += H * W * 3
    return desc, offsets, pos


def check_ragged(frames, max_frames: int, max_bytes: int, exact: bool = False):
    """``ragged_layout`` plus the checks of ``RaggedFrames.load`` against a capacity of ``max_frames`` frames and
    ``max_bytes`` packed bytes (exactly ``max_frames`` frames when ``exact``) -> (descriptors, offsets, packed bytes,
    whether the frames are on the host).  Raises TypeError / ValueError; touches no device."""
    desc, offsets, total = ragged_layout(frames)
    n = len(frames)
    if exact and n != max_frames:
        raise ValueError(f"this ragged batch takes exactly {max_frames} frames, got {n}")
    if n > max_frames:
        raise ValueError(f"{n} frames exceed the capacity of {max_frames}")
    if total > max_bytes:
        raise ValueError(f"the frames need {total} bytes, over the capacity of {max_bytes}")
    on_dev = [isinstance(f, torch.Tensor) and f.is_cuda for f in frames]
    if any(on_dev) and not all(on_dev):
        raise TypeError("a ragged batch takes host frames or CUDA frames, not a mix")
    return desc, offsets, total, not on_dev[0]


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class RaggedFrames:
    """Device buffers of one ragged batch: at most ``max_frames`` frames of any sizes and ``max_bytes`` bytes in all.

    One device buffer holds the acr_b200_frame descriptors, then each frame's square side (the input of
    acr_b200_cubic_tables), then the frames back to back, so one H2D copy from one pinned staging buffer carries a
    batch of host frames with its descriptors.  ``load`` fills the buffers on the current stream, ``launch`` enqueues
    the tables and the resize.  The buffers never move, so a CUDA graph can capture ``launch`` once and every replay
    after a ``load`` resizes the frames loaded last; ``exact=True`` (the graph form) then demands exactly
    ``max_frames`` frames per load.  Capacity and frame errors are raised by ``load`` before anything is written."""

    def __init__(self, max_frames: int, max_bytes: int, device=None, input_size: int = 512, exact: bool = False):
        if max_frames < 1 or max_bytes < 3 * max_frames:
            raise ValueError(f"RaggedFrames: need max_frames >= 1 and max_bytes >= 3 * max_frames "
                             f"(got {max_frames}, {max_bytes})")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.max_frames, self.max_bytes, self.input_size, self.exact = max_frames, max_bytes, input_size, exact
        self.meta_bytes = _round_up(max_frames * (FRAME_DTYPE.itemsize + 4), 256)
        S, dev = input_size, self.device
        self.buf = torch.empty(self.meta_bytes + max_bytes, dtype=torch.uint8, device=dev)
        self.desc = self.buf[:max_frames * FRAME_DTYPE.itemsize]
        self.sides = self.buf[self.desc.numel():self.desc.numel() + 4 * max_frames].view(torch.int32)
        self.packed = self.buf[self.meta_bytes:]
        self.coef = torch.empty(max_frames, S, 4, dtype=torch.int16, device=dev)
        self.ofs = torch.empty(max_frames, S, dtype=torch.int32, device=dev)
        self.out = torch.empty(max_frames, S, S, 3, dtype=torch.uint8, device=dev)
        self.offsets = torch.empty(max_frames, 10, dtype=torch.float32, device=dev)
        self._stage = None        # pinned; grown to meta + max_bytes on the first host-frame load
        self._copied = None       # event after the last copy out of _stage
        self.n = 0

    def _staging(self, nbytes: int) -> torch.Tensor:
        if self._copied is not None:
            self._copied.synchronize()      # the previous H2D read of the staging buffer is done
        if self._stage is None or self._stage.numel() < nbytes:
            size = self.meta_bytes if nbytes <= self.meta_bytes else self.meta_bytes + self.max_bytes
            self._stage = torch.empty(size, dtype=torch.uint8, pin_memory=True)
        return self._stage

    def check(self, frames):
        """Every check of ``load`` -> ``check_ragged``'s (descriptors, offsets, packed bytes, whether the frames are
        on the host).  Raises TypeError / ValueError; touches no device."""
        desc, offsets, total, host = check_ragged(frames, self.max_frames, self.max_bytes, self.exact)
        if not host and any(f.device != self.device for f in frames):
            raise ValueError(f"CUDA frames must live on {self.device}")
        return desc, offsets, total, host

    def load(self, frames) -> int:
        """Copy a list of (H, W, 3) uint8 BGR frames (numpy arrays or CPU tensors, or CUDA tensors on this device;
        not a mix of host and device frames) into the buffers, on the current stream.  Returns the frame count."""
        desc, _, total, host = self.check(frames)
        n = len(frames)
        stage = self._staging(self.meta_bytes + (total if host else 0))
        np_stage = stage.numpy()
        np_stage[:n * FRAME_DTYPE.itemsize] = desc.view(np.uint8)
        d0 = self.desc.numel()
        np_stage[d0:d0 + 4 * n] = desc["side"].astype(np.int32).view(np.uint8)
        if host:
            for f, d in zip(frames, desc):
                o = self.meta_bytes + int(d["offset"])
                dst = np_stage[o:o + int(d["H"]) * int(d["W"]) * 3].reshape(int(d["H"]), int(d["W"]), 3)
                np.copyto(dst, f.numpy() if isinstance(f, torch.Tensor) else f)
        nbytes = self.meta_bytes + (total if host else 0)
        with torch.cuda.device(self.device):
            self.buf[:nbytes].copy_(stage[:nbytes], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
            if not host:
                torch.cat([f.reshape(-1) for f in frames], out=self.packed[:total])
        self.n = n
        return n

    def load_shapes(self, shapes) -> int:
        """Like ``load`` for frames that are already packed in ``self.packed`` (written there by the device, e.g. by
        the JPEG decoder): copies only the descriptors of frames of the given (H, W), on the current stream."""
        if len(shapes) == 0:
            raise ValueError("a ragged batch needs at least one frame")
        desc, _, total = shapes_layout(shapes)
        n = len(shapes)
        if self.exact and n != self.max_frames:
            raise ValueError(f"this ragged batch takes exactly {self.max_frames} frames, got {n}")
        if n > self.max_frames or total > self.max_bytes:
            raise ValueError(f"{n} frames of {total} bytes exceed the capacity of {self.max_frames} frames / "
                             f"{self.max_bytes} bytes")
        stage = self._staging(self.meta_bytes)
        np_stage = stage.numpy()
        np_stage[:n * FRAME_DTYPE.itemsize] = desc.view(np.uint8)
        d0 = self.desc.numel()
        np_stage[d0:d0 + 4 * n] = desc["side"].astype(np.int32).view(np.uint8)
        with torch.cuda.device(self.device):
            self.buf[:self.meta_bytes].copy_(stage[:self.meta_bytes], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
        self.n = n
        return n

    def launch(self, with_offsets: bool = True):
        """Enqueue acr_b200_cubic_tables and acr_b200_preprocess_ragged for the loaded frames on the current stream
        -> ((n,S,S,3) uint8 RGB, (n,10) float32 offsets on the device, or None without ``with_offsets``)."""
        n, S = self.n, self.input_size
        if n == 0:
            raise ValueError("RaggedFrames.launch before load")
        lib = L.load()
        with L.on(self.device):
            stream = L.current_stream(self.device)
            L.check(lib.acr_b200_cubic_tables(L.ptr(self.sides), n, S, L.ptr(self.coef), L.ptr(self.ofs), stream),
                    "cubic_tables")
            L.check(lib.acr_b200_preprocess_ragged(L.ptr(self.packed), self.max_bytes, L.ptr(self.desc), n,
                                                   L.ptr(self.coef), L.ptr(self.ofs), S, L.ptr(self.out),
                                                   L.ptr(self.offsets) if with_offsets else None, stream),
                    "preprocess_ragged")
        return self.out[:n], (self.offsets[:n] if with_offsets else None)

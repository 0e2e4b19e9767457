"""Drop-in application wrapper ``acr.main.ACR`` (reference: /root/reference/acr/main.py:24-141),
hot path only: model -> parse -> MANO.  Rendering / visualisation / CLI loops are out of scope."""
from __future__ import annotations

import inspect
from typing import Callable, NamedTuple

import torch
import torch.nn as nn

from acr.config import args
from acr.mano_wrapper import MANOWrapper
from acr.model import ACR as ACR_v1
from acr.utils import justify_detection_state, load_model


def _check_hands_per_side(K):
    """A captured graph's parse and MANO launches are sized for the K it was captured with."""
    from acr.result_parser import ResultParser
    now = ResultParser.hands_per_side()
    if now != K:
        raise ValueError(f"this graph was captured with max_hands_per_side={K}, but it is now {now}: capture it again")


def _check_tracker(tracker, K):
    if tracker is not None and tracker.K != K:
        raise ValueError(f"this tracker is built for K={tracker.K}, but max_hands_per_side is {K}")


def _stream_buffers(tracker, batch, dev):
    """Static (B,) int32 stream ids and begin flags of a graph captured with a multi-stream tracker, else None."""
    if tracker is None or tracker.streams == 1:
        return None
    return (torch.zeros(batch, dtype=torch.int32, device=dev), torch.zeros(batch, dtype=torch.int32, device=dev))


def _check_streams(static, stream_ids, stream_begin):
    """A replay's stream ids / begin flags as tensors (stream_begin may stay None), checked against the graph's."""
    shape = tuple(static[0].shape)
    ids, begin = (None if v is None else torch.as_tensor(v) for v in (stream_ids, stream_begin))
    for name, t in (("stream_ids", ids), ("stream_begin", begin)):
        if t is not None and tuple(t.shape) != shape:
            raise ValueError(f"{name} must have shape {shape}, got {tuple(t.shape)}")
    if ids is None:
        raise ValueError("this graph tracks several streams: replay needs stream_ids, the stream slot of each frame")
    return ids, begin


def _check_copy(name, src, dst):
    """Raise unless ``dst.copy_(src)`` takes ``src``: a tensor whose shape broadcasts to ``dst``'s."""
    if not isinstance(src, torch.Tensor):
        raise TypeError(f"{name} must be a tensor, got {type(src).__name__}")
    if src.shape != dst.shape and (src.dim() > dst.dim() or
                                   any(s not in (1, d) for s, d in zip(reversed(src.shape), reversed(dst.shape)))):
        raise ValueError(f"{name} of shape {tuple(src.shape)} does not broadcast to the graph's {tuple(dst.shape)}")


class _InputStage(NamedTuple):
    """How a captured graph gets its frames.  ``check(*inputs)`` runs every check of a replay's inputs and writes
    nothing -> (what ``load`` takes, the frames' (B,10) host offsets rows for the part labels, or None when the
    offsets are on the device or the graph has no labels);
    ``load`` copies them into the graph's buffers; ``enqueue()`` launches the input kernels -> (frames, offsets) on the
    device, as ``fused_forward`` takes them; ``attrs`` are the replay's attributes of this input."""
    check: Callable
    load: Callable
    enqueue: Callable
    attrs: dict


def _label_buffer(part_labels, batch, dev, default_capacity):
    """The PartLabels of a captured graph: ``part_labels`` None / False = no labels, True = the default capacity, an
    int = that capacity in label bytes (pixels)."""
    if part_labels is None or part_labels is False:
        return None
    if part_labels is True:
        if default_capacity is None:
            raise ValueError("capture_graph(part_labels=...) takes the label capacity in pixels (the frames' "
                             "H*W summed over the batch), not True")
        part_labels = default_capacity
    from acr_b200 import ops as _ops
    return _ops.PartLabels(int(part_labels), batch, dev)


def _device_ints(v, B, dev, name):
    if v is None:
        return None
    t = torch.as_tensor(v)
    if tuple(t.shape) != (B,):
        raise ValueError(f"{name} must have shape ({B},), got {tuple(t.shape)}")
    return t.to(device=dev, dtype=torch.int32).contiguous()


class ACR(nn.Module):
    def __init__(self, args_set=None, state_dict=None, mano_assets=None):
        super().__init__()
        self.demo_cfg = {'mode': 'parsing', 'calc_loss': False}
        cfg = vars(args() if args_set is None else args_set)
        for k, v in cfg.items():
            setattr(self, k, v)
        self._build_model_(state_dict, mano_assets)

    def _build_model_(self, state_dict, mano_assets):
        model = ACR_v1().eval()
        if state_dict is not None:
            model.load_state_dict(state_dict, strict=True)
        else:
            model = load_model(self.model_path, model, prefix='module.', drop_prefix='', fix_loaded=False)
        self.model = model.cuda()
        self.mano_regression = MANOWrapper(mano_assets).cuda()

    def _track_results(self, outputs):
        """``track_hands``: the rows of this batch through the device tracker, which also filters poses / betas per
        track when ``temporal_optimization`` is on; sets outputs['track_id'].  With ``track_streams`` = 1 the batch
        is B consecutive frames of one stream; with more, meta_data['stream_ids'] gives each image's stream slot
        (batch_forward's ``stream_ids``), the frames of a stream in batch order, and a track is keyed by (stream,
        id)."""
        from acr.result_parser import ResultParser
        from acr_b200 import ops as _ops
        K = ResultParser.hands_per_side()
        S = int(getattr(self, 'track_streams', 1))
        meta = outputs['meta_data']
        bids = meta.get('batch_ids')
        if bids is None:
            raise ValueError("track_hands needs meta_data['batch_ids'] (batch_forward sets arange(B))")
        bids = torch.as_tensor(bids).flatten().cpu()
        B = int(bids.numel())
        pd = outputs['params_dict']
        dev = pd['poses'].device
        img = outputs['reorganize_idx']
        sid = sbeg = None
        if S == 1:
            if not torch.equal(bids, torch.arange(B, dtype=bids.dtype)):
                raise ValueError("track_hands treats the batch as consecutive frames of one stream: batch_ids must be "
                                 "arange(B)")
        else:
            if meta.get('stream_ids') is None:
                raise ValueError(f"track_streams={S}: track_hands needs meta_data['stream_ids'] (batch_forward's "
                                 "stream_ids), the stream slot of each image")
            if torch.unique(bids).numel() != B:
                raise ValueError("track_hands with several streams needs distinct batch_ids, one per image")
            # the rows carry batch ids; the tracker wants each row's position in the batch
            pos = torch.full((int(bids.max()) + 1,), -1, dtype=torch.int64)
            pos[bids.long()] = torch.arange(B)
            img = pos.to(dev)[torch.as_tensor(img, device=dev).long()]
            sid = _device_ints(meta['stream_ids'], B, dev, 'stream_ids')
            sbeg = _device_ints(meta.get('stream_begin'), B, dev, 'stream_begin')
        smooth = float(self.smooth_coeff) if getattr(self, 'temporal_optimization', False) else None
        cfg = (K, int(self.track_gate), int(self.track_max_missed), smooth, S)
        t = getattr(self, '_hand_tracker', None)
        if t is None or (t.K, t.gate, t.max_missed, t.smooth_coeff, t.streams) != cfg:  # new settings: new tracks
            t = self._hand_tracker = _ops.HandTracker(dev, *cfg)
        n = pd['poses'].shape[0]
        cen = torch.cat([outputs['l_centers_pred'], outputs['r_centers_pred']]).to(dev)     # (x, y) per row
        i32 = lambda v: v.to(device=dev, dtype=torch.int32)
        row_src = torch.stack([i32(img), i32(outputs['output_hand_type']),
                               i32(cen[:, 1] * 64 + cen[:, 0]), torch.zeros(n, dtype=torch.int32, device=dev)],
                              1).contiguous()
        poses, betas = pd['poses'].contiguous(), pd['betas'].contiguous()
        ids = _ops.track_rows(t, B, row_src, outputs['detection_flag'].float().contiguous(), poses, betas,
                              frame_stream=sid, frame_begin=sbeg)
        pd['poses'], pd['betas'] = poses, betas
        outputs['track_id'] = ids[:n].clone()

    @torch.no_grad()
    def process_results(self, outputs):
        if getattr(self, 'track_hands', False):
            self._track_results(outputs)
        # temporal optimisation (acr/main.py:69-83): OneEuro filters on poses / betas, one bank per hand type,
        # applied between parse and MANO -- here the device tracker at K = 1 with the gate open and no miss limit,
        # whose one track per side is that bank
        elif getattr(self, 'temporal_optimization', False):
            from acr.result_parser import ResultParser
            if ResultParser.hands_per_side() > 1:
                raise ValueError("temporal_optimization needs max_hands_per_side=1: the filter banks are per hand type, "
                                 "and several hands of one side are not tracked across frames")
            from acr_b200 import ops as _ops
            pd = outputs['params_dict']
            assert len(pd['poses']) == 2, 'temporal smoothing streams one frame (two hand slots) at a time'
            dev = pd['poses'].device
            if getattr(self, '_one_euro', None) is None:
                self._one_euro = _ops.HandTracker(dev, 1, _ops.TRACK_GATE_OPEN, _ops.TRACK_NO_MISS_LIMIT)
            self._one_euro.smooth_coeff = float(self.smooth_coeff)     # read per call; the history stays
            row_src = torch.zeros(2, 4, dtype=torch.int32, device=dev)  # one frame; any cell, as the gate is open
            row_src[:, 1] = outputs['output_hand_type']
            poses, betas = pd['poses'].contiguous(), pd['betas'].contiguous()
            _ops.track_rows(self._one_euro, 1, row_src, outputs['detection_flag_cache'].float().contiguous(), poses,
                            betas)
            pd['poses'], pd['betas'] = poses, betas
        outputs = self.mano_regression(outputs, outputs['meta_data'])
        return outputs

    @torch.no_grad()
    def batch_forward(self, images_rgb_u8, offsets=None, batch_ids=None, stream_ids=None, stream_begin=None):
        """B frames (uint8 BHWC RGB, already 512x512) -> reference-schema outputs incl. MANO.  ``stream_ids`` /
        ``stream_begin`` (B,): each image's stream slot and start-over flag for ``track_hands`` with
        ``track_streams`` > 1 (meta_data['stream_ids'] / ['stream_begin'])."""
        B = images_rgb_u8.shape[0]
        if offsets is None:
            offsets = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1)
        meta = {'image': images_rgb_u8, 'offsets': offsets,
                'batch_ids': torch.arange(B) if batch_ids is None else batch_ids}
        if stream_ids is not None:
            meta['stream_ids'] = stream_ids
        if stream_begin is not None:
            meta['stream_begin'] = stream_begin
        outputs = self.model(meta, **self.demo_cfg)
        return self.process_results(outputs)

    @torch.no_grad()
    def fused_forward(self, images_rgb_u8, offsets, out=None, peers=None, tracker=None, stream_ids=None,
                      stream_begin=None, part_labels=None):
        """Sync-free pipeline: backbone + heads + parse + MANO enqueued back to back; MANO runs over
        the worst case 2KB rows (K = ``max_hands_per_side``) and skips rows >= L+R on the device.  Returns dense
        buffers (zero copy: the parse buffers are shared per batch size, consume them before the next call).  ``peers``
        (acr_b200.dist.PeerVertexGather): the MANO kernel also stores vertices and row counts into every
        rank's gather buffer.  ``tracker`` (acr_b200.ops.HandTracker): the batch is B consecutive frames of one
        stream, tracked (and, with the tracker's smooth_coeff, filtered per track) between parse and MANO;
        mano['track_id'] is the tracker's id buffer.  With a multi-stream tracker (``streams`` > 1), ``stream_ids``
        (B,) int gives each image's stream slot (the frames of one stream in batch order) and ``stream_begin`` (B,)
        starts a slot over at each nonzero frame; a row's stream is ``stream_ids[reorganize_idx]``.  ``part_labels``
        (acr_b200.ops.PartLabels): each image's uint8 part labels at its frame's resolution (``offsets``) are written
        into that buffer, mano['part_labels'] is the buffer (zero copy, like the parse buffers: consume or copy the
        labels before the next call into the same buffer).  Host offsets are checked against its capacity before
        anything is enqueued; device offsets on the device (a frame that does not fit is flagged, not written)."""
        if tracker is not None and peers is not None:
            raise ValueError("a tracker follows one stream: it cannot be combined with a cross-rank vertex gather")
        if tracker is None and (stream_ids is not None or stream_begin is not None):
            raise ValueError("stream_ids / stream_begin need a tracker")
        B = images_rgb_u8.shape[0]
        dev = images_rgb_u8.device
        sid = _device_ints(stream_ids, B, dev, 'stream_ids')
        sbeg = _device_ints(stream_begin, B, dev, 'stream_begin')
        if tracker is not None and tracker.streams > 1 and sid is None:
            raise ValueError(f"this tracker follows {tracker.streams} streams: give stream_ids, the slot of each frame")
        meta = {'image': images_rgb_u8, 'offsets': offsets, 'batch_ids': None}
        from acr_b200 import ops as _ops
        if part_labels is not None and offsets is not None and not torch.as_tensor(offsets).is_cuda:
            part_labels.expect(torch.as_tensor(offsets, dtype=torch.float32).numpy())
        eng, bufs = self.model.forward_dense(meta)
        if part_labels is not None:
            if offsets is None:
                S = float(args().input_size)
                offsets = torch.tensor([[S, S, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1)
            _ops.part_labels(eng.view('segms'), offsets, part_labels)
        ids = _ops.track_hands(bufs, tracker, sid, sbeg) if tracker is not None else None
        ml, mr = self.mano_regression.models()
        mano = _ops.mano_forward(ml, mr, bufs.poses, bufs.betas, bufs.hand_type, 1, self.mano_regression.center_idx,
                                 bufs.cam, bufs.offsets_out, n_dev=bufs.counts[2:3], peers=peers, counts=bufs.counts)
        if args().cam_trans_mode in ('lstsq', 'pnp'):
            mano['cam_trans'] = _ops.cam_trans_mode(args().cam_trans_mode, mano['joints'], mano['pj2d'],
                                                    args().focal_length, 512.0, n_dev=bufs.counts[2:3])
        if ids is not None:
            mano['track_id'] = ids
        if part_labels is not None:
            mano['part_labels'] = part_labels
        return bufs, mano

    @torch.no_grad()
    def capture_graph(self, batch: int, device=None, tracker=None, part_labels=None):
        """CUDA-graph the whole sync-free pipeline (backbone + heads + parse + MANO + cam_trans, ~380 kernel
        launches) for a fixed batch size: returns ``replay(frames_u8, offsets) -> (bufs, mano)`` that copies
        the inputs into static buffers and launches ONE graph.  This is what makes the reference's
        frame-by-frame video / webcam loop (acr/main.py:183-201, batch 1) latency-bound by the GPU instead
        of by ~380 host-side launches.  The graph is bound to the ``max_hands_per_side`` it was captured with
        (``replay.hands_per_side``); a replay under another value raises.  With a ``tracker`` the graph also tracks:
        each replay continues the tracker's state from the previous one (``tracker.reset()`` starts over).  With a
        multi-stream tracker the replay is ``replay(frames_u8, offsets, stream_ids, stream_begin=None)``: (B,) stream
        slots and start-over flags per frame, copied into static buffers of the graph.  ``part_labels`` = a capacity in
        pixels (the most H*W summed over a replay's frames): the graph also writes each image's part labels into
        ``replay.part_labels`` (acr_b200.ops.PartLabels), which is mano['part_labels'].  A replay with host offsets
        that need more raises before anything is enqueued; with device offsets the device flags such frames."""
        dev = torch.device(device) if device is not None else next(self.model.parameters()).device
        frames = torch.zeros(batch, args().input_size, args().input_size, 3, dtype=torch.uint8, device=dev)
        offsets = torch.zeros(batch, 10, device=dev)
        labels = _label_buffer(part_labels, batch, dev, None)

        def check(frames_u8, offs):
            _check_copy("frames", frames_u8, frames)
            _check_copy("offsets", offs, offsets)
            host = labels is not None and not offs.is_cuda
            return (frames_u8, offs), offs.to(torch.float32).expand(batch, 10).numpy() if host else None

        def load(inputs):
            frames.copy_(inputs[0], non_blocking=True)
            offsets.copy_(inputs[1], non_blocking=True)

        stage = _InputStage(check, load, lambda: (frames, offsets), {"static_inputs": (frames, offsets)})
        return self._capture(batch, dev, tracker, labels, stage)

    @torch.no_grad()
    def capture_frames_graph(self, batch: int, max_frame_bytes: int, device=None, tracker=None, part_labels=None):
        """``capture_graph`` from raw frames: one CUDA graph of the ragged pre-processing (cubic tables, BGR->RGB,
        white pad, bicubic resize, offsets; acr_b200.preprocess.RaggedFrames) followed by ``fused_forward``.  Returns
        ``replay(frames) -> (bufs, mano)`` for a list of exactly ``batch`` BGR frames (numpy arrays, CPU or CUDA
        tensors) of any sizes, each replay its own, whose packed H*W*3 bytes sum to at most ``max_frame_bytes``.  Host
        frames travel in one H2D copy; a list that does not fit raises before anything is written.  Like
        ``capture_graph``, the graph is bound to its ``max_hands_per_side``, and a ``tracker`` is captured with it; with
        a multi-stream tracker the replay is ``replay(frames, stream_ids, stream_begin=None)``.  ``part_labels`` True (a
        capacity of ``max_frame_bytes // 3`` pixels, which every replay fits) or a capacity in pixels: the graph also
        writes each frame's part labels into ``replay.part_labels`` (acr_b200.ops.PartLabels, mano['part_labels']);
        ``replay.part_labels[i]`` is frame i's (H_i, W_i) view."""
        from acr_b200.preprocess import RaggedFrames
        import numpy as np
        dev = torch.device(device) if device is not None else next(self.model.parameters()).device
        rf = RaggedFrames(batch, max_frame_bytes, dev, args().input_size, exact=True)
        labels = _label_buffer(part_labels, batch, dev, max_frame_bytes // 3)
        stage = _InputStage(lambda frames: (frames, rf.check(frames)[1]), rf.load, rf.launch, {"frames": rf})
        return self._capture(batch, dev, tracker, labels, stage, warm=[np.full((1, 1, 3), 255, np.uint8)] * batch)

    @torch.no_grad()
    def capture_jpeg_graph(self, batch: int, max_coded_bytes: int, max_frame_bytes: int, tracker=None, device=None,
                           max_blocks: int = None, part_labels=None, max_scans: int = 0):
        """``capture_frames_graph`` from JPEG files: one CUDA graph of the device JPEG decode (acr_b200.jpeg), the
        ragged pre-processing and ``fused_forward``.  Returns ``replay(encoded_list) -> (bufs, mano)`` for exactly
        ``batch`` JPEG files (bytes-like) whose entropy-coded bytes sum to at most ``max_coded_bytes`` and
        whose decoded H*W*3 bytes sum to at most ``max_frame_bytes``; ``max_blocks`` caps the 8x8 coefficient blocks
        (default ``max_frame_bytes // 48 + 64 * batch``: enough for every sampling when each frame is at least 18
        pixels on each side; thin frames pad more per pixel, a 1x1920 frame needs 720 blocks, so give a larger cap).
        The replay parses the headers and checks the caps and the supported features before anything is written
        (ValueError / acr_b200.jpeg.JpegUnsupported); the decode's grids are sized by the caps and the device skips
        work past each file's size.  Corrupt entropy-coded data sets the per-file status words and gives that frame
        an all-black image; ``replay.jpeg.raise_on_status()`` waits and raises.  Like ``capture_graph``, the graph
        is bound to its ``max_hands_per_side``, and a ``tracker`` is captured with it; with a multi-stream tracker the replay is
        ``replay(encoded_list, stream_ids, stream_begin=None)``.  ``part_labels`` as in ``capture_frames_graph``: True
        (``max_frame_bytes // 3`` pixels) or a capacity, the labels in ``replay.part_labels``.

        With ``max_scans = 0`` the files must be single-scan (baseline or extended sequential); progressive and
        multi-scan sequential files raise JpegUnsupported.  ``max_scans`` > 0 decodes those on the device too, as long
        as their scans number at most ``max_scans`` in a replay (single-scan files never count; more raises
        ValueError naming the capacity).  Every scan's segment starts a decoder chunk of its own, so a file's chunks
        can exceed its coded bytes / 256 by one per scan: the chunk cap is ``max_coded_bytes / 256 + batch +
        max_scans``.  The coefficient planes are the frame's whatever the script, so ``max_blocks`` is unchanged."""
        from acr_b200 import jpeg
        from acr_b200.preprocess import RaggedFrames, shapes_layout
        import cv2
        import numpy as np
        dev = torch.device(device) if device is not None else next(self.model.parameters()).device
        if max_blocks is None:
            max_blocks = max_frame_bytes // 48 + 64 * batch
        rf = RaggedFrames(batch, max_frame_bytes, dev, args().input_size, exact=True)
        jb = jpeg.JpegBatch(batch, max_coded_bytes, max_frame_bytes,
                            -(-max_coded_bytes // jpeg.CHUNK) + batch + max_scans, max_blocks, dev, out=rf.packed,
                            max_scans=max_scans)
        labels = _label_buffer(part_labels, batch, dev, max_frame_bytes // 3)

        def check(encoded_list):
            encoded_list = list(encoded_list)
            lay, _ = jb.prepare(encoded_list, exact=True)
            shapes = [(int(d["H"]), int(d["W"])) for d in lay.desc]
            return (encoded_list, lay, shapes), None if labels is None else shapes_layout(shapes)[1]

        def load(prepared):
            encoded_list, lay, shapes = prepared
            rf.load_shapes(shapes)
            jb.load(encoded_list, lay)

        def enqueue():
            jb.launch(batch)
            return rf.launch()

        warm = [cv2.imencode(".jpg", np.full((1, 1, 3), 255, np.uint8))[1].tobytes()] * batch
        stage = _InputStage(check, load, enqueue, {"frames": rf, "jpeg": jb})
        return self._capture(batch, dev, tracker, labels, stage, warm=warm)

    def _capture(self, batch, dev, tracker, labels, stage, warm=None):
        """The capture methods' graph: ``stage``'s input kernels, then ``fused_forward`` with ``tracker`` and the
        ``labels`` buffer -> ``replay``, which takes ``stage.check``'s arguments (then ``stream_ids`` and
        ``stream_begin`` with a multi-stream tracker).  A replay runs every check before it writes anything, so one
        that raises leaves the graph's inputs as the last replay left them.  ``warm``: the warm-up's input, loaded
        through the stage (None: the buffers as they are)."""
        from acr.result_parser import ResultParser
        K = ResultParser.hands_per_side()
        _check_tracker(tracker, K)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                       # warm-up: builds the engine, sets func attributes
            if warm is not None:
                stage.load(stage.check(warm)[0])
            for _ in range(2):
                self.fused_forward(*stage.enqueue(), part_labels=labels)   # (without the tracker: its state stays)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        streams = _stream_buffers(tracker, batch, dev)
        if tracker is not None:
            tracker.ids(batch)                              # the id buffer exists before the capture
            if streams is not None:
                tracker.workspace(batch)                    # and the workspace
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            bufs, mano = self.fused_forward(*stage.enqueue(), tracker=tracker, stream_ids=streams and streams[0],
                                            stream_begin=streams and streams[1], part_labels=labels)

        params = list(inspect.signature(stage.check).parameters.values())
        if streams is not None:
            params += [inspect.Parameter(name, inspect.Parameter.POSITIONAL_OR_KEYWORD, default=None)
                       for name in ("stream_ids", "stream_begin")]
        signature = inspect.Signature(params)

        def replay(*args, **kwargs):
            inputs = signature.bind(*args, **kwargs).arguments
            stream_ids, stream_begin = (inputs.pop(name, None) for name in ("stream_ids", "stream_begin"))
            _check_hands_per_side(K)
            prepared, host_offsets = stage.check(**inputs)
            if streams is not None:
                stream_ids, stream_begin = _check_streams(streams, stream_ids, stream_begin)
            if labels is not None:
                labels.expect(host_offsets)                 # the last check: it keeps the frames' geometry
            stage.load(prepared)
            if streams is not None:
                streams[0].copy_(stream_ids, non_blocking=True)
                if stream_begin is None:
                    streams[1].zero_()
                else:
                    streams[1].copy_(stream_begin, non_blocking=True)
            graph.replay()
            return bufs, mano

        replay.__signature__ = signature
        replay.graph, replay.hands_per_side, replay.static_streams, replay.part_labels = graph, K, streams, labels
        for name, value in stage.attrs.items():
            setattr(replay, name, value)
        return replay

    @torch.no_grad()
    def single_image_forward(self, image_rgb_u8_512, path=None):
        meta = {'image': image_rgb_u8_512[None] if image_rgb_u8_512.dim() == 3 else image_rgb_u8_512,
                'offsets': torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]), 'batch_ids': torch.arange(1)}
        outputs = self.model(meta, **self.demo_cfg)
        outputs['detection_flag'], outputs['reorganize_idx'] = justify_detection_state(
            outputs['detection_flag'], outputs['reorganize_idx'])
        outputs['meta_data']['imgpath'] = [path]
        return outputs

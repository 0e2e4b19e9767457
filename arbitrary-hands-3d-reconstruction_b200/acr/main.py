"""Drop-in application wrapper ``acr.main.ACR`` (reference: /root/reference/acr/main.py:24-141),
hot path only: model -> parse -> MANO.  Rendering / visualisation / CLI loops are out of scope."""
from __future__ import annotations

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
        """``track_hands``: the rows of this batch (B consecutive frames of one stream) through the device tracker,
        which also filters poses / betas per track when ``temporal_optimization`` is on; sets outputs['track_id']."""
        from acr.result_parser import ResultParser
        from acr_b200 import ops as _ops
        K = ResultParser.hands_per_side()
        bids = outputs['meta_data'].get('batch_ids')
        if bids is None:
            raise ValueError("track_hands needs meta_data['batch_ids'] (batch_forward sets arange(B))")
        bids = torch.as_tensor(bids).flatten().cpu()
        B = int(bids.numel())
        if not torch.equal(bids, torch.arange(B, dtype=bids.dtype)):
            raise ValueError("track_hands treats the batch as consecutive frames of one stream: batch_ids must be "
                             "arange(B)")
        smooth = float(self.smooth_coeff) if getattr(self, 'temporal_optimization', False) else None
        cfg = (K, int(self.track_gate), int(self.track_max_missed), smooth)
        t = getattr(self, '_hand_tracker', None)
        if t is None or (t.K, t.gate, t.max_missed, t.smooth_coeff) != cfg:     # new settings start new tracks
            t = self._hand_tracker = _ops.HandTracker(outputs['params_dict']['poses'].device, *cfg)
        pd = outputs['params_dict']
        n = pd['poses'].shape[0]
        dev = pd['poses'].device
        cen = torch.cat([outputs['l_centers_pred'], outputs['r_centers_pred']]).to(dev)     # (x, y) per row
        i32 = lambda v: v.to(device=dev, dtype=torch.int32)
        row_src = torch.stack([i32(outputs['reorganize_idx']), i32(outputs['output_hand_type']),
                               i32(cen[:, 1] * 64 + cen[:, 0]), torch.zeros(n, dtype=torch.int32, device=dev)],
                              1).contiguous()
        poses, betas = pd['poses'].contiguous(), pd['betas'].contiguous()
        ids = _ops.track_rows(t, B, row_src, outputs['detection_flag'].float().contiguous(), poses, betas)
        pd['poses'], pd['betas'] = poses, betas
        outputs['track_id'] = ids[:n].clone()

    @torch.no_grad()
    def process_results(self, outputs):
        if getattr(self, 'track_hands', False):
            self._track_results(outputs)
        # temporal optimisation (acr/main.py:69-83): OneEuro filters on poses / betas, one bank per hand type,
        # applied between parse and MANO -- here one device kernel instead of host-side filter objects
        elif getattr(self, 'temporal_optimization', False):
            from acr.result_parser import ResultParser
            if ResultParser.hands_per_side() > 1:
                raise ValueError("temporal_optimization needs max_hands_per_side=1: the filter banks are per hand type, "
                                 "and several hands of one side are not tracked across frames")
            from acr_b200 import ops as _ops
            pd = outputs['params_dict']
            assert len(pd['poses']) == 2, 'temporal smoothing streams one frame (two hand slots) at a time'
            if getattr(self, '_one_euro', None) is None:
                self._one_euro = _ops.OneEuroState(pd['poses'].device)
            poses, betas = pd['poses'].contiguous(), pd['betas'].contiguous()
            _ops.one_euro_smooth(poses, betas, self._one_euro, float(self.smooth_coeff),
                                 hand_type=outputs['output_hand_type'], detection_flag=outputs['detection_flag_cache'].float())
            pd['poses'], pd['betas'] = poses, betas
        outputs = self.mano_regression(outputs, outputs['meta_data'])
        return outputs

    @torch.no_grad()
    def batch_forward(self, images_rgb_u8, offsets=None, batch_ids=None):
        """B frames (uint8 BHWC RGB, already 512x512) -> reference-schema outputs incl. MANO."""
        B = images_rgb_u8.shape[0]
        if offsets is None:
            offsets = torch.tensor([[512., 512, 0, 0, 0, 0, 0, 0, 0, 0]]).repeat(B, 1)
        meta = {'image': images_rgb_u8, 'offsets': offsets,
                'batch_ids': torch.arange(B) if batch_ids is None else batch_ids}
        outputs = self.model(meta, **self.demo_cfg)
        return self.process_results(outputs)

    @torch.no_grad()
    def fused_forward(self, images_rgb_u8, offsets, out=None, peers=None, tracker=None):
        """Sync-free pipeline: backbone + heads + parse + MANO enqueued back to back; MANO runs over
        the worst case 2KB rows (K = ``max_hands_per_side``) and skips rows >= L+R on the device.  Returns dense
        buffers (zero copy: the parse buffers are shared per batch size, consume them before the next call).  ``peers``
        (acr_b200.dist.PeerVertexGather): the MANO kernel also stores vertices and row counts into every
        rank's gather buffer.  ``tracker`` (acr_b200.ops.HandTracker): the batch is B consecutive frames of one
        stream, tracked (and, with the tracker's smooth_coeff, filtered per track) between parse and MANO;
        mano['track_id'] is the tracker's id buffer."""
        if tracker is not None and peers is not None:
            raise ValueError("a tracker follows one stream: it cannot be combined with a cross-rank vertex gather")
        B = images_rgb_u8.shape[0]
        meta = {'image': images_rgb_u8, 'offsets': offsets, 'batch_ids': None}
        eng, bufs = self.model.forward_dense(meta)
        from acr_b200 import ops as _ops
        ids = _ops.track_hands(bufs, tracker) if tracker is not None else None
        ml, mr = self.mano_regression.models()
        mano = _ops.mano_forward(ml, mr, bufs.poses, bufs.betas, bufs.hand_type, 1, self.mano_regression.center_idx,
                                 bufs.cam, bufs.offsets_out, n_dev=bufs.counts[2:3], peers=peers, counts=bufs.counts)
        if args().cam_trans_mode in ('lstsq', 'pnp'):
            mano['cam_trans'] = _ops.cam_trans_mode(args().cam_trans_mode, mano['joints'], mano['pj2d'],
                                                    args().focal_length, 512.0, n_dev=bufs.counts[2:3])
        if ids is not None:
            mano['track_id'] = ids
        return bufs, mano

    @torch.no_grad()
    def capture_graph(self, batch: int, device=None, tracker=None):
        """CUDA-graph the whole sync-free pipeline (backbone + heads + parse + MANO + cam_trans, ~380 kernel
        launches) for a fixed batch size: returns ``replay(frames_u8, offsets) -> (bufs, mano)`` that copies
        the inputs into static buffers and launches ONE graph.  This is what makes the reference's
        frame-by-frame video / webcam loop (acr/main.py:183-201, batch 1) latency-bound by the GPU instead
        of by ~380 host-side launches.  The graph is bound to the ``max_hands_per_side`` it was captured with
        (``replay.hands_per_side``); a replay under another value raises.  With a ``tracker`` the graph also tracks:
        each replay continues the tracker's state from the previous one (``tracker.reset()`` starts over)."""
        from acr.result_parser import ResultParser
        K = ResultParser.hands_per_side()
        _check_tracker(tracker, K)
        dev = torch.device(device) if device is not None else next(self.model.parameters()).device
        frames = torch.zeros(batch, args().input_size, args().input_size, 3, dtype=torch.uint8, device=dev)
        offsets = torch.zeros(batch, 10, device=dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                       # warm-up: builds the engine, sets func attributes
            for _ in range(2):
                self.fused_forward(frames, offsets)         # (without the tracker: its state stays as it is)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        if tracker is not None:
            tracker.ids(batch)                              # the id buffer exists before the capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            bufs, mano = self.fused_forward(frames, offsets, tracker=tracker)

        def replay(frames_u8, offs):
            _check_hands_per_side(K)
            frames.copy_(frames_u8, non_blocking=True)
            offsets.copy_(offs, non_blocking=True)
            graph.replay()
            return bufs, mano

        replay.graph, replay.static_inputs, replay.hands_per_side = graph, (frames, offsets), K
        return replay

    @torch.no_grad()
    def capture_frames_graph(self, batch: int, max_frame_bytes: int, device=None, tracker=None):
        """``capture_graph`` from raw frames: one CUDA graph of the ragged pre-processing (cubic tables, BGR->RGB,
        white pad, bicubic resize, offsets; acr_b200.preprocess.RaggedFrames) followed by ``fused_forward``.  Returns
        ``replay(frames) -> (bufs, mano)`` for a list of exactly ``batch`` BGR frames (numpy arrays, CPU or CUDA
        tensors) of any sizes, each replay its own, whose packed H*W*3 bytes sum to at most ``max_frame_bytes``.  Host
        frames travel in one H2D copy; a list that does not fit raises before anything is enqueued.  Like
        ``capture_graph``, the graph is bound to its ``max_hands_per_side``, and a ``tracker`` is captured with it."""
        from acr.result_parser import ResultParser
        from acr_b200.preprocess import RaggedFrames
        K = ResultParser.hands_per_side()
        _check_tracker(tracker, K)
        import numpy as np
        dev = torch.device(device) if device is not None else next(self.model.parameters()).device
        rf = RaggedFrames(batch, max_frame_bytes, dev, args().input_size, exact=True)
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):                       # warm-up: builds the engine, sets func attributes
            rf.load([np.full((1, 1, 3), 255, np.uint8)] * batch)
            for _ in range(2):
                self.fused_forward(*rf.launch())
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        if tracker is not None:
            tracker.ids(batch)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            bufs, mano = self.fused_forward(*rf.launch(), tracker=tracker)

        def replay(frames):
            _check_hands_per_side(K)
            rf.load(frames)
            graph.replay()
            return bufs, mano

        replay.graph, replay.frames, replay.hands_per_side = graph, rf, K
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

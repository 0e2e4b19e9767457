"""Hot-path subset of the reference's ``acr.utils`` with the same names and semantics
(/root/reference/acr/utils.py); heavy arithmetic goes through libacr_b200.so."""
from __future__ import annotations

import logging
import os

import torch

from acr_b200 import ops as _ops


def BHWC_to_BCHW(x):
    """acr/utils.py:226-231"""
    return x.unsqueeze(1).transpose(1, -1).squeeze(-1)


def rot6D_to_angular(rot6D):
    """acr/utils.py:378-382 -- (N, 6J) -> (N, 3J), one fused kernel instead of ~114 launches."""
    return _ops.rot6d_to_aa(rot6D)


def batch_orth_proj(X, camera, mode='2d', keep_dim=False):
    """acr/utils.py:384-390 (plain torch; the fused MANO kernel emits the same values directly)."""
    camera = camera.view(-1, 1, 3)
    X_camed = X[:, :, :2] * camera[:, :, 0].unsqueeze(-1)
    X_camed = X_camed + camera[:, :, 1:]
    if keep_dim:
        X_camed = torch.cat([X_camed, X[:, :, 2].unsqueeze(-1)], -1)
    return X_camed


def convert_kp2d_from_input_to_orgimg(kp2ds, offsets):
    """acr/utils.py:392-397; offsets = [pad_h,pad_w | crop t,r,b,l | pad t,r,b,l]"""
    offsets = offsets.float().to(kp2ds.device)
    img_pad_size, crop_trbl, pad_trbl = offsets[:, :2], offsets[:, 2:6], offsets[:, 6:10]
    leftTop = torch.stack([crop_trbl[:, 3] - pad_trbl[:, 3], crop_trbl[:, 0] - pad_trbl[:, 0]], 1)
    return (kp2ds + 1) * img_pad_size.unsqueeze(1) / 2 + leftTop.unsqueeze(1)


def justify_detection_state(detection_flag, reorganize_idx):
    """acr/utils.py:1098-1104"""
    if detection_flag.sum() == 0:
        detection_flag = False
    else:
        reorganize_idx = reorganize_idx[detection_flag.bool()].long()
        detection_flag = True
    return detection_flag, reorganize_idx


def copy_state_dict(cur_state_dict, pre_state_dict, prefix='module.', drop_prefix='', fix_loaded=False):
    """acr/utils.py:1106-1151: current key k is filled from checkpoint key prefix+k; missing keys are
    reported and skipped."""
    success, failed = [], []
    for k in cur_state_dict.keys():
        src = pre_state_dict.get(prefix + k.replace(drop_prefix, ''))
        if src is None:
            failed.append(k)
            continue
        try:
            cur_state_dict[k].copy_(src)
            success.append(k)
        except Exception:
            logging.info('copy param {} failed, mismatched'.format(k))
    logging.info('missing parameters of layers:{}, {}'.format(len(failed), failed))
    logging.info('success layers:{}/{}'.format(len(success), len(cur_state_dict)))
    return success


def load_model(path, model, prefix='module.', drop_prefix='', optimizer=None, **kwargs):
    """acr/utils.py:1153-1168"""
    logging.info('using fine_tune model: {}'.format(path))
    if not os.path.exists(path):
        logging.warning('model {} not exist!'.format(path))
        raise ValueError(path)
    pretrained = torch.load(path, map_location='cpu')
    if isinstance(pretrained, dict):
        pretrained = pretrained.get('model_state_dict', pretrained)
        pretrained = pretrained.get('state_dict', pretrained)
    copy_state_dict(model.state_dict(), pretrained, prefix=prefix, drop_prefix=drop_prefix, **kwargs)
    if hasattr(model, 'invalidate_engine'):
        model.invalidate_engine()
    return model


def reorganize_results(outputs, img_paths, reorganize_idx):
    """Host-side packaging of one batch into ``{img_path: [per-hand dict, ...]}`` with fp16 numpy payloads,
    detected hands only (acr/utils.py:1226-1271).  One D2H per tensor, like the reference."""
    import numpy as np
    to_np = lambda t, dt=np.float16: t.detach().cpu().numpy().astype(dt)
    detected = outputs['detection_flag_cache'].detach().cpu().numpy().astype(np.bool_)
    pd = outputs['params_dict']
    fields = dict(cam=to_np(pd['cam']), cam_trans=to_np(outputs['cam_trans']), poses=to_np(pd['poses']),
                  betas=to_np(pd['betas']), j3d=to_np(outputs['j3d']), verts=to_np(outputs['verts']),
                  pj2d=to_np(outputs['pj2d']), pj2d_org=to_np(outputs['pj2d_org']),
                  hand_type=to_np(outputs['output_hand_type'], np.int32))
    fields = {k: v[detected] for k, v in fields.items()}
    reorganize_idx = np.asarray(reorganize_idx)
    results = {}
    for vid in np.unique(reorganize_idx):
        rows = np.where(reorganize_idx == vid)[0]
        results[img_paths[rows[0]]] = [dict({k: v[r] for k, v in fields.items()}, detection_flag_cache=detected[r])
                                       for r in rows]
    return results


def save_results(image_folder, output_dir, results_dict):
    """acr/utils.py:124-129: pickle the packaged results as
    ``<output_dir>/<folder name>_hand<checkpoint file name>_<confidence threshold>.pkl``."""
    import pickle
    from acr.config import args
    model_name = args().model_path.split('/')[-1]
    path_name = image_folder.split('/')[-1]
    with open(output_dir + f'/{path_name}_hand{model_name}_{args().centermap_conf_thresh}.pkl', 'wb') as f:
        pickle.dump(results_dict, f)


def img_preprocess(image, imgpath=None, input_size=512, single_img_input=False, bbox=None):
    """Drop-in for acr/utils.py:1315-1337 on the device: ``image`` is a BGR frame (numpy HxWx3 uint8, or a CUDA
    uint8 tensor HxWx3 / NxHxWx3); returns the reference's dict with ``image`` (uint8 RGB, white-padded to a
    square and bicubic-resized to input_size) as a CUDA tensor and the 10-element ``offsets``.

    ``image`` may also be a list of BGR frames of any sizes (numpy arrays, CPU or CUDA tensors): they are resized in
    one launch, ``image`` is then (n, S, S, 3) and ``offsets`` (n, 10), each row in its own frame's pixels, and a list
    ``imgpath`` gives lists ``imgpath`` and ``name``."""
    from acr_b200.preprocess import preprocess_frames
    import numpy as np
    if isinstance(image, (list, tuple)):
        paths = None if imgpath is None else [imgpath] if isinstance(imgpath, str) else list(imgpath)
        if paths is not None and len(paths) != len(image):
            raise ValueError(f"{len(image)} frames but {len(paths)} image paths")
        out, offsets = preprocess_frames(list(image), input_size)
        input_data = {'image': out, 'offsets': offsets, 'data_set': 'internet'}
        if paths is not None:
            input_data.update({'imgpath': paths, 'name': [os.path.basename(p) for p in paths]})
        return input_data
    t = torch.from_numpy(np.ascontiguousarray(image)) if isinstance(image, np.ndarray) else image
    t = t.cuda(non_blocking=True)
    batched = t.dim() == 4
    out, offsets = preprocess_frames(t if batched else t[None], input_size)
    if not batched and not single_img_input:
        out, offsets = out[0], offsets[0]
    input_data = {'image': out, 'offsets': offsets, 'data_set': 'internet'}
    if imgpath is not None:
        input_data.update({'imgpath': imgpath, 'name': os.path.basename(imgpath)})
    return input_data


def img_preprocess_jpeg(encoded_list, paths=None, input_size=512, host_fallback=False, max_scans=0):
    """``img_preprocess`` of a list of JPEG files (encoded bytes): decoded on the device (acr_b200.jpeg.decode, equal
    to cv2.imdecode), then padded and resized in one launch.  Returns the same dict as ``img_preprocess`` of the
    decoded frames.  Unsupported files raise before anything is enqueued unless ``host_fallback``; ``max_scans`` > 0
    decodes progressive and multi-scan sequential files with up to that many scans in all on the device."""
    from acr_b200 import jpeg
    return img_preprocess(jpeg.decode(encoded_list, host_fallback=host_fallback, max_scans=max_scans), paths,
                          input_size)

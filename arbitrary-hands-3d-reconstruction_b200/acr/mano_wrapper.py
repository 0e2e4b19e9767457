"""Drop-in ``MANOWrapper`` (reference: /root/reference/acr/mano_wrapper.py:14-50): both hands, the
projection and (optionally) the camera translation in ONE kernel launch."""
from __future__ import annotations

import torch
import torch.nn as nn

from acr.config import args
from acr_b200 import ops as _ops
from mano.manolayer import ManoLayer


class MANOWrapper(nn.Module):
    def __init__(self, assets=None):
        super().__init__()
        cidx = args().align_idx if args().mano_mesh_root_align else None
        mk = lambda side: ManoLayer(ncomps=45, center_idx=cidx, side=side, mano_root=args().mano_root,
                                    use_pca=False, flat_hand_mean=False,
                                    asset=None if assets is None else assets[side])
        self.mano_layer = nn.ModuleDict({'r': mk('right'), 'l': mk('left')})
        self.mano_layer['l'].th_shapedirs[:, 0, :] *= -1      # acr/mano_wrapper.py:35
        self.center_idx = cidx

    def models(self):
        return self.mano_layer['l'].packed_model(), self.mano_layer['r'].packed_model()

    @torch.no_grad()
    def forward(self, outputs, meta_data):
        params_dict = outputs['params_dict']
        L, R = int(outputs['left_hand_num']), int(outputs['right_hand_num'])
        dev = params_dict['poses'].device
        hand_type = torch.cat((torch.zeros(L, dtype=torch.int32, device=dev),
                               torch.ones(R, dtype=torch.int32, device=dev)))
        outputs['output_hand_type'] = hand_type
        ml, mr = self.models()
        offsets = meta_data['offsets'].to(dev) if meta_data is not None and 'offsets' in meta_data else None
        out = _ops.mano_forward(ml, mr, params_dict['poses'][:L + R], params_dict['betas'][:L + R], hand_type, 1,
                                self.center_idx, params_dict['cam'][:L + R], offsets)
        outputs.update(verts=out['verts'], j3d=out['joints'], verts_camed=out['verts_camed'], pj2d=out['pj2d'])
        if 'pj2d_org' in out:
            outputs['pj2d_org'] = out['pj2d_org']
        # cam_trans: the reference runs cv2.solvePnPRansac per hand on the host (acr/utils.py:403-407,
        # 414-519) only to feed the renderer.  'pnp' = that RANSAC-EPnP on the device; 'lstsq' = its own
        # closed-form fall-back (estimate_translation_np :430-472) on the device; neither makes a D2H/H2D round
        # trip (SURVEY.md 8f-1); 'none' skips it.
        outputs['cam_trans'] = _ops.cam_trans_mode(args().cam_trans_mode, out['joints'], out['pj2d'],
                                                   args().focal_length, 512.0)
        return outputs

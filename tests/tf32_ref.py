"""fp32 -> tf32 rounding and the same-rounding restatement of the TF32 plan (test infrastructure).

The TF32 plan (``model_precision='tf32'``) stores fp32 and runs every conv but the stem on the tensor cores with tf32
operands.  Its two rounding points, both on conv operands:
  * weights: acr_b200_pack_conv(..., DT_TF32) rounds every BN-folded weight to the nearest tf32 value, ties away from
    zero (``tf32_round``).  The bias stays fp32.
  * activations: stored fp32; the conv kernel rounds each A operand stage to the nearest tf32 in shared memory
    (cvt.rna, ties away from zero: ``tf32_round``) before the MMAs read it.
A raw fp32 operand would be truncated by the tensor cores: they use the top 19 bits (sign, exponent, 10 mantissa bits)
and drop the low 13 (``tf32_truncate``).  Both are measured on the H100 by
tests/test_gpu_tf32.py::test_operand_rounding.
Everything else (products, sums, the stem, fuse sums, bilinear up-sampling, pooling) is fp32 or better.
"""
import torch

from oracle import net_ref

_LOW13 = 0x1FFF


def _finite(u):
    return (u & 0x7F800000) != 0x7F800000


def tf32_round(x: torch.Tensor) -> torch.Tensor:
    """Nearest tf32 value of every float32 element, ties away from zero (cvt.rna.tf32.f32); Inf / NaN unchanged."""
    u = x.detach().float().contiguous().view(torch.int32)
    return torch.where(_finite(u), (u + 0x1000) & ~_LOW13, u).view(torch.float32)


def tf32_truncate(x: torch.Tensor) -> torch.Tensor:
    """float32 -> tf32 toward zero: the low 13 mantissa bits cleared (what the tensor cores read of an fp32 operand)."""
    u = x.detach().float().contiguous().view(torch.int32)
    return torch.where(_finite(u), u & ~_LOW13, u).view(torch.float32)


act_round = tf32_round         # what a tensor-core conv of the TF32 plan makes of its fp32 activation operand


class TF32Net(net_ref._Net):
    """net_ref._Net with the rounding points of the TF32 plan: BN folded into the conv weights (the weight / bias split of
    acr_b200_pack_conv), the folded weights rounded by ``tf32_round`` and the input of every tensor-core conv by
    ``act_round``; stored activations stay fp32.  The stem (backbone.conv1) runs on the CUDA cores: exact.
    contact_layers[4|5] is evaluated in its folded form, as a 128 -> 109 1x1 tensor-core conv over the stored cam /
    params maps with a per-image fp32 bias."""

    def __init__(self, sd):
        super().__init__(sd)
        self.fold = True
        self._head_operands = 0

    def rnd(self, x):
        # _Net calls rnd where the 16-bit plans store.  Here storage is fp32, so only two kinds of calls round: the folded
        # final conv's weight matrices (2-D), and the two operands of that conv (the cam and params maps, the two calls
        # that follow the last head stack of a side; head_stack arms them)
        if self._head_operands:
            self._head_operands -= 1
            return act_round(x)
        return tf32_round(x) if x.dim() == 2 else x

    def head_stack(self, x, p):
        y = super().head_stack(x, p)
        if p.endswith("final_layers.4"):
            self._head_operands = 2
        return y

    def convbn(self, x, ckey, bkey=None, stride=1):
        if ckey == "backbone.conv1":
            return super().convbn(x, ckey, bkey, stride)    # the stem: fp32 on the CUDA cores (rnd leaves 4-D weights)
        w = self.sd[ckey + ".weight"].float()
        cb = self.sd.get(ckey + ".bias")
        if bkey:
            g, b = self.sd[bkey + ".weight"].float(), self.sd[bkey + ".bias"].float()
            m, v = self.sd[bkey + ".running_mean"].float(), self.sd[bkey + ".running_var"].float()
            sc = g / torch.sqrt(v + net_ref.EPS)
            sh = b - m * sc
        else:
            sc, sh = torch.ones(w.shape[0]), torch.zeros(w.shape[0])
        if cb is not None:
            sh = sh + cb.float() * sc
        return torch.nn.functional.conv2d(act_round(x), tf32_round(w * sc.view(-1, 1, 1, 1)), sh, stride, w.shape[-1] // 2)


def net_forward(sd, image_bhwc, return_backbone=False):
    """The TF32 plan's rounding points on an exact-arithmetic machine: image (B,512,512,3) -> the maps of net_ref."""
    with torch.no_grad():
        n = TF32Net(sd)
        x = n.backbone(image_bhwc)
        out = n.heads(x)
        if return_backbone:
            out["backbone"] = x
        return out

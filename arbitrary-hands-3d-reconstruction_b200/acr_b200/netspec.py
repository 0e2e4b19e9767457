"""Declarative description of the ACR network (HRNet-W32 trunk + SegmNet + heads).

The reference builds this network out of nested ``nn.Module`` classes
(/root/reference/acr/model.py:23-329 heads, :374-463 SegmNet, :470-539 blocks,
:571-686 HighResolutionModule, :691-881 HigherResolutionNet).  Here the same
topology is emitted as a flat op list (a tiny IR) that the launch-plan builder
turns into kernel launches and that the parameter registry turns into a
state-dict with the *reference's key names* (checkpoint compatibility,
/root/reference/acr/utils.py:1106-1168).

IR
--
``Tensor``  : per-image activation (C logical channels, H, W); stored NHWC.
``Op``      : kind in {"stem","conv","fuse","bilinear2x","coordcat","pool",
              "parthead"}; convs carry the state-dict keys of their weights.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

BN_EPS = 1e-5  # nn.BatchNorm2d default, used by every BN in acr/model.py


@dataclass
class Tensor:
    name: str
    C: int
    H: int
    W: int
    dtype: str = "act"  # "act" = bf16/fp16 activation, "f32" = fp32 map
    # channel view into a wider buffer (used for the 32+2 coord concat)
    base: Optional["Tensor"] = None
    c_off: int = 0


@dataclass
class Op:
    kind: str
    out: Tensor
    ins: List[Tensor] = field(default_factory=list)
    attrs: dict = field(default_factory=dict)


class NetSpec:
    """Op list + parameter registry (key -> (shape, kind))."""

    def __init__(self):
        self.ops: List[Op] = []
        self.params: "OrderedDict[str, Tuple[Tuple[int, ...], str]]" = OrderedDict()
        self.tensors: Dict[str, Tensor] = {}
        self._n = 0

    # ------------------------------------------------------------------ utils
    def _t(self, C, H, W, hint, dtype="act") -> Tensor:
        self._n += 1
        t = Tensor(f"t{self._n}_{hint}", C, H, W, dtype)
        self.tensors[t.name] = t
        return t

    def _reg(self, key, shape, kind):
        assert key not in self.params, key
        self.params[key] = (tuple(shape), kind)

    def _reg_bn(self, key, c):
        self._reg(key + ".weight", (c,), "bn_w")
        self._reg(key + ".bias", (c,), "bn_b")
        self._reg(key + ".running_mean", (c,), "bn_mean")
        self._reg(key + ".running_var", (c,), "bn_var")
        self._reg(key + ".num_batches_tracked", (), "bn_nbt")

    # -------------------------------------------------------------------- ops
    def conv(self, x: Tensor, wkey: str, bnkey: Optional[str], cout: int, k: int,
             s: int = 1, relu: bool = False, bias: bool = False,
             residual: Optional[Tensor] = None, out_dtype: str = "act",
             out: Optional[Tensor] = None, hint: str = "", pow11: bool = False, defer: bool = False):
        """``defer=True``: the parameters are registered HERE (registry order = the reference's construction order, which
        the seeded weights and goldens depend on) but the op is returned instead of appended, for the caller to place
        later in the schedule (-> (tensor, op))."""
        self._reg(wkey + ".weight", (cout, x.C, k, k), "conv_w")
        if bias:
            self._reg(wkey + ".bias", (cout,), "conv_b")
        if bnkey:
            self._reg_bn(bnkey, cout)
        Ho, Wo = x.H // s, x.W // s
        y = out if out is not None else self._t(cout, Ho, Wo, hint or wkey.split(".")[-1], out_dtype)
        op = Op("conv", y, [x] + ([residual] if residual is not None else []),
                dict(w=wkey, bn=bnkey, bias=bias, k=k, s=s, relu=relu,
                     residual=residual is not None, pow11=pow11))
        if defer:
            return y, op
        self.ops.append(op)
        return y

    def reg_conv(self, wkey: str, bnkey: Optional[str], cout: int, cin: int, k: int, bias: bool) -> None:
        """Parameter registration of one conv (+BN), in the position of the registry where it is called (the seeded
        synthetic weights and the golden fixtures depend on the registration ORDER, which follows the reference's
        module construction order)."""
        self._reg(wkey + ".weight", (cout, cin, k, k), "conv_w")
        if bias:
            self._reg(wkey + ".bias", (cout,), "conv_b")
        if bnkey:
            self._reg_bn(bnkey, cout)

    def conv_merged(self, x: Tensor, keys: List[Tuple[str, Optional[str]]], cout: int, k: int, s: int = 1,
                    relu: bool = False, bias: bool = False, hint: str = "merged") -> List[Tensor]:
        """Several convs of identical geometry that read the SAME input, run as ONE conv with their output
        channels concatenated (one pass over the input, N = len(keys) * cout per MMA instead of len(keys)
        launches of N = cout).  Returns the channel slices of the wide output, one per original conv.  The
        parameters are NOT registered here: the caller registers them with reg_conv where the reference builds them."""
        assert cout % 16 == 0
        wide = self._t(cout * len(keys), x.H // s, x.W // s, hint)
        slices = []
        for i, (wkey, _) in enumerate(keys):
            t = Tensor(f"{wide.name}_s{i}", cout, wide.H, wide.W, "act", base=wide, c_off=i * cout)
            self.tensors[t.name] = t
            slices.append(t)
        self.ops.append(Op("conv", wide, [x], dict(w=[w for w, _ in keys], bn=[b for _, b in keys], bias=bias, k=k, s=s,
                                                   relu=relu, residual=False, pow11=False, merged=cout)))
        return slices

    def deconv(self, x: Tensor, wkey: str, bnkey: str, cout: int, out: Optional[Tensor] = None) -> Tensor:
        """nn.ConvTranspose2d(x.C, cout, 4, stride 2, padding 1, bias=False) + BN + ReLU: (C,H,W) -> (cout,2H,2W).  The
        weight is registered in ConvTranspose2d's own layout (cin, cout, 4, 4)."""
        self._reg(wkey + ".weight", (x.C, cout, 4, 4), "deconv_w")
        self._reg_bn(bnkey, cout)
        y = out if out is not None else self._t(cout, 2 * x.H, 2 * x.W, wkey.split(".")[-1])
        self.ops.append(Op("deconv", y, [x], dict(w=wkey, bn=bnkey, k=4, s=2, relu=True, residual=False, pow11=False,
                                                   deconv=True)))
        return y

    def fuse(self, terms: List[Tuple[Tensor, int]], relu=True, out: Optional[Tensor] = None) -> Tensor:
        t0 = terms[0][0]
        H, W = t0.H << terms[0][1], t0.W << terms[0][1]
        y = out if out is not None else self._t(t0.C, H, W, "fuse")
        self.ops.append(Op("fuse", y, [t for t, _ in terms],
                           dict(shifts=[sh for _, sh in terms], relu=relu)))
        return y


# ---------------------------------------------------------------------------
# HRNet-W32 trunk   (reference: HigherResolutionNet.make_baseline / forward,
#                    acr/model.py:785-865)
# ---------------------------------------------------------------------------
WIDTHS = (32, 64, 128, 256)


def _basic_block(g: NetSpec, x: Tensor, p: str, c: int) -> Tensor:
    # acr/model.py:470-499  conv3x3-bn-relu, conv3x3-bn, += residual, relu
    y = g.conv(x, p + ".conv1", p + ".bn1", c, 3, relu=True)
    return g.conv(y, p + ".conv2", p + ".bn2", c, 3, relu=True, residual=x)


def _bottleneck(g: NetSpec, x: Tensor, p: str, planes: int, down: bool) -> Tensor:
    # acr/model.py:501-539  1x1 -> 3x3 -> 1x1(x4) (+ 1x1 downsample on the first block)
    res = x
    if down:
        res = g.conv(x, p + ".downsample.0", p + ".downsample.1", planes * 4, 1)
    y = g.conv(x, p + ".conv1", p + ".bn1", planes, 1, relu=True)
    y = g.conv(y, p + ".conv2", p + ".bn2", planes, 3, relu=True)
    return g.conv(y, p + ".conv3", p + ".bn3", planes * 4, 1, relu=True, residual=res)


def _hr_module(g: NetSpec, prefix: str, xs: List[Tensor], multi_scale_output: bool,
               out0: Optional[Tensor] = None, WIDTHS: Tuple[int, ...] = None, fold_fuse: bool = False) -> List[Tensor]:
    # acr/model.py:571-686; 4 BasicBlocks per branch, then the fuse layers
    WIDTHS = WIDTHS or globals()["WIDTHS"]
    nb = len(xs)
    xs = list(xs)
    for b in range(nb):
        for blk in range(4):
            xs[b] = _basic_block(g, xs[b], f"{prefix}.branches.{b}.{blk}", WIDTHS[b])
    outs = []
    for i in range(nb if multi_scale_output else 1):
        terms = []
        folded = None      # (index in terms, deferred conv op): the sum of output i is folded into this conv's epilogue
        for j in range(nb):
            if j == i:
                terms.append((xs[j], 0))
            elif j > i:  # 1x1 conv + BN at low resolution, nearest-upsampled by 2**(j-i)
                p = f"{prefix}.fuse_layers.{i}.{j}"
                z = g.conv(xs[j], p + ".0", p + ".1", WIDTHS[i], 1)
                terms.append((z, j - i))
            else:        # chain of (i-j) stride-2 3x3 convs; ReLU on all but the last
                t = xs[j]
                for k in range(i - j):
                    p = f"{prefix}.fuse_layers.{i}.{j}.{k}"
                    last = k == i - j - 1
                    if fold_fuse and last and j == i - 1:
                        # the one-conv chain from the next finer branch: output i = relu(sum of terms) is computed in THIS
                        # conv's epilogue (its own term never goes to memory), after every other term exists
                        t, op = g.conv(t, p + ".0", p + ".1", WIDTHS[i], 3, s=2, relu=False, defer=True)
                        folded = (len(terms), op)
                    else:
                        t = g.conv(t, p + ".0", p + ".1", WIDTHS[i] if last else WIDTHS[j], 3, s=2,
                                   relu=not last)
                terms.append((t, 0))
        # reference sums in order j = 0..nb-1 (acr/model.py:677-684)
        if folded is None:
            outs.append(g.fuse(terms, relu=True, out=out0 if i == 0 else None))
        else:
            pos, op = folded
            others = [tm for q, tm in enumerate(terms) if q != pos]
            op.ins = [op.ins[0]] + [t for t, _ in others]
            op.attrs.update(relu=True, extra=[(t.name, sh) for t, sh in others], extra_pos=pos)
            g.ops.append(op)
            outs.append(op.out)
    return outs


WIDTHS_W48 = (48, 96, 192, 384)


BACKBONES = ("hrnet", "resnet50")


def _resnet_bottleneck(g: NetSpec, x: Tensor, p: str, planes: int, stride: int, down: bool) -> Tensor:
    # acr/model.py:501-539 with the stride on conv2; registry order = construction order (conv1, bn1, conv2, bn2, conv3,
    # bn3, then the downsample that _make_layer (:738-752) hands to the first block)
    y = g.conv(x, p + ".conv1", p + ".bn1", planes, 1, relu=True)
    y = g.conv(y, p + ".conv2", p + ".bn2", planes, 3, s=stride, relu=True)
    out, op3 = g.conv(y, p + ".conv3", p + ".bn3", planes * 4, 1, relu=True, residual=x, defer=True)
    if down:   # 1x1 stride-s conv + BN (padding 0: it reads input pixel (s*y, s*x))
        op3.ins[1] = g.conv(x, p + ".downsample.0", p + ".downsample.1", planes * 4, 1, s=stride)
    g.ops.append(op3)
    return out


def _resnet50_trunk(g: NetSpec, img: Tensor, S: int, feat: Tensor) -> None:
    """ResNet-50 + three deconvs, ending in ``feat`` (32 channels at S/4)."""
    g._reg("backbone.conv1.weight", (64, 3, 7, 7), "conv_w")
    g._reg_bn("backbone.bn1", 64)
    x = g._t(64, S // 2, S // 2, "stem7")
    g.ops.append(Op("stem", x, [img], dict(w="backbone.conv1", bn="backbone.bn1", k=7)))
    y = g._t(64, S // 4, S // 4, "maxpool")
    g.ops.append(Op("maxpool", y, [x], {}))
    x, cin = y, 64
    for L, (planes, blocks, stride) in enumerate(((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)), 1):
        for i in range(blocks):
            s = stride if i == 0 else 1
            x = _resnet_bottleneck(g, x, f"backbone.layer{L}.{i}", planes, s, down=(i == 0 and (s != 1 or cin != planes * 4)))
            cin = planes * 4
    for j, cout in enumerate((256, 128, 32)):   # deconv_layers = [ConvT, BN, ReLU] x 3
        x = g.deconv(x, f"backbone.deconv_layers.{3 * j}", f"backbone.deconv_layers.{3 * j + 1}", cout,
                     out=feat if j == 2 else None)


def build_acr_spec(input_size: int = 512, merge_stems: bool = True, widths: Tuple[int, ...] = WIDTHS,
                   fold_fuse: bool = False, backbone: str = "hrnet") -> NetSpec:
    """Full ACR network for one image of ``input_size`` x ``input_size``.  ``merge_stems=False`` keeps the eight
    head stem convs as eight launches (A/B timing of the merged form).  ``fold_fuse``: the fuse sums of the coarser
    outputs (i >= 1) of every HighResolutionModule (acr/model.py:677-684) run in the epilogue of the stride-2 conv that
    produces their term from the next finer branch: out_i = relu(conv(x_{i-1}) + sum of the other terms, nearest-
    upsampled) -- that conv's output and a fuse launch per output disappear (15 of 23 fuse launches).  Off by default:
    the saved fuse kernels are paid back in the convs' epilogues.

    ``widths``: branch widths of the HRNet trunk.  (32, 64, 128, 256) is the reference's network (the only one it
    contains: /root/reference/acr/model.py:796-797, SURVEY F1/F2).  WIDTHS_W48 = (48, 96, 192, 384) is the HRNet-W48
    trunk BASELINE.json's configs[4] names: it has no reference implementation -- the same topology with wider
    branches, the heads reading a (widths[0] + 2)-channel map -- so its PARITY IS UNPINNED (no golden can exist); it is
    measured for throughput and pinned op by op only against the oracle's per-op restatement.

    ``backbone="resnet50"``: the ResNet-50 trunk of BASELINE.json's configs 1-2.  The reference contains no ResNet trunk
    (SURVEY F1/F2: ``--backbone`` is only a log tag there), so this spec FIXES one definition and its parity is
    unpinned, like W48.  It is built from the reference's own blocks: conv1 7x7 s2 p3 3->64 (no bias) + bn1 + ReLU on
    x/255*2-1 (as acr/model.py:832), MaxPool 3x3 s2 p1, then _make_layer(Bottleneck, 64/128/256/512, 3/4/6/3, stride
    1/2/2/2) (:501-539, :738-752: stride on the 3x3 conv2, 1x1 stride-s downsample + BN whenever the stride or width
    changes) -> 2048 channels at S/32, then 3 x [ConvTranspose2d k4 s2 p1 (no bias), BN, ReLU] with widths 256, 128, 32
    (``backbone.deconv_layers.{0,1,3,4,6,7}``) -> 32 channels at S/4.  The trunk so ends in the same contract as
    HigherResolutionNet (backbone_channels = 32, :697): SegmNet (:395 hard-codes 32 input channels), the coord concat,
    both final-layer stacks and the part branch are the reference's own network, and every non-trunk key keeps the W32
    model's name and shape, so the heads of a real checkpoint load unchanged.  The input size must be a multiple of
    512: layer4 (S/32) runs on whole 16x16 tiles."""
    if backbone not in BACKBONES:
        raise ValueError(f"backbone must be one of {BACKBONES}, got {backbone!r}")
    g = NetSpec()
    g.backbone = backbone
    S = input_size
    img = Tensor("image", 3, S, S, "u8")
    g.tensors[img.name] = img
    F = S // 4
    if backbone == "resnet50":
        if S % 512:
            raise ValueError(f"the ResNet-50 trunk needs an input size that is a multiple of 512 (layer4 runs at S/32 on whole "
                             f"16x16 tiles), got {S}")
        g.widths = (32,)
        xcat = g._t(34, F, F, "xcat")
        feat = Tensor("feat32", 32, F, F, "act", base=xcat, c_off=0)
        g.tensors[feat.name] = feat
        _resnet50_trunk(g, img, S, feat)
        _heads(g, xcat, feat, merge_stems)
        return g
    g.widths = tuple(widths)
    W0, W1, W2, W3 = g.widths

    # ---- stem (acr/model.py:831-839): x/255*2-1, conv3x3 s2 + BN + ReLU, twice
    g._reg("backbone.conv1.weight", (64, 3, 3, 3), "conv_w")
    g._reg_bn("backbone.bn1", 64)
    x = g._t(64, S // 2, S // 2, "stem1")
    g.ops.append(Op("stem", x, [img], dict(w="backbone.conv1", bn="backbone.bn1")))
    x = g.conv(x, "backbone.conv2", "backbone.bn2", 64, 3, s=2, relu=True)

    # ---- layer1: 4 Bottlenecks 64 -> 256 (acr/model.py:794)
    for i in range(4):
        x = _bottleneck(g, x, f"backbone.layer1.{i}", 64, down=(i == 0))

    # ---- transition1 + stage2 (acr/model.py:796-805, 841-847)
    xs = [g.conv(x, "backbone.transition1.0.0", "backbone.transition1.0.1", W0, 3, relu=True),
          g.conv(x, "backbone.transition1.1.0.0", "backbone.transition1.1.0.1", W1, 3, s=2, relu=True)]
    xs = _hr_module(g, "backbone.stage2.0", xs, True, WIDTHS=g.widths, fold_fuse=fold_fuse)

    # ---- transition2 + stage3 (4 modules, 3 branches)
    xs.append(g.conv(xs[-1], "backbone.transition2.2.0.0", "backbone.transition2.2.0.1", W2, 3, s=2, relu=True))
    for m in range(4):
        xs = _hr_module(g, f"backbone.stage3.{m}", xs, True, WIDTHS=g.widths, fold_fuse=fold_fuse)

    # ---- transition3 + stage4 (3 modules, 4 branches; last keeps only branch 0)
    xs.append(g.conv(xs[-1], "backbone.transition3.3.0.0", "backbone.transition3.3.0.1", W3, 3, s=2, relu=True))
    # the backbone output lands in channels [0:32) of the 34-channel coord-concat buffer
    xcat = g._t(W0 + 2, F, F, "xcat")
    feat = Tensor("feat32", W0, F, F, "act", base=xcat, c_off=0)   # ("feat32": the name, not the width)
    g.tensors[feat.name] = feat
    for m in range(3):
        last = m == 2
        xs = _hr_module(g, f"backbone.stage4.{m}", xs, not last, out0=feat if last else None, WIDTHS=g.widths, fold_fuse=fold_fuse)
    x = xs[0]
    assert x is feat
    _heads(g, xcat, feat, merge_stems)
    return g


def _heads(g: NetSpec, xcat: Tensor, feat: Tensor, merge_stems: bool) -> None:
    """Everything after the trunk (acr/model.py:47-65 head_forward), reading the trunk's feature ``feat`` = channels
    [0, W0) of the (W0 + 2)-channel coord-concat buffer ``xcat``."""
    W0, F = feat.C, feat.H
    # coord channels 32,33 are constants written once (acr/model.py:52, 340-369)
    g.ops.append(Op("coordcat", xcat, [feat], {}))

    # ---- SegmNet (acr/model.py:374-463): bilinear x2, DoubleConv 32->16->64, conv 64->33+BN+ReLU, conv 33->33
    up = g._t(W0, 2 * F, 2 * F, "bilin")
    g.ops.append(Op("bilinear2x", up, [feat], {}))
    pu = "backbone.hand_segm.segm_head.upsampler.up1.conv.double_conv"
    y = g.conv(up, pu + ".0", pu + ".1", 16, 3, relu=True, bias=True)
    y = g.conv(y, pu + ".3", pu + ".4", 64, 3, relu=True, bias=True)
    ps = "backbone.hand_segm.segm_head.segm_net.double_conv"
    y = g.conv(y, ps + ".0", ps + ".1", 33, 3, relu=True, bias=True)
    segm = g.conv(y, ps + ".3", None, 33, 3, bias=True, hint="segm")
    g.tensors["segms"] = segm

    # ---- global heads (acr/model.py:68-101, 288-313): 8 stacks on the 34-ch map
    heads = {}
    raw128 = {}
    # the eight head stems (conv3x3 s2 34->64 + BN + ReLU, acr/model.py:288-296) all read the coord-concat map: they run
    # as two merged convs of N = 4 x 64 (one per side), each a single pass over the 128x128x34 input
    stems = {}
    for side in ("l", "r") if merge_stems else ():
        keys = [(f"{side}_final_layers.{idx}.0.0", f"{side}_final_layers.{idx}.0.1") for idx in (1, 2, 3, 4)]
        for idx, t in zip((1, 2, 3, 4), g.conv_merged(xcat, keys, 64, 3, s=2, relu=True, bias=True, hint=f"{side}_stems")):
            stems[(side, idx)] = t
    for side in ("l", "r"):
        # params (106) and cam (3, scale channel through 1.1**x) heads write 16-bit slices [0,112) and
        # [112,128) of one 128-channel tensor: the input of the folded contact_layers[4|5] conv
        raw128[side] = g._t(128, F // 2, F // 2, f"{side}_raw128")
        slices = {"params": Tensor(f"{side}_params_raw", 106, F // 2, F // 2, "act", base=raw128[side], c_off=0),
                  "cam": Tensor(f"{side}_cam_raw", 3, F // 2, F // 2, "act", base=raw128[side], c_off=112)}
        for t in slices.values():
            g.tensors[t.name] = t
        for idx, (nm, co) in {1: ("params", 106), 2: ("center", 1), 3: ("cam", 3), 4: ("prior", 106)}.items():
            p = f"{side}_final_layers.{idx}"
            if merge_stems:
                g.reg_conv(p + ".0.0", p + ".0.1", 64, xcat.C, 3, bias=True)    # runs inside the merged stem conv above
                h = stems[(side, idx)]
            else:
                h = g.conv(xcat, p + ".0.0", p + ".0.1", 64, 3, s=2, relu=True, bias=True)
            for blk in range(2):
                h = _basic_block(g, h, f"{p}.1.{blk}.0", 64)
            if nm in slices:
                heads[(side, nm)] = g.conv(h, p + ".2", None, co, 1, bias=True, out=slices[nm], pow11=(nm == "cam"))
            else:
                heads[(side, nm)] = g.conv(h, p + ".2", None, co, 1, bias=True, out_dtype="f32",
                                           hint=f"{side}_{nm}")
    for k, t in heads.items():
        g.tensors[f"{k[0]}_{k[1]}_raw"] = t

    # ---- part branch (acr/model.py:116-166)
    contact = g.conv(xcat, "contact_layers.1.0", "contact_layers.1.1", 256, 3, relu=True, bias=True,
                     hint="contact")
    g._reg("cam_shape_layers.1.0.weight", (64, 256, 1, 1), "conv_w")
    g._reg("cam_shape_layers.1.0.bias", (64,), "conv_b")
    for i in (2, 3):
        g._reg(f"contact_layers.{i}.weight", (1, 6, 256, 16, 1, 1), "lc_w")
    for i in (2, 3):
        g._reg(f"cam_shape_layers.{i}.weight", (10, 1024), "lin_w")
        g._reg(f"cam_shape_layers.{i}.bias", (10,), "lin_b")
    for i in (4, 5):
        g._reg(f"contact_layers.{i}.weight", (109, 218, 1, 1), "conv_w")
        g._reg(f"contact_layers.{i}.bias", (109,), "conv_b")
    # attention pooling + per-joint heads + final 218->109 1x1 conv (folded, see plan builder)
    pooled = g._t(256, 32, 1, "pooled", "f32")
    g.ops.append(Op("pool", pooled, [contact, segm], {}))
    g.tensors["pooled"] = pooled
    for side in ("l", "r"):
        t = g._t(109, F // 2, F // 2, f"{side}_params_maps", "f32")
        g.ops.append(Op("parthead", t, [pooled, raw128[side]], dict(side=side)))
        g.tensors[f"{side}_params_maps"] = t
        g.tensors[f"{side}_center_map"] = heads[(side, "center")]
        g.tensors[f"{side}_prior_maps"] = heads[(side, "prior")]

    # ---- dead-but-present parameters (acr/model.py:181, 262-286): kept so that
    #      state_dict() has the reference's 2067 keys; never executed.
    g._reg("segmentation_layers.1.0.weight", (256, W0 + 2, 3, 3), "conv_w")
    g._reg("segmentation_layers.1.0.bias", (256,), "conv_b")
    g._reg_bn("segmentation_layers.1.1", 256)
    g._reg("segmentation_layers.2.0.weight", (33, 256, 1, 1), "conv_w")
    g._reg("segmentation_layers.2.0.bias", (33,), "conv_b")


def op_flops(op: Op) -> float:
    """2*MAC count of one conv-like op per image (0 for the others).  A transposed conv counts its LIVE taps only: every
    output pixel of the k4 s2 p1 form sees 2x2 of the 16 taps."""
    if op.kind == "conv":
        x, y = op.ins[0], op.out
        return 2.0 * y.H * y.W * y.C * x.C * op.attrs["k"] ** 2
    if op.kind == "deconv":
        x, y = op.ins[0], op.out
        return 2.0 * y.H * y.W * y.C * x.C * 4
    if op.kind == "stem":
        return 2.0 * op.out.H * op.out.W * 64 * 3 * op.attrs.get("k", 3) ** 2
    return 0.0


def conv_flops_per_image(spec: NetSpec) -> float:
    """2*MAC count of every executed Conv2d/ConvTranspose2d/Linear + the two pooling matmuls
    (SURVEY.md section 8d: 102.12 GFLOP/img for HRNet-W32 at 512x512)."""
    fl = sum(op_flops(op) for op in spec.ops)
    F = spec.tensors["feat32"].H
    fl += 2.0 * F * F * 64 * 256               # cam_shape_layers[1] 1x1 conv 256->64
    fl += 2 * 2.0 * F * F * 109 * 218 / 4      # contact_layers[4,5] at (F/2)^2
    fl += 2 * 2.0 * 1024 * 10                  # shape Linear
    fl += 2 * 2.0 * 16 * 6 * 256               # LocallyConnected2d
    fl += 2.0 * 32 * F * F * (256 + 64)        # Hadamard matmuls
    return fl

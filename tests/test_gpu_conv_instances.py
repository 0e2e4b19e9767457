"""GPU: every reachable (conv_tc_kernel instance, ping-pong, short epilogue, TMA store, fp32 output, N split) combination
of the wgmma conv, each held per element to the fp64 bound of tests/pack_ref.py, and each launch pinned to the
restated plan of tests/conv_plan_ref.py.

``MATRIX`` is plain data (tests/test_cpu_conv_plan.py imports it without a GPU and checks that it reaches every
combination the plan can produce).  Every case checks:
  * each output element within ``pack_ref.check_bound`` of the exact conv of the rounded operands (the x-paired,
    stride-2 x-paired and transposed forms from their original weights, through the engine's own packing), and 16-bit
    outputs whose rounding the bound decides rounded to nearest (``pack_ref.direction_counts``);
  * no stray store: the output sits between guard bytes of a NaN pattern that must come back bit-identical; channels
    [cout, cout_pad) are zero; channels the op does not own (cout_pad up to the pixel stride, or past cout for the
    transposed conv's channel slice) keep their NaN pattern;
  * the launch, recorded by torch.profiler (CUPTI activity tracing), is the restated instance (T, CK, MODE, NT) with the
    restated grid and dynamic shared memory (for these launches the trace's "shared memory" is the dynamic bytes the
    launch asked for), which ties SA, SB and the TMA-store stage to the restatement.
"""
import ctypes as C
import json
import os
import re
import tempfile
import time
import zlib
from dataclasses import dataclass, replace

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests import conv_plan_ref as R
from tests.helpers import ctensor, rup

pytestmark = pytest.mark.gpu

BF16, F16, TF32 = L.DT_BF16, L.DT_F16, L.DT_TF32
DT_NAME = {BF16: "bf16", F16: "fp16", TF32: "tf32"}
GUARD = 4096            # NaN-pattern bytes before and after every output


@dataclass(frozen=True)
class Case:
    """One op-level conv.  H, W: the dense input's spatial size (x-paired form: W dense pixels, W / 2 pairs).
    cin_pad / in_stride: None = cin rounded up to 16; in_stride < cin_pad leaves a K tail that only TMA out-of-bounds
    zeros fill.  out_stride: the output's pixel stride (None = cout_pad); wider rows hold channels the op does not own."""
    dt: int
    form: str           # "conv", "xpair", "s2x", "deconv"
    B: int
    H: int
    W: int
    cin: int
    cout: int
    k: int = 3
    s: int = 1
    cin_pad: int = None
    in_stride: int = None
    out_stride: int = None
    residual: bool = False
    pow11: bool = False
    bias_img: bool = False
    out_f32: bool = False
    tma: bool = False
    relu: bool = True
    ch_scale: bool = False
    xflags: int = 4     # x-paired form: ACR_CONV_XPAIR (4, corner MMAs of the side taps) or 0 (full block-sparse)

    @property
    def id(self):
        f = self.form if self.form != "conv" else f"k{self.k}s{self.s}"
        cp = "" if self.cin_pad in (None, rup(self.cin, 16)) else f"/{self.cin_pad}"
        st = "" if self.in_stride in (None, self.cin_pad, rup(self.cin, 16)) else f"s{self.in_stride}"
        tags = [t for t, on in (("res", self.residual), ("pow11", self.pow11), ("bimg", self.bias_img),
                                ("f32", self.out_f32), ("tma", self.tma), ("chs", self.ch_scale)) if on]
        if self.form == "xpair":
            tags.append(f"flags{self.xflags}")
        if self.out_stride:
            tags.append(f"ostride{self.out_stride}")
        return (f"{DT_NAME[self.dt]}-{f}-B{self.B}-{self.H}x{self.W}-{self.cin}{cp}{st}-{self.cout}"
                + "".join("-" + t for t in tags))


def _pads(c: Case):
    cin_pad = c.cin_pad or rup(c.cin, 16)
    return cin_pad, c.in_stride or cin_pad, 64 if c.form == "xpair" else rup(c.cout, 16)


def conv_args(c: Case) -> R.ConvArgs:
    """The ConvArgs the library builds for a case (plan.cu make_conv_args) -> the plan restatement's input."""
    cin_pad, in_stride, cout_pad = _pads(c)
    out_stride = c.out_stride or cout_pad
    common = dict(dt=c.dt, batch=c.B, cout_pad=cout_pad, out_stride=64 if c.form == "xpair" else out_stride, residual=c.residual, out_f32=c.out_f32,
                  bias_per_image=c.bias_img, pow11=c.pow11, tma_env=c.tma)
    if c.form == "xpair":
        return R.ConvArgs(in_H=c.H, in_W=c.W // 2, out_H=c.H, out_W=c.W // 2, cin_pad=64, in_stride=64, k=3, stride=1,
                          xpair=bool(c.xflags & L.CONV_XPAIR), **common)   # (flags 0: a plain 64 -> 64 conv)
    if c.form == "s2x":
        return R.ConvArgs(in_H=c.H, in_W=c.W // 2, out_H=c.H // 2, out_W=c.W // 2, cin_pad=64, in_stride=64, in_C=64,
                          k=3, stride=2, s2x=True, **common)
    if c.form == "deconv":
        return R.ConvArgs(in_H=c.H, in_W=c.W, out_H=2 * c.H, out_W=2 * c.W, cin_pad=cin_pad, in_stride=in_stride, k=4,
                          stride=2, deconv=True, **common)
    return R.ConvArgs(in_H=c.H, in_W=c.W, out_H=c.H // c.s, out_W=c.W // c.s, cin_pad=cin_pad, in_stride=in_stride,
                      k=c.k, stride=c.s, **common)


# ------------------------------------------------------------------------------------------------------- the matrix
# Channel configurations (form, cin, cout, k, s, extra Case fields).  A comment names the instance MODE / NT and the
# runtime branches the configuration was picked for; the 32 KB TMA-store stage moves some of them to streamed weights,
# and what each case reaches is what tests/conv_plan_ref.py says (tests/test_cpu_conv_plan.py prints it).  Streamed weights come from cout_pad > 256 or from
# enough taps x channel chunks; cout 272 is three virtual tiles of 96 whose last one reads weight rows past cout_pad;
# cin < cin_pad with in_stride < cin_pad is a K tail filled by TMA out-of-bounds zeros.
_S16 = [
    # CK = 16 (cin_pad an odd multiple of 16)
    ("conv", 1392, 64, 1, 1, {}),                       # 0 / 64, streamed
    ("conv", 720, 128, 1, 1, {}),                       # 0 / 128
    ("conv", 13, 272, 1, 1, {}),                        # 0 / 128, 3 N splits, rows past cout_pad
    ("conv", 176, 48, 3, 2, {}),                        # 0 / 64, stride 2 from four parity views
    ("conv", 176, 64, 3, 1, {}),                        # PATCH / 64, streamed
    ("conv", 80, 112, 3, 1, {}),                        # PATCH / 128
    ("conv", 16, 272, 3, 1, {}),                        # PATCH / 128, N split
    ("conv", 144, 80, 1, 1, {}),                        # RESIDENT / 128, lockstep
    ("conv", 144, 144, 1, 2, {}),                       # RESIDENT / 128, lockstep, N split, 1x1 stride 2
    ("conv", 16, 80, 1, 1, dict(out_stride=96)),        # RESIDENT / 128, ping-pong, rows wider than cout_pad
    ("conv", 16, 144, 1, 1, {}),                        # RESIDENT / 128, ping-pong, N split
    ("conv", 144, 16, 1, 1, {}),                        # RESIDENT / 64, lockstep
    ("conv", 5, 16, 1, 1, {}),                          # RESIDENT / 64, ping-pong
    ("conv", 34, 80, 3, 1, dict(cin_pad=48)),           # PATCH|RESIDENT / 128, lockstep
    ("conv", 48, 144, 3, 1, {}),                        # PATCH|RESIDENT / 128, lockstep, N split
    ("conv", 16, 80, 3, 1, {}),                         # PATCH|RESIDENT / 128, ping-pong
    ("conv", 16, 144, 3, 1, {}),                        # PATCH|RESIDENT / 128, ping-pong, N split
    ("conv", 48, 16, 3, 1, {}),                         # PATCH|RESIDENT / 64, lockstep
    ("conv", 16, 16, 3, 1, {}),                         # PATCH|RESIDENT / 64, ping-pong
    ("conv", 34, 64, 3, 2, dict(cin_pad=48)),           # RESIDENT / 64, stride 2 (the head stem's form)
    # CK = 32
    ("conv", 1312, 64, 1, 1, {}),
    ("conv", 672, 128, 1, 1, {}),
    ("conv", 32, 272, 1, 1, {}),
    ("conv", 608, 16, 3, 1, {}),                        # PATCH / 64, streamed
    ("conv", 96, 112, 3, 1, {}),                        # PATCH / 128
    ("conv", 32, 256, 3, 1, {}),                        # PATCH / 128, N split (2 x 128)
    ("conv", 288, 80, 1, 1, {}),
    ("conv", 288, 144, 1, 1, {}),
    ("conv", 32, 80, 1, 1, {}),
    ("conv", 32, 144, 1, 1, {}),
    ("conv", 288, 16, 1, 1, {}),
    ("conv", 32, 16, 1, 1, {}),
    ("conv", 96, 80, 3, 1, {}),
    ("conv", 32, 240, 3, 1, {}),                        # PATCH|RESIDENT / 128, lockstep, N split
    ("conv", 32, 80, 3, 1, {}),
    ("conv", 32, 144, 3, 1, dict(out_stride=160)),
    ("conv", 96, 16, 3, 1, {}),
    ("conv", 32, 16, 3, 1, {}),
    ("conv", 32, 64, 3, 2, {}),                         # stride 2, four parity views
    # CK = 64
    ("conv", 1024, 64, 1, 1, {}),                       # 0 / 64
    ("conv", 512, 128, 1, 1, {}),                       # 0 / 128
    ("conv", 64, 272, 1, 1, {}),                        # 0 / 128, N split
    ("conv", 320, 96, 1, 1, {}),                        # RESIDENT / 128, lockstep
    ("conv", 256, 176, 1, 2, {}),                       # RESIDENT / 128, lockstep, N split, 1x1 stride 2
    ("conv", 48, 80, 1, 1, dict(cin_pad=64)),           # RESIDENT / 128, ping-pong, K tail
    ("conv", 64, 144, 1, 1, dict(out_stride=256)),      # RESIDENT / 128, ping-pong, N split
    ("conv", 448, 16, 1, 1, {}),                        # RESIDENT / 64, lockstep
    ("conv", 64, 16, 1, 1, {}),                         # RESIDENT / 64, ping-pong
    ("conv", 448, 16, 3, 1, {}),                        # PATCH|P1 / 64, streamed
    ("conv", 64, 112, 3, 1, {}),                        # PATCH|P1 / 128
    ("conv", 48, 144, 3, 1, dict(cin_pad=64)),          # PATCH|P1 / 128, N split, K tail
    ("conv", 192, 16, 3, 1, {}),                        # PATCH|RESIDENT|P1 / 64, lockstep
    ("conv", 64, 16, 3, 1, {}),                         # PATCH|RESIDENT|P1 / 64, ping-pong
    ("conv", 64, 80, 3, 1, dict(out_stride=128)),       # PATCH|RESIDENT|P1 / 128, ping-pong
    ("conv", 96, 64, 3, 2, dict(cin_pad=128)),          # RESIDENT / 64, stride 2, K tail
    ("s2x", 32, 112, 3, 2, {}),                         # S2X / 128, streamed
    ("s2x", 32, 144, 3, 2, {}),                         # S2X / 128, streamed, N split
    ("s2x", 32, 80, 3, 2, {}),                          # RESIDENT|S2X / 128, ping-pong
    ("s2x", 32, 16, 3, 2, {}),                          # RESIDENT|S2X / 64, ping-pong
    ("s2x", 32, 32, 3, 2, {}),
    ("deconv", 64, 16, 4, 2, {}),                       # DECONV / 64
    ("deconv", 64, 80, 4, 2, {}),                       # DECONV / 128
    ("deconv", 128, 144, 4, 2, {}),                     # DECONV / 128, N split
    ("deconv", 64, 32, 4, 2, dict(out_stride=48)),      # DECONV / 64 into channels [0, 32) of a 48-wide buffer
    ("xpair", 32, 32, 3, 1, dict(xflags=4)),            # PATCH|RESIDENT|XPAIR / 64, ping-pong
    ("xpair", 32, 32, 3, 1, dict(xflags=0)),
]
# TF32 (channels are fp32: CK = 32 for cin_pad an odd multiple of 16, CK = 64 for multiples of 32)
_S32 = [
    ("conv", 1520, 32, 1, 1, {}), ("conv", 624, 80, 1, 1, {}), ("conv", 16, 272, 1, 1, {}),
    ("conv", 304, 16, 3, 1, {}), ("conv", 48, 112, 3, 1, {}), ("conv", 16, 272, 3, 1, {}),
    ("conv", 144, 80, 1, 1, {}), ("conv", 144, 144, 1, 1, {}), ("conv", 16, 80, 1, 1, {}), ("conv", 16, 144, 1, 1, dict(out_stride=160)),
    ("conv", 144, 16, 1, 1, {}), ("conv", 16, 16, 1, 1, {}),
    ("conv", 48, 80, 3, 1, {}), ("conv", 16, 80, 3, 1, {}), ("conv", 16, 144, 3, 1, {}), ("conv", 48, 16, 3, 1, {}),
    ("conv", 13, 16, 3, 1, {}), ("conv", 34, 64, 3, 2, dict(cin_pad=48)),
    ("conv", 640, 64, 1, 1, {}), ("conv", 320, 128, 1, 1, {}), ("conv", 32, 272, 1, 1, {}),
    ("conv", 160, 96, 1, 1, {}), ("conv", 128, 176, 1, 2, {}), ("conv", 32, 80, 1, 1, {}), ("conv", 32, 144, 1, 1, {}),
    ("conv", 224, 16, 1, 1, {}), ("conv", 32, 16, 1, 1, {}),
    ("conv", 224, 16, 3, 1, {}), ("conv", 32, 112, 3, 1, {}), ("conv", 24, 144, 3, 1, dict(cin_pad=32)),
    ("conv", 96, 16, 3, 1, {}), ("conv", 32, 16, 3, 1, {}), ("conv", 32, 80, 3, 1, {}),
    ("conv", 64, 64, 3, 2, {}),
]
# epilogues: the short loop, the general loop with a residual, the TMA-store epilogue, fp32 output (the head's final
# convs: per-image bias, 1.1 ** channel 0); the transposed conv takes none of the optional terms
_E16 = [dict(), dict(residual=True), dict(tma=True), dict(out_f32=True, relu=False, bias_img=True),
        dict(out_f32=True, relu=False, pow11=True, residual=True)]
_E32 = [dict(out_f32=True), dict(out_f32=True, residual=True), dict(out_f32=True, relu=False, pow11=True, bias_img=True)]
# geometries: (B, output H, output W), a one-tile output first; distinct images at batch 2 and 3
_GEO = [(1, 16, 16), (2, 16, 32), (3, 32, 16), (2, 32, 32)]


def _case(dt, spec, epi, gi, ch_scale):
    form, cin, cout, k, s, extra = spec
    B, Ho, Wo = _GEO[gi % len(_GEO)]
    H, W = (Ho, Wo) if form == "deconv" else (Ho * s, Wo * s)      # (the transposed conv: input tiles, output 2H x 2W)
    if form == "xpair":
        W = 2 * Wo                                           # Wo pairs = 2 Wo dense pixels
    c = Case(dt=dt, form=form, B=B, H=H, W=W, cin=cin, cout=cout, k=k, s=s, ch_scale=ch_scale and not epi.get("pow11"),
             **extra, **epi)
    if c.cin_pad and c.in_stride is None and c.cin_pad > rup(cin, 8):
        c = replace(c, in_stride=rup(cin, 8))                # K tail: the channels past in_stride are not in memory
    return c


_E_DECONV = [dict(), dict(out_f32=True, relu=False), dict(tma=True)]   # (TMA store: not for the transposed conv)
# the x-paired conv: a per-image bias and 1.1 ** channel 0 index the packed 64-channel row (both pixels of a pair), which
# has no meaning on the dense tensor; the engine uses neither with it
_E_XPAIR = [dict(), dict(residual=True), dict(tma=True), dict(out_f32=True, relu=False),
            dict(out_f32=True, relu=False, residual=True)]


def _fill_specs():
    """Channel configurations for the combinations the hand-picked ones miss, cheapest first (fp64 reference cost):
    1x1 and 3x3 stride-1 convs with cin_pad in steps of 16 and the output widths at which the plan changes (nsub 64 /
    128 for the TMA store, 80..112 for NT = 128 without it, 144..384 for N splits), and stride-2 x-paired widths."""
    couts = [16, 32, 48, 64, 80, 96, 112, 128, 144, 192, 240, 256, 272, 384]
    specs = [("conv", cin, cout, k, 1, {}) for cin in range(16, 2049, 16) for cout in couts for k in (1, 3)]
    specs += [("s2x", 32, cout, 3, 2, {}) for cout in couts]
    return sorted(specs, key=lambda sp: sp[1] * sp[2] * sp[3] * sp[3])


def _build_matrix():
    """The hand-picked channel configurations x epilogues x types, then the fill configurations; a case is kept when it
    reaches a combination (tests/conv_plan_ref.combination) no earlier case reached -- the forms with their own packing
    keep every case of their hand-picked configurations."""
    seen, out, gi = set(), [], 0
    for fill in (False, True):
        for dts, specs, epis in (((BF16, F16), _S16, _E16), ((TF32,), _S32, _E32)):
            for spec in (_fill_specs() if fill else specs):
                if fill and dts == (TF32,) and spec[0] == "s2x":
                    continue
                for epi in {"deconv": _E_DECONV, "xpair": _E_XPAIR}.get(spec[0], epis):
                    for dt in dts:
                        c = _case(dt, spec, epi, gi, ch_scale=gi % 2 == 1)
                        try:
                            combo = R.combination(R.prepare(conv_args(c)))
                        except R.Rejected:
                            if not fill:
                                raise
                            continue          # (fill configurations past a form's limits)
                        if combo in seen and (fill or spec[0] == "conv"):
                            continue
                        seen.add(combo)
                        out.append(c)
                        gi += 1
    return out


# past one tile per SM: 396 virtual tiles = 3 per CTA on 132 SMs (ping-pong team barriers wrap an odd number of times),
# or 296 = 2 or 3 per CTA; the fp64 references of these run on full-size maps
TILE_CASES = [
    Case(BF16, "conv", 3, 176, 192, 64, 64, 3, 1, residual=True),                      # PATCH|RESIDENT|P1 / 64, ping-pong
    Case(F16, "conv", 2, 144, 176, 64, 144, 1, 1, ch_scale=True),                      # RESIDENT / 128, ping-pong, N split
    Case(BF16, "deconv", 37, 16, 16, 64, 144, 4, 2),                                   # DECONV / 128, N split, parities
    Case(F16, "deconv", 37, 16, 16, 64, 32, 4, 2, out_stride=48),
    Case(TF32, "conv", 3, 176, 192, 32, 16, 3, 1, out_f32=True, residual=True),        # tf32 P1 resident, ping-pong
    Case(BF16, "xpair", 3, 176, 384, 32, 32, 3, 1, residual=True),
    Case(F16, "s2x", 3, 352, 384, 32, 16, 3, 2, ch_scale=True),
    Case(BF16, "conv", 3, 176, 192, 32, 80, 3, 1, tma=False, residual=True),           # CK = 32 PATCH|RESIDENT ping-pong
]

MATRIX = _build_matrix() + TILE_CASES


# ------------------------------------------------------------------------------------------------------------ runner
def _pack(w, cb, bn, cin_pad, cout_pad, dt):
    """acr_b200_pack_conv -> (words [cout_pad][k*k][cin_pad] (uint16, float32 for TF32), fp32 bias[cout_pad])."""
    from tests.pack_ref import word_type
    w = np.ascontiguousarray(w, np.float32)
    cout, cin, k, _ = w.shape
    wp = np.zeros((cout_pad, k * k, cin_pad), word_type(dt))
    bias = np.zeros(cout_pad, np.float32)
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in [w, cb] + list(bn or [None] * 4)]
    q = lambda a: None if a is None else a.ctypes.data
    L.check(L.load().acr_b200_pack_conv(*(q(a) for a in keep), 1e-5, cout, cin, k, cout_pad, cin_pad, dt,
                                        wp.ctypes.data, bias.ctypes.data), "pack_conv")
    return wp, bias


_ENGINES = {}


def _engine(dt):
    from acr_b200.engine import Engine
    if dt not in _ENGINES:
        _ENGINES[dt] = Engine(None, 1, "cpu", act_dtype=torch.bfloat16 if dt == BF16 else torch.float16, dry_run=True)
    return _ENGINES[dt]


def _traced(fn):
    """Runs fn under torch.profiler (CUDA activity) -> the conv_tc_kernel launches recorded: [(key, grid, smem)].
    A session now and then delivers no activity record for its one launch (on an H100: 3 of 632 sessions in one run, one
    case three times in a row in another); fn is then run again, at most four times, after a pause -- the conv is
    deterministic and overwrites its output."""
    for attempt in range(5):
        if attempt:
            time.sleep(0.2 * attempt)
        out = _trace_once(fn)
        if out:
            return out
    return out


def _trace_once(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    out = []
    for e in ev:
        m = re.search(r"conv_tc_kernel<(\d+), ([\w:]+), (\d+), (\d+)>", e.get("name", ""))
        if m and e.get("cat") == "kernel":
            a = e.get("args", {})
            out.append(((m.group(2), int(m.group(1)), int(m.group(3)), int(m.group(4))), a.get("grid"), a.get("shared memory")))
    return out


def run_case(c: Case):
    """-> dict(got, exp, acc, tdt, guards_ok, pad_ok, foreign_ok, launches)."""
    from tests import pack_ref as P
    from tests.tf32_ref import act_round
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    a = conv_args(c)
    cin_pad, in_stride, cout_pad = a.cin_pad, a.in_stride, a.cout_pad
    tf32 = c.dt == TF32
    sdt = torch.float32 if tf32 else (torch.bfloat16 if c.dt == BF16 else torch.float16)   # storage type
    esz = 4 if tf32 else 2
    out_stride = a.out_stride
    odt = torch.float32 if c.out_f32 else sdt
    oesz = 4 if c.out_f32 else 2
    cin = c.cin
    # ---- operands (input NCHW fp32 before storage rounding)
    x = torch.randn(c.B, cin, c.H, c.W, generator=g)
    if c.ch_scale:
        x = x * torch.exp2(torch.round(torch.linspace(-6, 6, cin))).view(1, cin, 1, 1)
    bn = [torch.rand(c.cout, generator=g) + 0.5, torch.randn(c.cout, generator=g) * 0.1,
          torch.randn(c.cout, generator=g) * 0.1, torch.rand(c.cout, generator=g) + 0.5]
    bnn = [t.numpy() for t in bn]
    Ho, Wo = (a.out_H, a.out_W) if c.form not in ("xpair", "s2x") else (a.out_H, 2 * a.out_W if c.form == "xpair" else a.out_W)
    if c.form == "deconv":
        w = torch.randn(cin, c.cout, 4, 4, generator=g) * (2.0 / (cin * 4)) ** 0.5
        from acr_b200.engine import deconv_parity_weights
        par = deconv_parity_weights(w.numpy())
        wps = [_pack(par[p], None, bnn, cin_pad, cout_pad, c.dt)[0] for p in range(4)]
        _, bias = _pack(par[0], None, bnn, cin_pad, cout_pad, c.dt)
        wp = np.stack(wps)
        wq, bq = P.pack_conv_ref(w.numpy(), None, bnn, c.dt, scale_axis=1)
    else:
        w = torch.randn(c.cout, cin, c.k, c.k, generator=g) * (2.0 / (cin * c.k * c.k)) ** 0.5
        cb = torch.randn(c.cout, generator=g) * 0.1
        if c.form in ("xpair", "s2x"):
            from acr_b200.engine import _Blob
            sd = {"c.weight": w.numpy(), "c.bias": cb.numpy(), **{f"b.{n}": t for n, t in
                                                                   zip(("weight", "bias", "running_mean", "running_var"), bnn)}}
            blob = _Blob()
            w_off, b_off = _engine(c.dt)._pack_conv(sd, blob, "c", "b", True, 64, cout_pad, pair=c.form == "xpair",
                                                    s2x=c.form == "s2x")
        else:
            wp, bias = _pack(w.numpy(), cb.numpy(), bnn, cin_pad, cout_pad, c.dt)
        wq, bq = P.pack_conv_ref(w.numpy(), cb.numpy(), bnn, c.dt)
    wf = torch.from_numpy(P.words_to_f64(wq, c.dt))
    # input as stored: NHWC, in_stride channels (the x-paired forms: dense 32 channels)
    xs = torch.zeros(c.B, c.H, c.W, in_stride if c.form not in ("xpair", "s2x") else cin, dtype=sdt)
    xs[..., :cin] = x.permute(0, 2, 3, 1).to(sdt)
    xf = xs[..., :cin].float().permute(0, 3, 1, 2).contiguous()
    res = None
    if c.residual:
        res = torch.randn(c.B, c.cout, Ho, Wo, generator=g)
        rs = torch.zeros(c.B, Ho, Wo, cout_pad if c.form != "xpair" else c.cout, dtype=sdt)
        rs[..., :c.cout] = res.permute(0, 2, 3, 1).to(sdt)
        res = rs[..., :c.cout].float().permute(0, 3, 1, 2).contiguous()
    bimg = None
    if c.bias_img:
        bimg = torch.zeros(c.B, cout_pad)
        bimg[:, :c.cout] = torch.randn(c.B, c.cout, generator=g) * 0.1
    # ---- arena: [x | residual | guard | out | guard | per-image bias]
    off_r = rup(xs.numel() * esz, 1024)
    off_o = rup(off_r + (rs.numel() * esz if c.residual else 0), 1024) + GUARD
    if c.form == "xpair":
        onum = c.B * Ho * Wo * c.cout                          # dense 32-channel output = (H, W/2, 64) pairs
    else:
        onum = c.B * Ho * Wo * out_stride
    obytes = onum * oesz
    off_b = rup(off_o + obytes + GUARD, 1024)
    arena = torch.zeros(off_b + c.B * cout_pad * 4 + 1024, dtype=torch.uint8)
    arena[:xs.numel() * esz] = xs.view(torch.uint8).flatten()
    if c.residual:
        arena[off_r: off_r + rs.numel() * esz] = rs.view(torch.uint8).flatten()
    arena[off_o - GUARD: off_o + obytes + GUARD] = 0xFF                   # NaN in bf16, fp16 and fp32
    if bimg is not None:
        arena[off_b: off_b + bimg.numel() * 4] = bimg.view(torch.uint8).flatten()
    before = arena[off_o - GUARD: off_o + obytes + GUARD].clone()
    # ---- the op
    tdt_rec = L.DT_F32 if tf32 else c.dt
    op = L.Op()
    op.kind, op.n_in = L.OP_CONV, 2 if c.residual else 1
    if c.form == "xpair":
        op.in_[0] = ctensor(0, 64, c.H, c.W // 2, 64, tdt_rec)
        if c.residual:
            op.in_[1] = ctensor(off_r, 64, Ho, Wo // 2, 64, tdt_rec)
        op.out = ctensor(off_o, 64, Ho, Wo // 2, 64, L.DT_F32 if c.out_f32 else tdt_rec)
    elif c.form == "s2x":
        op.in_[0] = ctensor(0, 64, c.H, c.W // 2, 64, tdt_rec)
        if c.residual:
            op.in_[1] = ctensor(off_r, c.cout, Ho, Wo, cout_pad, tdt_rec)
        op.out = ctensor(off_o, c.cout, Ho, Wo, out_stride, L.DT_F32 if c.out_f32 else tdt_rec)
    else:
        op.in_[0] = ctensor(0, cin, c.H, c.W, in_stride, tdt_rec)
        if c.residual:
            op.in_[1] = ctensor(off_r, c.cout, Ho, Wo, cout_pad, tdt_rec)
        op.out = ctensor(off_o, c.cout, Ho, Wo, out_stride, L.DT_F32 if c.out_f32 else tdt_rec)
    if c.bias_img:
        op.aux[0] = ctensor(off_b, cout_pad, 1, 1, cout_pad, L.DT_F32)
    op.k, op.stride, op.relu, op.has_residual = a.k, a.stride, int(c.relu), int(c.residual)
    op.cin_pad, op.cout_pad = cin_pad, cout_pad
    op.shift[0] = ((c.xflags if c.form == "xpair" else 0) | (L.CONV_S2X if c.form == "s2x" else 0) |
                   (L.CONV_DECONV if c.form == "deconv" else 0) | (L.CONV_BIAS_PER_IMAGE if c.bias_img else 0) |
                   (L.CONV_POW11_CH0 if c.pow11 else 0))
    if c.form in ("xpair", "s2x"):
        blob_bytes = np.frombuffer(blob.tobytes(), np.uint8).copy()
    else:
        pad = (-wp.nbytes) % 256
        blob_bytes = np.concatenate([wp.view(np.uint8).reshape(-1), np.zeros(pad, np.uint8), bias.view(np.uint8)])
        w_off, b_off = 0, wp.nbytes + pad
    op.w_offset[0], op.w_offset[1] = w_off, b_off
    d_arena = arena.cuda()
    d_blob = torch.from_numpy(blob_bytes).cuda()
    old = os.environ.get("ACR_B200_TMA_OUT")
    os.environ["ACR_B200_TMA_OUT"] = "1" if c.tma else "0"      # read when the plan is made, inside run_op
    try:
        launches = _traced(lambda: L.check(L.load().acr_b200_run_op(
            C.byref(op), c.B, d_arena.data_ptr(), d_blob.data_ptr(), None, c.dt,
            torch.cuda.current_stream().cuda_stream), "run_op"))
    finally:
        if old is None:
            del os.environ["ACR_B200_TMA_OUT"]
        else:
            os.environ["ACR_B200_TMA_OUT"] = old
    after = d_arena[off_o - GUARD: off_o + obytes + GUARD].cpu()
    guards_ok = bool(torch.equal(after[:GUARD], before[:GUARD]) and torch.equal(after[-GUARD:], before[-GUARD:]))
    raw_out = after[GUARD: GUARD + obytes]
    if c.form == "xpair":
        o = raw_out.view(odt).view(c.B, Ho, Wo, c.cout)
        pad_ok, foreign_ok = True, True
        got = o.float().permute(0, 3, 1, 2)
    else:
        o = raw_out.view(odt).view(c.B, Ho, Wo, out_stride)
        own = c.cout if c.form == "deconv" else cout_pad       # the transposed conv's slice: channels past cout
        pad_ok = bool((o[..., c.cout:cout_pad].float() == 0).all())
        foreign = o[..., own:].contiguous().view(torch.uint8) if own < out_stride else torch.zeros(0, dtype=torch.uint8)
        foreign_ok = bool((foreign == 0xFF).all())
        got = o[..., :c.cout].float().permute(0, 3, 1, 2)
    # ---- fp64 expectation
    xe = act_round(xf) if tf32 else xf
    u_acc = P.U_ACC_TC
    if c.form == "deconv":
        exp, acc = P.conv_with_bound(xe, wf, torch.from_numpy(bq), 2, u_acc, relu=c.relu, deconv=True)
    else:
        b = bimg[:, :c.cout, None, None] if c.bias_img else torch.from_numpy(bq)
        exp, acc = P.conv_with_bound(xe, wf, b, a.stride, u_acc, residual=res, pow11=c.pow11, relu=c.relu)
    return dict(got=got, exp=exp, acc=acc, tdt=odt, guards_ok=guards_ok, pad_ok=pad_ok, foreign_ok=foreign_ok,
                launches=launches)


@pytest.mark.parametrize("case", MATRIX, ids=lambda c: c.id)
def test_conv_instance(case):
    from tests.pack_ref import check_bound, direction_counts, direction_ok
    torch.set_num_threads(min(32, os.cpu_count()))
    plan = R.prepare(conv_args(case), torch.cuda.get_device_properties(0).multi_processor_count)
    r = run_case(case)
    worst, n_bad = check_bound(r["got"], r["exp"], r["acc"], r["tdt"])
    if r["tdt"] == torch.float32:
        (toward, away) = (0, 0)
    else:
        (toward, away), _ = direction_counts(r["got"], r["exp"], r["acc"], r["tdt"])
    print(f"{case.id}: {R.kernel_name(plan.key)} pingpong {plan.pingpong} plain {plan.plain} tma_out {plan.tma_out} "
          f"nsplit {plan.nsplit} SA {plan.SA} SB {plan.SB} grid {plan.grid} smem {plan.smem}: worst err/bound {worst:.3f}, "
          f"decided off-RNE {toward} / {away}; trace {r['launches']}")
    assert r["guards_ok"], "bytes before or after the output were written"
    assert r["pad_ok"], "channels [cout, cout_pad) are not zero"
    assert r["foreign_ok"], "channels the op does not own were written"
    assert n_bad == 0, f"{n_bad} elements above their bound (worst err/bound {worst:.3f})"
    assert direction_ok(toward, away), f"rounding direction: {toward} toward zero vs {away} away"
    # the launch is the restated one
    assert len(r["launches"]) == 1, r["launches"]
    key, grid, smem = r["launches"][0]
    assert key == plan.key, f"launched {R.kernel_name(key)}, the plan restatement says {R.kernel_name(plan.key)}"
    assert grid is not None and list(grid) == [plan.grid, 1, 1], f"grid {grid}, restated {plan.grid}"
    assert smem is not None and smem == plan.smem, f"dynamic shared memory {smem}, restated {plan.smem}"

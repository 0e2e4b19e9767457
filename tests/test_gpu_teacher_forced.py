"""GPU parity, teacher forced: EVERY launch of the network plan is compared with the oracle's restatement of
that op (oracle/op_ref.py, unrounded fp32 parameters) applied to the plan's OWN stored inputs.  No error
accumulates from op to op and the seeded random network cannot amplify storage round-off, so the bound is
the per-op one: storage rounding of weights and of the one output (2^-7 of the op's output range for bf16,
2^-10 for fp16, 2e-5 for the fp32 validation plan).  This pins fuse layers, bilinear up-sampling, coord
channels, every head stack, the attention pooling, the part head and the folded final conv individually --
a wrong align_corners, BN eps, coord formula, tap order or weight key shows up as an O(1) error of ONE op.

On top of that max-norm check, every conv, fuse, bilinear and coord op is held per ELEMENT to an fp64 bound
(tests/pack_ref.py), so a small channel or a small value near a ReLU zero cannot hide under the op's largest value: the
exact result of the plan's stored inputs and of the weights the conv kernel reads (its packed words in the live weight
blob, asserted equal bit for bit to the packer's restatement), plus the accumulation bound, plus one rounding to the
output type.  So are the stems (3x3 and ResNet's 7x7, the bias pair of the tensor-core form included), the attention
pooling (its 16-bit softmax weights included) and the part head; each bound is derived next to the code that forms it."""
import os

import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10, torch.float32: 2e-5}


@pytest.fixture(scope="module")
def sd():
    from acr_b200.synth import load_bn_calibration, synth_state_dict
    return synth_state_dict(0, bn_stats=load_bn_calibration(0))


@pytest.fixture(scope="module")
def image():
    # one frame: the sweep re-computes every op on the CPU.  At batch 1 a kernel that reads another image's data reads its
    # own; the batch dimension is covered by tests/test_gpu_batch.py (every op teacher forced on three distinct frames,
    # every launch per image against batch 1)
    gi = torch.Generator().manual_seed(123)
    return torch.randint(0, 256, (2, 512, 512, 3), generator=gi, dtype=torch.uint8)[1:]


def _pare(eng, s):
    """(B,106) contact + shape offsets of side s: the part head packs them densely (106 floats per image)."""
    return eng.view(f"{s}_pare").float().cpu().reshape(-1)[: eng.batch * 106].view(eng.batch, 106)


def _out_type(eng, t):
    return torch.float32 if eng.f32 or t.dtype == "f32" else eng.act_dtype


def conv_bound(eng, i, sdn, blob, get):
    """Conv record i of the plan (``eng.recs[i]`` of the engine that built it): asserts that its packed weights in the
    live blob equal the restatement of tests/pack_ref.py bit for bit, and returns (got, fp64 exp, acc, output type) for
    the per-element bound -- the exact conv, with the weights the kernel reads, of the plan's own stored input."""
    from acr_b200 import lib as L
    from tests import pack_ref as P
    from tests.tf32_ref import act_round
    r, o = eng.recs[i], eng._cops[i]
    a = r.get("attrs", {})
    e = P.engine_conv_expectation(eng, i, sdn)
    live = P.blob_words(blob, o.w_offset[0], e["words"])
    assert np.array_equal(live.view(np.uint8), e["words"].view(np.uint8)), f"op {i}: packed weights differ from the restatement"
    if e["bias"] is not None:
        assert np.array_equal(P.blob_words(blob, o.w_offset[1], e["bias"]).view(np.uint32), e["bias"].view(np.uint32)), \
            f"op {i}: packed bias differs from the restatement"
    t = r["ins"][0]
    x = eng.view(t).float().cpu()[..., : (e["w"].shape[0] if e.get("deconv") else e["w"].shape[1])].permute(0, 3, 1, 2)
    if eng.tf32:
        x = act_round(x)                    # the conv rounds its fp32 operand to tf32 in shared memory
    # fp64 accumulation in the validation plan's CUDA-core conv; fp32 on the tensor cores / in the CUDA-core 16-bit conv
    u_acc = 2.0 ** -52 if eng.f32 and not eng.tf32 else P.U_ACC_TC
    b = e["b"]
    if b is None:                           # folded part-head conv: the per-image bias row the part head wrote
        b = torch.from_numpy(eng.view(r["aux"][0]).float().cpu().numpy().reshape(eng.batch, -1)[:, :e["w"].shape[0]])[..., None, None]
    res = get(r["ins"][1]) if a.get("residual") else None
    extra = a.get("extra")
    exp, acc = P.conv_with_bound(x, e["w"], b, a.get("s", 1), u_acc, residual=res, pow11=bool(a.get("pow11")),
                                 relu=bool(a.get("relu")) and not extra, deconv=bool(e.get("deconv")),
                                 pre_round=P.U32 if eng.f32 and not eng.tf32 else 0.0)
    if extra:   # folded fuse sum: the other terms, nearest-upsampled, added in fp32 after the conv, then ReLU
        terms = [torch.nn.functional.interpolate(get(tt).double(), scale_factor=2 ** sh, mode="nearest") if sh else get(tt).double()
                 for tt, (_, sh) in zip(r["ins"][1:], a["extra"])]
        tot = sum(tt.abs() for tt in terms)
        exp, acc = exp + sum(terms), acc + len(terms) * P.U32 * (exp.abs() + acc + tot)
        exp = torch.relu(exp) if a["relu"] else exp
    got = get(r["out"])
    n = min(got.shape[1], exp.shape[1])
    return got[:, :n], exp[:, :n], acc[:, :n], _out_type(eng, r["out"])


def _elementwise_bounds(eng, r, get):
    """(got, fp64 exp, acc) of the fuse / bilinear / coord ops, each from the plan's own stored inputs.
    fuse: the kernel sums n stored terms in fp32 in the reference's order; each of the n - 1 additions adds at most
      2^-24 of its partial sum, so acc = (n - 1) 2^-24 sum|t|; ReLU does not increase an error.
    bilinear x2 (align_corners): the kernel forms the source coordinate f = x (in - 1) / (out - 1) in fp32 (a rounded
      ratio times x: |df| <= 2 * 2^-24 f <= 2^-23 in) and interpolates with weights 1 - l, l of l = f - floor(f); each weight
      is off by at most |df| + 2^-24 and every output mixes four values with weights of at most 1, so the weights add at
      most 4 (2^-23 in + 2^-24) max|v| and the six fp32 operations of the formula 6 * 2^-24 * sum|v|; sum|v| <= 4 max|v|
      over the 3 x 3 input neighbourhood of the output's source pixel.
    coord: x / (W - 1) * 2 - 1 in fp32: the division and the subtraction each round once, |x / (W - 1)| <= 1 and the
      result is in [-1, 1], so acc = 2 * 2^-24 * 2."""
    from acr_b200 import lib as L
    from oracle import op_ref
    U = 2.0 ** -24
    a = r.get("attrs", {})
    if r["kind"] == L.OP_FUSE:
        terms = [get(t).double() for t in r["ins"]]
        up = [torch.nn.functional.interpolate(t, scale_factor=2 ** sh, mode="nearest") if sh else t
              for t, sh in zip(terms, a["shifts"])]
        exp = op_ref.fuse(terms, a["shifts"], a["relu"])
        return get(r["out"]), exp, (len(up) - 1) * U * sum(t.abs() for t in up)
    if r["kind"] == L.OP_BILINEAR2X:
        x = get(r["ins"][0]).double()
        exp = op_ref.bilinear2x(x)
        n = max(x.shape[-2:])
        loc = torch.nn.functional.max_pool2d(x.abs(), 3, 1, 1)
        loc = torch.nn.functional.interpolate(loc, scale_factor=2, mode="nearest")
        return get(r["out"]), exp, (4 * (2.0 ** -23 * n + U) + 6 * U * 4) * loc
    xc = eng.view(r["out"]).float().cpu()
    H, W = xc.shape[1], xc.shape[2]
    lx = torch.arange(W, dtype=torch.float64) / (W - 1) * 2 - 1
    ly = torch.arange(H, dtype=torch.float64) / (H - 1) * 2 - 1
    exp = torch.stack([lx.view(1, W).expand(H, W), ly.view(H, 1).expand(H, W)])[None].expand(xc.shape[0], -1, -1, -1)
    w0 = eng.spec.widths[0]
    return xc[..., w0:w0 + 2].permute(0, 3, 1, 2), exp, torch.full_like(exp, 4 * U)


def stem_bound(eng, i, sdn, blob, image):
    """(got, fp64 exp, acc, output type) of a stem record: conv1 + bn1 + ReLU on the frame, or the im2col gather.

    Every form normalises a byte b as (float)b / 255.f * 2.f - 1.f in fp32, as the reference does; the reference of this
    check starts from that fp32 value x.
    im2col (16-bit plans): stores RNE_T(x): acc = 0, the bound is the output rounding alone.
    tensor-core stem (3x3, and ResNet's 7x7): operands RNE_T(x) and the packed weights (pinned to the restatement in the
      live blob), products exact in fp32; the BN bias enters the GEMM as two 16-bit parts hi = RNE_T(b), lo = RNE_T(b - hi)
      against constant-one taps, so the sum sees hi + lo, off b by |b - hi - lo| (computed exactly, per channel); K + 2 terms
      (K = 32 or 160 channels and the pair) accumulate with the tensor cores' 2^-22 per addition.
    CUDA-core stem (fp32 storage: the validation and TF32 plans): fp32 operands x and fp32 folded weights (pinned in the
      blob), 27 fmaf (or fp64 adds) on the bias: each rounds at most 2^-24 of a partial sum, covered by 29 * 2^-22 (S + |b|)."""
    from acr_b200 import lib as L
    from tests import pack_ref as P
    r, o = eng.recs[i], eng._cops[i]
    tdt = _out_type(eng, r["out"])
    got = eng.map_nchw(r["out"]).cpu()
    if r["kind"] == L.OP_IM2COL_STEM:
        from oracle import op_ref
        return got[:, :27], op_ref.im2col_stem(image).double(), torch.zeros(1, dtype=torch.float64), tdt
    st = r["attrs"].get("stem", r["attrs"])
    x = ((image.float() / 255.0) * 2.0 - 1.0).permute(0, 3, 1, 2)          # fp32, the kernels' operation order
    w = np.asarray(sdn[st["w"] + ".weight"], np.float32)
    if r["kind"] == L.OP_STEM:                                                # fp32 weights [(ky,kx,ci)][co], fp32 bias
        wq, b = P.pack_conv_ref(w, None, P.bn_of(sdn, st["bn"]), L.DT_F32)
        words = np.ascontiguousarray(wq.transpose(2, 3, 1, 0).reshape(27, 64))
        dev, bsum = 0.0, torch.from_numpy(b).double()
    else:
        kch = 32 if w.shape[-1] == 3 else 160
        wq, b = P.pack_conv_ref(w, None, P.bn_of(sdn, st["bn"]), eng.plan_dt)
        words = P.layout_stem(wq, kch)
        x = x.to(eng.act_dtype).float()                                      # the 16-bit operand built in shared memory
        bt = torch.from_numpy(b)
        hi = bt.to(eng.act_dtype).float()
        lo = (bt - hi).to(eng.act_dtype).float()                             # b - hi is exact in fp32
        bsum = hi.double() + lo.double()
        dev = (bt.double() - bsum).abs().view(1, -1, 1, 1)
    assert np.array_equal(P.blob_words(blob, o.w_offset[0], words).view(np.uint8), words.view(np.uint8)), \
        f"op {i}: packed stem weights differ from the restatement"
    assert np.array_equal(P.blob_words(blob, o.w_offset[1], b).view(np.uint32), b.view(np.uint32)), f"op {i}: stem bias"
    wf = torch.from_numpy(P.words_to_f64(wq, eng.plan_dt if r["kind"] != L.OP_STEM else L.DT_F32))
    exp, acc = P.conv_with_bound(x, wf, bsum, 2, P.U_ACC_TC)
    exp = torch.relu(exp + (torch.from_numpy(b).double().view(1, -1, 1, 1) - bsum.view(1, -1, 1, 1)))
    return got, exp, acc + dev, tdt


def pool_bounds(eng, pool_in, get):
    """(label, got, fp64 exp, acc) of the attention pooling, from the plan's stored features f (B,256,HW) and logits l
    (parts 1..32 at every other pixel): exact softmax a_p = exp(l_p - M) / Z, E = sum_p a_p f_p.

    What the kernels use instead of exp(l_p - M): per chunk of pixels exp(l_p - m_c) by __expf (2 + 1.173 |x| ulp, CUDA C
    Programming Guide), rounded to the storage type T (relative 2^-8 bf16, 2^-11 fp16, 0 for the fp32 plans; an fp16
    weight below 2^-14 loses up to tau = 2^-25 absolutely), then scaled by expf(m_c - M) (2 ulp) / S (1/2 ulp).  So each
    effective weight is Z a_p (1 + e_p) + t_p with |e_p| <= eta, |t_p| <= tau, the same weights in the numerator and the
    denominator, and
        |pooled - E| <= (eta sum_p a_p |f_p - E| + tau / Z sum_p |f_p - E|) / (1 - eta - HW tau / Z)
    plus the fp32 accumulation of the HW products and the 2 * chunks merge steps and of the denominator:
    (HW + 2 chunks + 8) 2^-22 (sum_p a_p |f_p| + |E|).  eta also takes the rounding of the exponent arguments (R 2^-24 each
    for the two of them, R = max l - min l of the part)."""
    from acr_b200.engine import POOL_CHUNKS
    f = get(pool_in[0]).double()
    B, C = f.shape[:2]
    f = f.reshape(B, C, -1)
    l = get(pool_in[1])[:, 1:33, ::2, ::2].double().reshape(B, 32, -1)
    HW = l.shape[-1]
    M = l.amax(-1, keepdim=True)
    w = torch.exp(l - M)
    Z = w.sum(-1, keepdim=True)                                               # (B, 32, 1)
    a = w / Z
    E = torch.einsum("bjp,bcp->bcj", a, f)
    R = (M - l.amin(-1, keepdim=True)).squeeze(-1)                            # (B, 32)
    u16 = 0.0 if eng.f32 else (2.0 ** -8 if eng.act_dtype == torch.bfloat16 else 2.0 ** -11)
    tau = 2.0 ** -25 if eng.act_dtype == torch.float16 else 2.0 ** -126
    eta = u16 + (2 + 1.173 * R) * 2.0 ** -23 + 2 * 2.0 ** -23 + 2.0 ** -24 + 2 * R * 2.0 ** -24
    T1, T2 = torch.empty(B, C, 32, dtype=torch.float64), torch.empty(B, C, 32, dtype=torch.float64)
    for j in range(32):
        d = (f - E[:, :, j:j + 1]).abs()
        T1[:, :, j], T2[:, :, j] = (d * a[:, j:j + 1, :]).sum(-1), d.sum(-1)
    eta_, tz = eta[:, None, :], tau / Z.squeeze(-1)[:, None, :]
    acc = (eta_ * T1 + tz * T2) / (1 - eta_ - HW * tz)
    acc = acc + (HW + 2 * POOL_CHUNKS + 8) * 2.0 ** -22 * (torch.einsum("bjp,bcp->bcj", a, f.abs()) + E.abs())
    pooled = eng.view("pooled").float().cpu().view(B, 256, 32)
    return pooled, E, acc


def part_head_bounds(eng, pooled, sdf):
    """[(label, got, fp64 exp, acc)] of the part head, from the stored pooled feature (fp32): the contact offsets (256
    fmaf), the shape features W pooled + b (256 fmaf, error A each) and Linear(1024 -> 10) on them (1024 fmaf and shuffle
    sums: |Lw| A + 1026 * 2^-22 (|Lw| |sf| + |lb|)), and the per-image bias b + W[:, 112:] . pare of the folded final conv
    (106 fmaf; the pare it reads is the stored one).  Each fp32 operation rounds at most 2^-24 of a partial sum; 2^-22 per
    term covers that with room for the summation order."""
    U = 2.0 ** -22
    B = eng.batch
    p = pooled.double()
    out = []
    ws_w, ws_b = sdf["cam_shape_layers.1.0.weight"].double()[:, :, 0, 0], sdf["cam_shape_layers.1.0.bias"].double()
    ws = torch.einsum("oc,bcj->boj", ws_w, p) + ws_b.view(1, -1, 1)
    A = 258 * U * (torch.einsum("oc,bcj->boj", ws_w.abs(), p.abs()) + ws_b.abs().view(1, -1, 1))
    for s in "lr":
        sl, li = (slice(16, 32), 2) if s == "l" else (slice(0, 16), 3)
        lw = sdf[f"contact_layers.{li}.weight"].double()[0, :, :, :, 0, 0]      # (6,256,16)
        off = torch.einsum("bcj,ocj->boj", p[:, :, sl], lw).transpose(1, 2).reshape(B, 96)
        off_a = 258 * U * torch.einsum("bcj,ocj->boj", p[:, :, sl].abs(), lw.abs()).transpose(1, 2).reshape(B, 96)
        Lw, Lb = sdf[f"cam_shape_layers.{li}.weight"].double(), sdf[f"cam_shape_layers.{li}.bias"].double()
        x, xa = ws[:, :, sl].reshape(B, -1), A[:, :, sl].reshape(B, -1)
        sh = x @ Lw.T + Lb
        sh_a = xa @ Lw.abs().T + 1026 * U * (x.abs() @ Lw.abs().T + Lb.abs())
        pare = _pare(eng, s)
        out.append((f"part head {s}", pare, torch.cat([off, sh], 1), torch.cat([off_a, sh_a], 1)))
        ci = 4 if s == "l" else 5
        Wf, bf = sdf[f"contact_layers.{ci}.weight"].double().reshape(109, 218)[:, 112:], sdf[f"contact_layers.{ci}.bias"].double()
        pd = pare.double()
        bias = eng.view(f"{s}_bias_img").float().cpu().reshape(-1)[: B * 112].view(B, 112)[:, :109]
        out.append((f"part head {s} per-image bias", bias, pd @ Wf.T + bf, 108 * U * (pd.abs() @ Wf.abs().T + bf.abs())))
    return out


def _report_bounds(brows):
    """Prints the worst err / bound per op class, the rounding directions and the per-channel scale spread; asserts."""
    from tests.pack_ref import direction_ok
    by = {}
    for cls, i, label, worst, nbad, (tw, aw), (ta, aa), spread in brows:
        w = by.setdefault(cls, [0.0, 0, 0, 0, 0, 0, 1.0, 0])
        by[cls] = [max(w[0], worst), w[1] + nbad, w[2] + tw, w[3] + aw, w[4] + ta, w[5] + aa, min(w[6], spread), w[7] + 1]
    for cls, (worst, nbad, tw, aw, ta, aa, spread, n) in sorted(by.items()):
        print(f"  bound {cls}: {n} checks, worst err/bound {worst:.3f}, off-RNE toward zero / away: decided {tw} / {aw}, "
              f"all {ta} / {aa}; smallest channel max / op max {spread:.2e}")
    bad = [(i, l, f"{w:.3f}", nb) for _, i, l, w, nb, _, _, _ in brows if nb]
    assert not bad, f"{len(bad)} ops with elements above the per-element fp64 bound: {bad[:8]}"
    skew = [(i, l, tw, aw) for _, i, l, _, _, (tw, aw), _, _ in brows if not direction_ok(tw, aw)]
    assert not skew, f"rounding direction skewed (toward zero, away) in {len(skew)} ops: {skew[:8]}"


def sweep(eng, sd, image, tol):
    """-> list of (op index, description, rel err).  Asserts the per-element fp64 bound of every launch (conv and stem
    weights pinned to the restatement in the live blob) but the ResNet max-pool (bit-exact in tests/test_gpu_resnet.py),
    and that no 16-bit output whose rounding the bound decides is off round-to-nearest;
    the max-norm errors it returns are asserted by the caller."""
    from acr_b200 import lib as L
    from oracle import op_ref
    from tests.pack_ref import check_bound, direction_counts
    sdf = {k: v.float() for k, v in sd.items() if v.dtype.is_floating_point}
    sdn = {k: v.numpy() for k, v in sdf.items()}
    blob = eng.weights.cpu().numpy()
    base = getattr(eng, "_eng", eng)            # test_gpu_resnet views the engine without some records
    rec_index = {id(r): j for j, r in enumerate(base.recs)}
    get = lambda t: eng.map_nchw(t).cpu()
    rows, brows = [], []
    pool_in = None
    for i, r in enumerate(eng.recs):
        kind, a = r["kind"], r.get("attrs", {})
        bchecks = []     # (class, label, got, fp64 expected, acc, output type)
        if kind in (L.OP_CONV, L.OP_CONV_REF):
            cls = "conv " + ("stem im2col" if "stem" in a else "folded part-head" if "fold_side" in a else
                             "merged" if a.get("merged") else "fuse-folded" if a.get("extra") else "x-paired"
                             if base._cops[rec_index[id(r)]].shift[0] & 4 else "s2x" if base._cops[rec_index[id(r)]].shift[0] & 8 else
                             f"k{a['k']} s{a['s']}" + (" pow11" if a.get("pow11") else ""))
            got, exp, acc, tdt = conv_bound(base, rec_index[id(r)], sdn, blob, get)
            bchecks.append((cls, f"conv {a.get('w', a.get('stem', a.get('fold_side')))}", got, exp, acc, tdt))
        elif kind in (L.OP_FUSE, L.OP_BILINEAR2X, L.OP_COORD):
            cls = {L.OP_FUSE: "fuse", L.OP_BILINEAR2X: "bilinear x2", L.OP_COORD: "coord"}[kind]
            got, exp, acc = _elementwise_bounds(eng, r, get)
            bchecks.append((cls, cls, got, exp, acc, _out_type(eng, r["out"])))
        elif kind in (L.OP_STEM, L.OP_STEM_TC, L.OP_IM2COL_STEM):
            cls = {L.OP_STEM: "stem (CUDA cores)", L.OP_STEM_TC: "stem (tensor cores)", L.OP_IM2COL_STEM: "stem im2col"}[kind]
            got, exp, acc, tdt = stem_bound(base, rec_index[id(r)], sdn, blob, image)
            bchecks.append((cls, cls, got, exp, acc, tdt))
        elif kind == L.OP_PARTHEAD:
            got, exp, acc = pool_bounds(eng, pool_in, get)
            bchecks.append(("attention pooling", "attention pooling", got, exp, acc, torch.float32))
            for label, got, exp, acc in part_head_bounds(eng, got, sdf):
                bchecks.append(("part head" + (" per-image bias" if "bias" in label else ""), label, got, exp, acc, torch.float32))
        for cls, label, got, exp, acc, tdt in bchecks:
            worst, nbad = check_bound(got, exp, acc, tdt)
            dirs = ((0, 0), (0, 0)) if tdt == torch.float32 else direction_counts(got, exp, acc, tdt)
            ch = exp.abs().amax(dim=[d for d in range(exp.dim()) if d != 1])
            spread = float(ch[ch > 0].min() / ch.max()) if bool((ch > 0).any()) else 1.0
            brows.append((cls, i, label, worst, nbad, dirs[0], dirs[1], spread))
        checks = []      # (label, got, expected)
        if kind in (L.OP_CONV, L.OP_CONV_REF):
            if "stem" in a:
                checks.append(("stem 27->64 1x1 on im2col", get(r["out"]), op_ref.stem_from_cols(get(r["ins"][0])[:, :27], sdf)))
            elif "fold_side" in a:
                s = a["fold_side"]
                raw = eng.view(r["ins"][0]).float().cpu()                      # (B,64,64,128): params 0..105, cam 112..114
                prm, cam = raw[..., :106].permute(0, 3, 1, 2), raw[..., 112:115].permute(0, 3, 1, 2)
                pare = _pare(eng, s)
                checks.append((f"contact_layers[{'4' if s == 'l' else '5'}] folded 218->109", get(r["out"]),
                               op_ref.final_params(prm, cam, pare, sdf, s)))
            elif a.get("merged"):          # convs on the same input run as one wide conv: every slice against its own conv
                x, got, each = get(r["ins"][0]), get(r["out"]), a["merged"]
                for j, (wk, bk) in enumerate(zip(a["w"], a["bn"])):
                    checks.append((f"conv {wk} (slice {j} of a merged conv)", got[:, j * each:(j + 1) * each],
                                   op_ref.conv_bn_act(x, sdf, wk, bk, a["s"], a["relu"])))
            elif a.get("extra"):           # a fuse sum folded into the conv that produces one of its terms
                conv = op_ref.conv_bn_act(get(r["ins"][0]), sdf, a["w"], a["bn"], a["s"], False)
                others, shifts, pos = [get(t) for t in r["ins"][1:]], [sh for _, sh in a["extra"]], a["extra_pos"]
                exp = op_ref.fuse(others[:pos] + [conv] + others[pos:], shifts[:pos] + [0] + shifts[pos:], a["relu"])
                checks.append((f"conv {a['w']} + folded fuse sum of {len(others) + 1} terms", get(r["out"]), exp))
            else:
                res = get(r["ins"][1]) if a["residual"] else None
                exp = op_ref.conv_bn_act(get(r["ins"][0]), sdf, a["w"], a["bn"], a["s"], a["relu"], res, a["pow11"])
                checks.append((f"conv {a['w']} k{a['k']} s{a['s']}", get(r["out"]), exp))
        elif kind == L.OP_STEM:
            checks.append(("stem (CUDA-core form)", get(r["out"]), op_ref.stem(image, sdf)))
        elif kind == L.OP_STEM_TC:
            checks.append(("stem (wgmma, operand built in shared memory)", get(r["out"]), op_ref.stem(image, sdf)))
        elif kind == L.OP_IM2COL_STEM:
            checks.append(("im2col of the normalised frame", get(r["out"])[:, :27], op_ref.im2col_stem(image)))
        elif kind == L.OP_FUSE:
            checks.append((f"fuse x{len(r['ins'])}", get(r["out"]), op_ref.fuse([get(t) for t in r["ins"]], a["shifts"], a["relu"])))
        elif kind == L.OP_BILINEAR2X:
            checks.append(("bilinear x2", get(r["out"]), op_ref.bilinear2x(get(r["ins"][0]))))
        elif kind == L.OP_COORD:
            xc = eng.view(r["out"]).float().cpu()
            exp = op_ref.coord(xc.shape[1], xc.shape[2])[None].expand(xc.shape[0], -1, -1, -1)
            w0 = eng.spec.widths[0]
            checks.append(("coord channels", xc[..., w0:w0 + 2].permute(0, 3, 1, 2), exp))
            assert float(xc[..., w0 + 2:].abs().max()) == 0.0, "pad channels of the coord concat are not zero"
        elif kind == L.OP_POOL:
            pool_in = r["ins"]                                                  # partials are checked after the merge
        elif kind == L.OP_PARTHEAD:
            B = eng.batch
            pooled = eng.view("pooled").float().cpu().view(B, 256, 32)
            checks.append(("attention pooling (softmax over HW x features)", pooled,
                           op_ref.attention_pool(get(pool_in[0]), get(pool_in[1]))))
            for s in "lr":
                pare = _pare(eng, s)
                checks.append((f"part head {s}: LocallyConnected2d + Linear", pare, op_ref.part_offsets(pooled, sdf, s)))
        else:
            raise AssertionError(f"op kind {kind} has no teacher-forced check")
        for label, got, exp in checks:
            assert torch.isfinite(got).all(), (i, label)
            rows.append((i, label, rel_err(got.numpy(), exp.numpy())))
    _report_bounds(brows)
    return rows


def _run(sd, image, dtype, widths=None):
    from acr_b200.engine import Engine
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs (measured 40x slower at 128)
    eng = Engine(sd, image.shape[0], "cuda", dtype, reuse_memory=False, widths=widths)   # every intermediate tensor is kept
    eng.run(image.cuda())
    torch.cuda.synchronize()
    rows = sweep(eng, sd, image, TOL[dtype])
    worst = sorted(rows, key=lambda r: -r[2])[:5]
    print(f"teacher-forced sweep {dtype}: {len(rows)} checks over {len(eng.recs)} launches; worst:",
          [(i, l, f"{e:.2e}") for i, l, e in worst])
    assert len(rows) >= len(eng.recs) - 1
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[dtype]]
    assert not bad, f"{len(bad)} ops above {TOL[dtype]:.2e}: {bad[:8]}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_every_op_teacher_forced_16bit(sd, image, dtype):
    """The product plans (wgmma conv, x-paired 32-channel convs, tensor-core stem and pooling)."""
    _run(sd, image, dtype)


def test_every_op_teacher_forced_with_folded_fuse_sums(sd, image, monkeypatch):
    """Opt-in plan (ACR_B200_FOLD_FUSE=1): the fuse sums of the coarser HR-module outputs computed in the epilogue of the
    stride-2 conv that produces one of their terms (extra terms nearest-upsampled in the epilogue)."""
    monkeypatch.setenv("ACR_B200_FOLD_FUSE", "1")
    _run(sd, image, torch.bfloat16)


def test_every_op_teacher_forced_fp32_validation_plan(sd, image):
    """The fp32 validation plan (model_precision='fp32'): fp32 storage, fp64 accumulate."""
    _run(sd, image, torch.float32)


def test_every_op_teacher_forced_hrnet_w48(image):
    """The HRNet-W48 trunk of BASELINE configs[4]: the reference has no such network (parity unpinned: no golden can
    exist), so every launch of its plan is pinned against the oracle's per-op restatement instead -- 48/96/192/384-
    channel convs (zero-filled K tails, N split at 384 outputs), fuse layers, heads on the 50-channel coord concat."""
    from acr_b200.netspec import WIDTHS_W48, build_acr_spec
    from acr_b200.synth import synth_state_dict
    sd48 = synth_state_dict(3, spec=build_acr_spec(512, widths=WIDTHS_W48))
    _run(sd48, image, torch.bfloat16, widths=WIDTHS_W48)


def test_heads_only_plan_teacher_forced(sd, image):
    """The ACR.head_forward plan (ops after the trunk) on an external feature."""
    from acr_b200.engine import Engine
    from oracle import net_ref
    torch.set_num_threads(min(32, os.cpu_count()))   # > 64 threads oversubscribe these small convs (measured 40x slower at 128)
    x = net_ref._Net(sd).backbone(image)
    eng = Engine(sd, 1, "cuda", torch.bfloat16, reuse_memory=False, head_only=True)
    eng.run_heads(x.cuda())
    torch.cuda.synchronize()
    rows = sweep(eng, sd, image, TOL[torch.bfloat16])
    bad = [(i, l, e) for i, l, e in rows if not e <= TOL[torch.bfloat16]]
    assert len(rows) >= 55 and not bad, bad[:8]

"""The conv weight packer, bit for bit: acr_b200_pack_conv and every engine form built on it (x-paired, stride-2 x-paired,
transposed conv, merged convs, the folded part-head conv, the 3x3 and 7x7 stems) against the numpy restatement of
tests/pack_ref.py -- BN folded in the packer's fp32 order, then rounded to nearest even (bf16 / fp16) or to the nearest
tf32 with ties away from zero (TF32).  The conv tests on the GPU take these words as their reference, so a packer that
truncated or double-rounded would otherwise go unseen: its bias stays below their tolerances."""
import numpy as np
import pytest

from acr_b200 import lib as L
from tests import pack_ref as P
from tests.helpers import pack_conv_host

DTS = [L.DT_BF16, L.DT_F16, L.DT_TF32, L.DT_F32]
DT_IDS = ["bf16", "f16", "tf32", "f32"]


def _host_pack(w, cb, bn, cin_pad, cout_pad, dt):
    """acr_b200_pack_conv into a buffer of the storage type (tests.helpers.pack_conv_host holds 16-bit words only)."""
    lib = L.load()
    cout, cin, k, _ = w.shape
    wp = np.zeros((cout_pad, k * k, cin_pad), P.word_type(dt))
    bias = np.zeros(cout_pad, np.float32)
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in [w, cb] + list(bn or [None] * 4)]
    q = lambda a: None if a is None else a.ctypes.data
    L.check(lib.acr_b200_pack_conv(q(keep[0]), q(keep[1]), q(keep[2]), q(keep[3]), q(keep[4]), q(keep[5]), 1e-5, cout,
                                   cin, k, cout_pad, cin_pad, dt, wp.ctypes.data, bias.ctypes.data), "pack_conv")
    return wp, bias


def _rounding_values(rng, n, dt):
    """fp32 values that exercise the rounding: exact ties of the storage type (even and odd kept bits), neighbours of
    powers of two, fp16 subnormals and values at fp16's overflow threshold, plus plain normals."""
    drop = {L.DT_BF16: 16, L.DT_F16: 13, L.DT_TF32: 13, L.DT_F32: 1}[dt]
    lo, hi = (-14, 15) if dt == L.DT_F16 else (-30, 30)          # exponents inside the type's normal range
    e = rng.integers(lo, hi, n)
    mant = rng.integers(0, 1 << 23, n, dtype=np.int64)
    ties = (mant >> drop << drop) | (1 << (drop - 1))             # exactly half way between two storage values
    sign = rng.integers(0, 2, n).astype(np.int64) << 31
    tie_v = ((sign | ((e + 127).astype(np.int64) << 23) | ties).astype(np.uint32)).view(np.float32)
    p2 = np.exp2(e.astype(np.float32))
    near = np.concatenate([p2 * (1 - 2.0 ** -24 * rng.integers(1, 300, n)), p2 * (1 + 2.0 ** -23 * rng.integers(1, 300, n))])
    sub = rng.uniform(2.0 ** -25, 2.0 ** -14, n) * rng.choice([-1, 1], n)           # fp16 subnormal range
    edge = np.array([65504, 65519.996, 65520, -65520, 2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.0001, 3 * 2.0 ** -26])
    v = np.concatenate([tie_v, near.astype(np.float32), sub.astype(np.float32), edge.astype(np.float32),
                        rng.standard_normal(n).astype(np.float32)])
    return v.astype(np.float32)


def _check_words(got, exp, what):
    assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, exp.shape, got.dtype, exp.dtype)
    bits = np.uint16 if got.itemsize == 2 else np.uint32
    bad = np.flatnonzero((np.ascontiguousarray(got).view(bits) != np.ascontiguousarray(exp).view(bits)).reshape(-1))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} words differ, first at flat index {bad[:5]}: " \
                          f"{got.reshape(-1)[bad[:5]]} vs {exp.reshape(-1)[bad[:5]]}"


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_pack_conv_rounds_to_nearest_bit_exact(dt):
    """No BN (scale 1): the packed words are the storage type's rounding of the raw weights -- ties, neighbours of powers of
    two, subnormals -- in a padded (cout 21 -> 32, cin 13 -> 64) layout whose padding slots are exactly zero."""
    rng = np.random.default_rng(dt)
    v = _rounding_values(rng, 400, dt)
    cout, cin, k = 21, 13, 3
    w = np.resize(rng.permutation(v), cout * cin * k * k).reshape(cout, cin, k, k).astype(np.float32)
    cb = rng.standard_normal(cout).astype(np.float32)
    wp, bias = _host_pack(w, cb, None, 64, 32, dt)
    wq, b = P.pack_conv_ref(w, cb, None, dt)
    _check_words(wp, P.layout_plain(wq, 32, 64), "weights")
    _check_words(bias, P._pad(b, 32), "bias")
    if dt in (L.DT_BF16, L.DT_F16):      # the restatement itself: RNE of the ties (the kept bits decide the direction)
        exact = P.words_to_f64(wq, dt).reshape(-1)
        src = w.reshape(-1).astype(np.float64)
        err = np.abs(exact - src)
        assert np.isfinite(exact).sum() >= exact.size - 8 and (err[np.isfinite(exact)] <= np.abs(src[np.isfinite(exact)])
                                                              * 2.0 ** (-8 if dt == L.DT_BF16 else -11) + 2.0 ** -25).all()


@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_pack_conv_folds_bn_bit_exact(dt):
    """BN folded in the packer's fp32 order (scale = g / sqrt(var + eps), shift = beta - mean * scale + cb * scale), with
    running_var 0 and 1e-30 on some channels (scale ~ 316 g), then rounded: weights and bias bit for bit."""
    rng = np.random.default_rng(10 + dt)
    cout, cin, k = 37, 19, 3
    w = (rng.standard_normal((cout, cin, k, k)) * 0.1).astype(np.float32)
    w.reshape(-1)[:200] = _rounding_values(rng, 40, dt)[:200] * 1e-3
    cb = rng.standard_normal(cout).astype(np.float32)
    var = rng.random(cout).astype(np.float32) + 0.5
    var[:3] = [0.0, 1e-30, 1e-7]
    bn = [rng.random(cout).astype(np.float32) + 0.5, rng.standard_normal(cout).astype(np.float32),
          rng.standard_normal(cout).astype(np.float32), var]
    wp, bias = _host_pack(w, cb, bn, 32, 48, dt)
    wq, b = P.pack_conv_ref(w, cb, bn, dt)
    _check_words(wp, P.layout_plain(wq, 48, 32), "weights")
    _check_words(bias, P._pad(b, 48), "bias")


def test_pack_conv_host_helper_matches():
    """tests.helpers.pack_conv_host (the op tests' packer call) produces the same words."""
    rng = np.random.default_rng(3)
    w = rng.standard_normal((5, 7, 3, 3)).astype(np.float32)
    bn = [rng.random(5).astype(np.float32) + 0.5, rng.standard_normal(5).astype(np.float32),
          rng.standard_normal(5).astype(np.float32), rng.random(5).astype(np.float32) + 0.5]
    for dt in (L.DT_BF16, L.DT_F16):
        wp, bias = pack_conv_host(w, None, bn, 16, 16, dt)
        wq, b = P.pack_conv_ref(w, None, bn, dt)
        _check_words(wp, P.layout_plain(wq, 16, 16), "weights")
        _check_words(bias, P._pad(b, 16), "bias")


# ------------------------------------------------------------------------------------------------- engine forms
def _engine(dt):
    import torch
    from acr_b200.engine import Engine
    if dt == L.DT_TF32:
        return Engine(None, 1, "cpu", torch.float32, dry_run=True, tf32=True)
    return Engine(None, 1, "cpu", {L.DT_BF16: torch.bfloat16, L.DT_F16: torch.float16, L.DT_F32: torch.float32}[dt],
                  dry_run=True)


def _conv_sd(rng, key, cout, cin, k, bias=False, bn=True, transposed=False):
    shape = (cin, cout, k, k) if transposed else (cout, cin, k, k)
    sd = {f"{key}.weight": (rng.standard_normal(shape) * (2 / (cin * k * k)) ** 0.5).astype(np.float32)}
    if bias:
        sd[f"{key}.bias"] = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    if bn:
        var = rng.random(cout).astype(np.float32) + 0.5
        var[0] = 0.0                                         # tiny running_var: scale = g / sqrt(eps)
        sd.update({f"{key}_bn.weight": rng.random(cout).astype(np.float32) + 0.5,
                   f"{key}_bn.bias": (rng.standard_normal(cout) * 0.1).astype(np.float32),
                   f"{key}_bn.running_mean": (rng.standard_normal(cout) * 0.1).astype(np.float32),
                   f"{key}_bn.running_var": var})
    return sd


def _unpack(blob, w_off, b_off, words_like, bias_len):
    raw = np.frombuffer(blob.tobytes(), np.uint8)
    w = P.blob_words(raw, w_off, words_like)
    b = None if b_off is None else raw[b_off: b_off + 4 * bias_len].view(np.float32)
    return w, b


FORMS = ["plain", "xpair", "s2x", "deconv", "merged", "fold_side", "stem3", "stem7"]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("dt", DTS, ids=DT_IDS)
def test_engine_packings_bit_exact(dt, form):
    """Every packed form the engine builds, read back from its weight blob: each original weight (OIHW, or (cin, cout, 4,
    4) for the transposed conv) sits at the index the kernel reads it from as the restated rounding of w * scale; every
    other slot is zero; the bias is the restated fp32 shift."""
    from acr_b200.engine import _Blob
    if dt == L.DT_F32 and form in ("xpair", "s2x"):
        pytest.skip("the fp32 validation plan has no x-paired forms")
    rng = np.random.default_rng(100 * FORMS.index(form) + dt)
    eng, blob = _engine(dt), _Blob()
    wt = P.word_type(dt)
    if form == "plain":          # cin 34 -> one 64-channel K chunk, cout 33 -> 48
        sd = _conv_sd(rng, "c", 33, 34, 3, bias=True)
        w_off, b_off = eng._pack_conv(sd, blob, "c", "c_bn", True, 64, 48)
        wq, b = P.pack_conv_ref(sd["c.weight"], sd["c.bias"], P.bn_of(sd, "c_bn"), dt)
        exp_w, exp_b = P.layout_plain(wq, 48, 64), P._pad(b, 48)
    elif form == "xpair":
        sd = _conv_sd(rng, "c", 32, 32, 3)
        w_off, b_off = eng._pack_conv(sd, blob, "c", "c_bn", False, 64, 64, pair=True)
        wq, b = P.pack_conv_ref(sd["c.weight"], None, P.bn_of(sd, "c_bn"), dt)
        exp_w, exp_b = P.layout_xpair(wq), np.tile(b, 2)
    elif form == "s2x":
        sd = _conv_sd(rng, "c", 48, 32, 3)
        w_off, b_off = eng._pack_conv(sd, blob, "c", "c_bn", False, 64, 48, s2x=True)
        wq, b = P.pack_conv_ref(sd["c.weight"], None, P.bn_of(sd, "c_bn"), dt)
        exp_w, exp_b = P.layout_s2x(wq, 48), P._pad(b, 48)
    elif form == "deconv":       # ConvTranspose2d(k4, s2, p1) 72 -> 40, padded to 128 / 48
        sd = _conv_sd(rng, "c", 40, 72, 4, transposed=True)
        w_off, b_off = eng._pack_deconv(sd, blob, "c", "c_bn", 128, 48)
        wq, b = P.pack_conv_ref(sd["c.weight"], None, P.bn_of(sd, "c_bn"), dt, scale_axis=1)
        exp_w, exp_b = P.layout_deconv(wq, 48, 128), P._pad(b, 48)
    elif form == "merged":       # three 3x3 convs 48 -> 40 on one input, each padded to 48 outputs
        sd = {}
        for j in range(3):
            sd.update(_conv_sd(rng, f"c{j}", 40, 48, 3, bias=True))
        w_off, b_off = eng._pack_merged(sd, blob, ["c0", "c1", "c2"], ["c0_bn", "c1_bn", "c2_bn"], True, 3, 64, 48)
        ws, bs = [], []
        for j in range(3):
            wq, b = P.pack_conv_ref(sd[f"c{j}.weight"], sd[f"c{j}.bias"], P.bn_of(sd, f"c{j}_bn"), dt)
            ws.append(P.layout_plain(wq, 48, 64))
            bs.append(P._pad(b, 48))
        exp_w, exp_b = np.concatenate(ws), np.concatenate(bs)
    elif form == "fold_side":    # contact_layers[4] (109, 218) folded onto the 128-wide head tensor, no BN
        W = (rng.standard_normal((109, 218, 1, 1)) * 0.1).astype(np.float32)
        w_off, b_off = eng._pack_raw(blob, eng.fold_weights({"contact_layers.4.weight": W}, "l"), 128, 112), None
        Wm = W.reshape(109, 218)
        weff = np.zeros((109, 128, 1, 1), np.float32)             # params 0..105 <- W[:, 3:109]; cam 112..114 <- both
        for c in range(106):
            weff[:, c, 0, 0] = Wm[:, 3 + c]
        for c in range(3):
            weff[:, 112 + c, 0, 0] = Wm[:, c] + Wm[:, 109 + c]
        wq, _ = P.pack_conv_ref(weff, None, None, dt)
        exp_w, exp_b = P.layout_plain(wq, 112, 128), None
    else:                        # the stems: (64, 3, k, k) + BN as one GEMM over the (ky*k+kx)*3+ci channels
        k, kch = (3, 32) if form == "stem3" else (7, 160)
        sd = _conv_sd(rng, "s", 64, 3, k)
        w_off, b_off = eng._pack_stem(sd, blob, "s", "s_bn", kch)
        wq, b = P.pack_conv_ref(sd["s.weight"], None, P.bn_of(sd, "s_bn"), dt)
        exp_w, exp_b = P.layout_stem(wq, kch), b
    assert exp_w.dtype == wt
    got_w, got_b = _unpack(blob, w_off, b_off, exp_w, 0 if exp_b is None else exp_b.size)
    _check_words(got_w, exp_w, f"{form} weights")
    if exp_b is not None:
        _check_words(got_b.copy(), exp_b.astype(np.float32), f"{form} bias")

"""CPU: the TF32 plan (model_precision='tf32') -- weight packing, plan layout, cache keys, C ABI checks, the SASS of its
conv kernel instances and the restatement's rounding helpers."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from tests.helpers import ctensor
from tests.tf32_ref import tf32_round, tf32_truncate

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LIB = os.path.join(ROOT, "arbitrary-hands-3d-reconstruction_b200", "lib", "libacr_b200.so")
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def _np_round_nearest(a):
    """numpy reference: nearest tf32 value, ties away from zero (add half an ulp of tf32 to the magnitude, clear 13 bits)."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x1000) & ~np.uint64(0x1FFF)).astype(np.uint32)
    return np.where((u & 0x7F800000) == 0x7F800000, u.astype(np.uint32), r).view(np.float32)


def _np_truncate(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return (u & np.uint32(0xFFFFE000)).view(np.float32)


def _pack(w, bn, cb, dt):
    cout, cin, k, _ = w.shape
    cin_pad, cout_pad = (cin + 15) // 16 * 16, (cout + 15) // 16 * 16
    wp = np.zeros((cout_pad, k * k, cin_pad), np.float32)
    bias = np.zeros(cout_pad, np.float32)
    q = lambda a: None if a is None else a.ctypes.data
    L.check(L.load().acr_b200_pack_conv(w.ctypes.data, q(cb), *(q(b) for b in bn), 1e-5, cout, cin, k, cout_pad, cin_pad,
                                        dt, wp.ctypes.data, bias.ctypes.data), "pack_conv")
    return wp, bias


@pytest.mark.parametrize("k,cin,cout", [(3, 34, 64), (1, 128, 109), (3, 64, 33)])
def test_pack_tf32_is_round_to_nearest_of_the_fp32_pack(k, cin, cout):
    rng = np.random.default_rng(k * 1000 + cin + cout)
    w = rng.standard_normal((cout, cin, k, k)).astype(np.float32) * 0.1
    bn = [(rng.random(cout) + 0.5).astype(np.float32), (rng.standard_normal(cout) * 0.1).astype(np.float32),
          (rng.standard_normal(cout) * 0.1).astype(np.float32), (rng.random(cout) + 0.5).astype(np.float32)]
    cb = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    w32, b32 = _pack(w, bn, cb, L.DT_F32)
    wtf, btf = _pack(w, bn, cb, L.DT_TF32)
    assert np.array_equal(wtf.view(np.uint32), _np_round_nearest(w32).view(np.uint32))
    assert not (wtf.view(np.uint32) & 0x1FFF).any(), "packed tf32 weights must have their low 13 bits zero"
    assert np.array_equal(btf.view(np.uint32), b32.view(np.uint32)), "the bias stays fp32"
    assert (wtf != w32)[:cout, :, :cin].mean() > 0.9   # random fp32 weights are almost never tf32-representable


def test_rounding_helpers_match_numpy_bit_reference():
    rng = np.random.default_rng(0)
    a = np.concatenate([rng.standard_normal(100000).astype(np.float32) * 10.0 ** rng.integers(-30, 30, 100000),
                        np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 3.4e38, -3.4e38, 1e-40, -1e-40], np.float32),
                        # ties: exactly half a tf32 ulp above a tf32 value -> away from zero
                        (np.array([1.0, -1.0, 1.5, -3.0], np.float32).view(np.uint32) | 0x1000).view(np.float32)])
    t = torch.from_numpy(a)
    assert np.array_equal(tf32_round(t).numpy().view(np.uint32), _np_round_nearest(a).view(np.uint32))
    assert np.array_equal(tf32_truncate(t).numpy().view(np.uint32), _np_truncate(a).view(np.uint32))
    ties = tf32_round(torch.from_numpy(a[-4:])).numpy()
    assert np.array_equal(np.abs(ties), np.abs(a[-4:]) + np.float32(2.0 ** -11) * np.array([1, 1, 1, 2], np.float32))
    assert torch.isnan(tf32_round(torch.tensor([float("nan")]))).all()


def _recs(eng):
    """the op list without the conv engine choice (the validation plan's convs are CONV_REF records)"""
    out = []
    for r in eng.recs:
        kind = L.OP_CONV if r["kind"] == L.OP_CONV_REF else r["kind"]
        out.append((kind, r["out"].name, tuple(t.name for t in r["ins"]), tuple(t.name for t in r.get("aux", [])),
                    repr(sorted(r.get("attrs", {}).items())), bool(r.get("block"))))
    return out


@pytest.mark.parametrize("widths", [None, "w48"])
def test_tf32_plan_has_the_fp32_plan_layout(widths):
    from acr_b200.engine import Engine
    from acr_b200.netspec import WIDTHS_W48
    w = WIDTHS_W48 if widths else None
    f32 = Engine(None, 2, "cpu", torch.float32, dry_run=True, widths=w)
    tf = Engine(None, 2, "cpu", torch.float32, tf32=True, dry_run=True, widths=w)
    assert _recs(tf) == _recs(f32)
    assert tf.arena_bytes == f32.arena_bytes
    assert all(r["kind"] != L.OP_CONV_REF for r in tf.recs) and not tf.debug_ref_conv
    assert tf.block_starts == [] and tf.plan_dt == L.DT_TF32 and tf.dt == L.DT_F32
    kinds = [r["kind"] for r in tf.recs]
    assert kinds.count(L.OP_STEM) == 1 and L.OP_STEM_TC not in kinds and L.OP_IM2COL_STEM not in kinds
    assert kinds.count(L.OP_CONV) == sum(1 for r in f32.recs if r["kind"] == L.OP_CONV_REF)


@pytest.mark.parametrize("kw", [dict(act_dtype=torch.float32, tf32=True), dict(act_dtype=torch.bfloat16, tf32=True)])
def test_tf32_rejects_resnet_and_16bit_storage(kw):
    from acr_b200.engine import Engine
    with pytest.raises(L.AcrB200Error):
        Engine(None, 1, "cpu", dry_run=True, backbone="resnet50" if kw["act_dtype"] == torch.float32 else "hrnet", **kw)


def test_tf32_and_fp32_engines_do_not_share_a_cache_key_or_weights(monkeypatch):
    import acr.model as M
    from acr.config import args
    made = []

    class FakeEngine:
        def __init__(self, sd, batch, dev, dt, size, weights=None, tf32=False, **kw):
            self.dt, self.tf32, self.given = dt, tf32, weights
            self.weights = object()
            made.append(self)

    monkeypatch.setattr(M, "Engine", FakeEngine)
    model = M.ACR()
    old = args().model_precision
    try:
        args().model_precision = "fp32"
        e32 = model.engine(1, "cpu")
        args().model_precision = "tf32"
        etf = model.engine(1, "cpu")
        assert etf is not e32 and etf.tf32 and not e32.tf32 and etf.dt == e32.dt == torch.float32
        assert etf.given is None, "the tf32 plan must not re-use the fp32 plan's weight blob"
        assert model.engine(2, "cpu").given is etf.weights        # same mode: the blob is shared
        assert len({k[1:] for k in model._engines}) == 2 and len(model._blobs) == 2
        args().model_precision = "fp32"
        assert model.engine(1, "cpu") is e32
    finally:
        args().model_precision = old


def _fuse_op(dt_out=L.DT_F32, dt_in=L.DT_F32):
    op = L.Op()
    op.kind, op.n_in = L.OP_FUSE, 1
    op.in_[0] = ctensor(0, 16, 16, 16, 16, dt_in)
    op.out = ctensor(16 * 16 * 16 * 4, 16, 16, 16, 16, dt_out)
    op.shift[0] = 0
    return op


def test_abi_tf32_is_an_act_dtype_not_a_tensor_dtype():
    lib = L.load()
    arena = (C.c_uint8 * (4 * 16 * 16 * 16 * 4))()
    blob = (C.c_uint8 * 256)()
    plan = C.c_void_p()
    # accepted as the plan's act_dtype (a fuse-only plan: no tensor map, nothing touches a device)
    ops = (L.Op * 1)(_fuse_op())
    assert lib.acr_b200_plan_create(ops, 1, 1, C.addressof(arena), C.sizeof(arena), C.addressof(blob), 256, L.DT_TF32,
                                    C.byref(plan)) == L.OK
    lib.acr_b200_plan_destroy(plan)
    assert lib.acr_b200_plan_create(ops, 1, 1, C.addressof(arena), C.sizeof(arena), C.addressof(blob), 256, 5,
                                    C.byref(plan)) == -1
    # rejected as a tensor dtype, in plan_create and run_op
    for op in (_fuse_op(dt_out=L.DT_TF32), _fuse_op(dt_in=L.DT_TF32)):
        ops = (L.Op * 1)(op)
        for act in (L.DT_TF32, L.DT_F32):
            assert lib.acr_b200_plan_create(ops, 1, 1, C.addressof(arena), C.sizeof(arena), C.addressof(blob), 256, act,
                                            C.byref(plan)) == -1
            assert b"TF32" in lib.acr_b200_last_error()
            assert lib.acr_b200_run_op(C.byref(op), 1, C.addressof(arena), C.addressof(blob), None, act, None) == -1
    assert lib.acr_b200_run_op(C.byref(_fuse_op()), 1, C.addressof(arena), C.addressof(blob), None, 7, None) == -1
    # accepted by the packer
    w = np.ones((16, 16, 1, 1), np.float32)
    wp, b = np.zeros((16, 1, 16), np.float32), np.zeros(16, np.float32)
    assert lib.acr_b200_pack_conv(w.ctypes.data, None, None, None, None, None, 1e-5, 16, 16, 1, 16, 16, L.DT_TF32,
                                  wp.ctypes.data, b.ctypes.data) == L.OK


def _sass_by_function():
    sass = subprocess.run([CUOBJDUMP, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in sass.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
        elif cur is not None and "HGMMA" in line:
            cur.append(line)
    return funcs


def test_tf32_conv_instance_set_uses_tf32_wgmma_without_spills():
    if not (os.path.exists(LIB) and os.path.exists(CUOBJDUMP)):
        pytest.skip("library not built or no cuobjdump")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import sass_audit
        rows = sass_audit.audit(LIB)
    finally:
        sys.path.pop(0)
    tf = {n: r for n, r in rows.items() if n.startswith("conv_tc_kernel<") and ", float," in n}
    # CK 64: the two non-patch modes (1x1 and stride-2 convs) and the two single-box forms (MODE_PATCH | MODE_P1, with
    # and without MODE_RESIDENT; every tf32 3x3 stride-1 conv with 64-channel chunks takes one); CK 32: the four generic
    # modes; each at N = 64 and 128
    want = {f"conv_tc_kernel<{ck}, float, {mode}, {nt}>" for ck, modes in ((64, (0, 2, 17, 19)), (32, (0, 1, 2, 3)))
            for mode in modes for nt in (64, 128)}
    assert set(tf) == want, sorted(tf)
    for n, r in tf.items():
        assert r["LDL"] == 0 and r["STL"] == 0, f"{n}: {r['LDL']} LDL / {r['STL']} STL"
        assert r["HGMMA"] > 0 and r["UTMALDG"] > 0, n
        assert r["USETMAXREG"] == 2, n
    hg = {f: lines for f, lines in _sass_by_function().items() if "conv_tc_kernel" in f}
    tf_mangled = [f for f in hg if re.search(r"conv_tc_kernelILi(64|32)EfLi", f)]
    assert len(tf_mangled) == 16
    for f in tf_mangled:
        assert hg[f] and all(re.search(r"HGMMA\.64x(64|128)x8\.F32\.TF32", l) for l in hg[f]), f
    for f, lines in hg.items():
        if f not in tf_mangled:
            assert not any("TF32" in l for l in lines), f

"""The fp32 tail on the GPU (acr_b200_mano_forward with its projection outputs, acr_b200_cam_trans,
acr_b200_rot6d_to_aa, acr_b200_rodrigues, acr_b200_one_euro_smooth) against the float64 statements of
tests/tail_ref.py, per element and within their derived bounds, on the kernels' masking, alignment and branch edges.

Every call goes through the C ABI with caller-owned buffers: an output is a 16-byte aligned window inside a larger
buffer, the window prefilled with one NaN pattern and the guards around it with another, so that after a launch the
guards must be bit-identical, every element of a row below n must have been written and every row from n on must not.
Each test prints the worst err/bound it met per output."""
import ctypes as C
import math
from collections import defaultdict

import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from oracle.mano_ref import JOINT_REORDER, TIPS
from oracle.preprocess_ref import img_preprocess
from tests import tail_ref as T

pytestmark = pytest.mark.gpu
U = T.U
GUARD, FILL = 0x7FC0BEEF, 0x7FC12345      # two quiet-NaN bit patterns
NG = 64                                    # guard floats on each side: the window stays 16-byte aligned
SIDE = ("left", "right")
TIP_OUT = [JOINT_REORDER.index(16 + t) for t in range(5)]


class Win:
    """A (rows, ...) fp32 output window between two guards."""

    def __init__(self, *shape):
        self.shape, self.numel = shape, int(np.prod(shape))
        self.buf = torch.full((2 * NG + self.numel,), GUARD, dtype=torch.int32, device="cuda")
        self.buf[NG:NG + self.numel] = FILL
        self.ptr = self.buf.data_ptr() + 4 * NG
        assert self.ptr % 16 == 0

    def bits(self):
        b = self.buf.cpu().numpy()
        assert (b[:NG] == GUARD).all() and (b[NG + self.numel:] == GUARD).all(), "a guard region was written"
        return b[NG:NG + self.numel].reshape(self.shape)

    def read(self, n):
        """rows [0, n) as fp32, after checking the guards, that every element below row n was written and that no
        row from n on was."""
        w = self.bits()
        assert (w[:n] != FILL).all(), "an element inside the valid rows was not written"
        assert (w[n:] == FILL).all(), "a row at or beyond n was written"
        return w[:n].view(np.float32)


def dev(a, dtype=np.float32):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


class Stats(defaultdict):
    def __init__(self):
        super().__init__(float)

    def within(self, name, got, exp, bound):
        err = np.abs(np.asarray(got, np.float64) - exp)
        r = err / bound
        i = np.unravel_index(np.argmax(r), r.shape)
        assert r[i] <= 1, f"{name}: element {i} got {np.asarray(got)[i]!r} expected {exp[i]!r} err {err[i]:.3e} bound {bound[i]:.3e}"
        self[name] = max(self[name], float(r[i]))

    def show(self, title):
        print(f"\n{title}: worst err/bound  " + "  ".join(f"{k} {v:.3f}" for k, v in sorted(self.items())))


# ---------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def assets():
    from acr_b200.synth import make_synthetic_mano
    return {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}


@pytest.fixture(scope="module")
def models(assets):
    """Packed models as the pipeline packs them: the left one with its shapedirs x-flipped."""
    from acr_b200 import ops
    return ops.pack_mano_model(assets["left"], True, "cuda"), ops.pack_mano_model(assets["right"], False, "cuda")


_OFFS = {}


def offsets_rows(n):
    """(n,10) offsets rows of landscape, portrait and square frames of several sizes, from the oracle's
    img_preprocess: pad sizes and the top / left paddings differ from row to row."""
    sizes = [(24, 40), (40, 24), (32, 32), (10, 50), (51, 9), (30, 31), (64, 48), (7, 20)]
    for hw in sizes:
        if hw not in _OFFS:
            _OFFS[hw] = img_preprocess(np.zeros((hw[0], hw[1], 3), np.uint8), 8)[1]
    return np.stack([_OFFS[sizes[i % len(sizes)]] for i in range(n)]).astype(np.float32)


def make_hands(n, seed):
    """Seeded poses (Gaussians of 0.5 rad on even rows, 1.5 rad on odd ones) and betas with the edge rows first: all
    zero, root rotation at pi, 1e-6 everywhere, 20 pi on one joint, betas at +3 and -3; cam scales 0.3 .. 3 with
    translations of both signs."""
    rng = np.random.default_rng(seed)
    poses = rng.standard_normal((n, 48)) * np.where(np.arange(n) % 2, 1.5, 0.5)[:, None]
    betas = rng.standard_normal((n, 10))
    edge = [lambda i: poses.__setitem__(i, 0), lambda i: poses.__setitem__((i, slice(0, 3)), [math.pi, 0, 0]),
            lambda i: poses.__setitem__(i, 1e-6), lambda i: poses.__setitem__((i, slice(12, 15)), [0, 20 * math.pi, 0]),
            lambda i: betas.__setitem__(i, 3), lambda i: betas.__setitem__(i, -3)]
    for i, f in enumerate(edge[:n]):
        f(i)
    cam = rng.uniform(-1, 1, (n, 3))
    cam[:, 0] = rng.permutation(np.linspace(0.3, 3, n))
    return poses.astype(np.float32), betas.astype(np.float32), cam.astype(np.float32), offsets_rows(n)


def side_pattern(name, n):
    i = np.arange(n)
    return {"left": np.zeros(n, int), "right": np.ones(n, int), "alternate": i % 2,
            "odd_one": (i % 8 == 3).astype(int), "odd_last": 1 - (i == n - 1).astype(int)}[name]


def reference(assets, poses, betas, sides, center_idx):
    """mano_forward64 row by row side: dict of (n, ...) arrays."""
    out = {}
    for s in (0, 1):
        rows = np.flatnonzero(sides == s)
        if rows.size == 0:
            continue
        m = T.mano_forward64(assets[SIDE[s]], poses[rows], betas[rows], SIDE[s], None if center_idx < 0 else center_idx)
        for k, v in m.items():
            out.setdefault(k, np.zeros((len(sides),) + v.shape[1:]))[rows] = v
    return out


def run_mano(models, poses, betas, hand_type, default_side, n_dev, center_idx, cam, offs, want=("camed", "pj2d", "org"),
             only_model=None):
    """One launch of acr_b200_mano_forward on guarded windows -> (rc, windows).  ``hand_type`` None passes NULL;
    ``only_model`` passes that side's packed model alone."""
    n = poses.shape[0]
    w = dict(verts=Win(n, 778, 3), joints=Win(n, 21, 3), center=Win(n, 3))
    if cam is not None:
        if "camed" in want:
            w["verts_camed"] = Win(n, 778, 3)
        w["pj2d"] = Win(n, 21, 2)
        if offs is not None:
            w["pj2d_org"] = Win(n, 21, 2)
    ml, mr = models
    if only_model is not None:
        ml, mr = (ml, None) if only_model == 0 else (None, mr)
    keep = [dev(poses), dev(betas), dev(hand_type, np.int32), None if n_dev is None else dev([n_dev], np.int32),
            dev(cam), dev(offs)]
    p = lambda k: w[k].ptr if k in w else None
    rc = L.load().acr_b200_mano_forward(L.ptr(ml), L.ptr(mr), L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2]),
                                        int(default_side), L.ptr(keep[3]), n, int(center_idx), L.ptr(keep[4]),
                                        L.ptr(keep[5]), p("verts"), p("joints"), p("center"), p("verts_camed"),
                                        p("pj2d"), p("pj2d_org"), stream())
    torch.cuda.synchronize()
    return rc, w


def check_mano(st, w, ref, sides, n_eff, cam, offs):
    """Every per-element assertion on one launch's windows, rows [0, n_eff)."""
    v, j, c = w["verts"].read(n_eff), w["joints"].read(n_eff), w["center"].read(n_eff)
    if n_eff == 0:
        for k in ("verts_camed", "pj2d", "pj2d_org"):
            if k in w:
                w[k].read(0)
        return
    r = {k: a[:n_eff] for k, a in ref.items()}
    st.within("verts", v, r["verts"], r["b_verts"])
    st.within("joints", j, r["joints"], r["b_joints"])
    st.within("center", c, r["center"], r["b_center"] + 1e-45)
    # the five tip joints are the hand's own side's tip vertices, bit for bit
    for i in range(n_eff):
        tv = v[i, TIPS[SIDE[sides[i]]]]
        assert (j[i, TIP_OUT].view(np.int32) == tv.view(np.int32)).all(), f"row {i}: tip joints are not verts[tips]"
    if cam is None:
        return
    cam64 = cam[:n_eff].astype(np.float64)
    s, t = cam64[:, None, 0:1], cam64[:, None, 1:]
    pj = w["pj2d"].read(n_eff)
    st.within("pj2d step", pj, s * j[..., :2] + t, T.project_step_bound(j[..., :2].astype(np.float64), s, t))
    proj = T.project64(r["verts"], r["joints"], cam[:n_eff], None if offs is None else offs[:n_eff], r["b_verts"], r["b_joints"])
    st.within("pj2d", pj, proj["pj2d"], proj["b_pj2d"])
    if "verts_camed" in w:
        vc = w["verts_camed"].read(n_eff)
        assert (vc[..., 2].view(np.int32) == v[..., 2].view(np.int32)).all(), "verts_camed z is not verts z"
        st.within("verts_camed step", vc[..., :2], s * v[..., :2] + t,
                  T.project_step_bound(v[..., :2].astype(np.float64), s, t))
        st.within("verts_camed", vc, proj["verts_camed"], proj["b_verts_camed"])
    if "pj2d_org" in w:
        org = w["pj2d_org"].read(n_eff)
        o = offs[:n_eff].astype(np.float64)
        pad = o[:, None, 0:2]
        lt = np.stack([o[:, 5] - o[:, 9], o[:, 2] - o[:, 6]], 1)[:, None]
        st.within("pj2d_org step", org, (pj + 1.0) * pad / 2 + lt, T.org_step_bound(pj.astype(np.float64), pad, lt))
        st.within("pj2d_org", org, proj["pj2d_org"], proj["b_pj2d_org"])


# ------------------------------------------------------------------------------------------------------ MANO forward
@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 15, 16, 17, 513])
def test_mano_rows_sides_and_masks(models, assets, n):
    """Group of 8 hands full and partial, every side pattern inside a group, n_dev absent / 0 / 1 / n-5 / n / n+3
    (clamped to n), all outputs."""
    st = Stats()
    poses, betas, cam, offs = make_hands(n, 100 + n)
    patterns = ["alternate", "odd_one"] if n == 513 else ["left", "right", "alternate", "odd_one", "odd_last"]
    for pat in patterns:
        sides = side_pattern(pat, n)
        ref = reference(assets, poses, betas, sides, 9)
        n_devs = [None] + ([0, 1, n - 5, n, n + 3] if pat in ("alternate", "odd_last") else [])
        for nd in n_devs:
            if nd is not None and nd < 0:
                continue
            rc, w = run_mano(models, poses, betas, sides, 1, nd, 9, cam, offs)
            assert rc == L.OK
            check_mano(st, w, ref, sides, n if nd is None else min(nd, n), cam, offs)
    st.show(f"mano_forward n={n}")


@pytest.mark.parametrize("default_side", [0, 1])
def test_mano_default_side_with_one_model(models, assets, default_side):
    st = Stats()
    for n in (1, 9, 16):
        poses, betas, cam, offs = make_hands(n, 200 + n)
        sides = np.full(n, default_side)
        ref = reference(assets, poses, betas, sides, 9)
        rc, w = run_mano(models, poses, betas, None, default_side, None, 9, cam, offs, only_model=default_side)
        assert rc == L.OK
        check_mano(st, w, ref, sides, n, cam, offs)
    rc, w = run_mano(models, poses, betas, None, default_side, None, 9, cam, offs, only_model=1 - default_side)
    assert rc == -1     # ACR_B200_EINVAL: the requested side's model is missing
    for win in w.values():
        win.read(0)
    st.show(f"mano_forward hand_type=NULL default_side={default_side}")


@pytest.mark.parametrize("n", [9, 17])
def test_mano_output_sets(models, assets, n):
    """Outputs are optional independently: no cam; cam without offsets; cam + offsets without verts_camed; all."""
    st = Stats()
    poses, betas, cam, offs = make_hands(n, 300 + n)
    sides = side_pattern("alternate", n)
    ref = reference(assets, poses, betas, sides, 9)
    for c, o, want in ((None, None, ()), (cam, None, ("camed",)), (cam, offs, ()), (None, offs, ()), (cam, offs, ("camed",))):
        rc, w = run_mano(models, poses, betas, sides, 1, n - 2, 9, c, o, want)
        assert rc == L.OK
        assert ("verts_camed" in w) == (c is not None and "camed" in want) and ("pj2d_org" in w) == (c is not None and o is not None)
        check_mano(st, w, ref, sides, n - 2, c, o)
    st.show(f"mano_forward output sets n={n}")


def test_mano_center_joints(models, assets):
    """No centre, every kinematic joint as centre; a fingertip returns ACR_B200_ENOTSUP and launches nothing."""
    st = Stats()
    n = 9
    poses, betas, cam, offs = make_hands(n, 400)
    sides = side_pattern("alternate", n)
    for ci in range(-1, 21):
        rc, w = run_mano(models, poses, betas, sides, 1, None, ci, cam, offs)
        if ci >= 0 and JOINT_REORDER[ci] >= 16:
            assert rc == -3, ci
            for win in w.values():
                win.read(0)
            continue
        assert rc == L.OK
        check_mano(st, w, reference(assets, poses, betas, sides, ci), sides, n, cam, offs)
    st.show("mano_forward centres")


def test_mano_row_independent_bits(models):
    """A hand's outputs do not depend on its row, its group's other hands or n: the same hand at rows 0, 1, 7, 8 and
    512 (both 16-byte alignments of its vertex block, first and last slot of a group, a partial group) is
    bit-identical in every output."""
    hp, hb, hc, ho = (a[7:8] for a in make_hands(8, 500))
    base = None
    for row, n in ((0, 1), (1, 2), (7, 8), (8, 9), (512, 513), (3, 16)):
        poses, betas, cam, offs = make_hands(n, 510 + n)
        sides = side_pattern("alternate", n)
        sides[row] = 0
        for a, h in ((poses, hp), (betas, hb), (cam, hc), (offs, ho)):
            a[row] = h[0]
        rc, w = run_mano(models, poses, betas, sides, 1, None, 9, cam, offs)
        assert rc == L.OK
        got = {k: win.read(n)[row].view(np.int32).copy() for k, win in w.items()}
        if base is None:
            base = got
        for k in base:
            assert (got[k] == base[k]).all(), f"{k} of the same hand differs at row {row} of {n}"


def test_mano_root_rotation_equivariance(models, assets):
    """Centred on joint 9, replacing the root rotation R by Q R rotates every centred vertex and joint by Q.  The
    rotated root is rounded to fp32, which the float64 statement of BOTH inputs accounts for: the kernel's two
    results must satisfy ||Q got(R) - got(Q R)|| <= ||b(R)||_2 + ||b(Q R)||_2 + ||Q exp(R) - exp(Q R)||."""
    st = Stats()
    n = 16
    poses, betas, _, _ = make_hands(n, 600)
    rng = np.random.default_rng(601)
    Q = T.aa_to_rotmat64(rng.standard_normal((n, 3)))
    R0 = T.rodrigues64(poses[:, :3])
    poses2 = poses.copy()
    poses2[:, :3] = T.rotmat_to_aa64(Q @ R0)[0].astype(np.float32)
    sides = side_pattern("alternate", n)
    res = []
    for p in (poses, poses2):
        rc, w = run_mano(models, p, betas, sides, 1, None, 9, None, None)
        assert rc == L.OK
        res.append((w["verts"].read(n).astype(np.float64), w["joints"].read(n).astype(np.float64),
                    reference(assets, p, betas, sides, 9)))
    for k, i in (("verts", 0), ("joints", 1)):
        rot = np.einsum("nab,nvb->nva", Q, res[0][i])
        resid = np.linalg.norm(np.einsum("nab,nvb->nva", Q, res[0][2][k]) - res[1][2][k], axis=-1)
        assert (resid <= 8 * U * np.linalg.norm(res[1][2][k], axis=-1).max() * 4).all(), "the statement is not equivariant"
        bound = np.linalg.norm(res[0][2]["b_" + k], axis=-1) + np.linalg.norm(res[1][2]["b_" + k], axis=-1) + resid
        st.within(k, np.linalg.norm(rot - res[1][i], axis=-1), np.zeros_like(bound), bound)
    st.show("mano_forward root equivariance")


# --------------------------------------------------------------------------------------------------------- rotations
def run_rot(fn, x, n, width):
    out = Win(n, width)
    keep = dev(x)
    rc = getattr(L.load(), fn)(L.ptr(keep), n, out.ptr, stream())
    torch.cuda.synchronize()
    assert rc == L.OK
    return out.read(n)


def test_rot6d_to_aa_every_row():
    x, tags = T.structured_rot6d(0)
    g = np.random.default_rng(5).standard_normal((4096 * 16, 6)).astype(np.float32)
    for name, rows in (("structured", x), ("gaussian", g)):
        aa = run_rot("acr_b200_rot6d_to_aa", rows, rows.shape[0], 3)
        r, v = T.check_rot6d(rows, aa)
        print(f"\nrot6d_to_aa {name} ({rows.shape[0]} rows): worst err/bound as rotation {r:.3f}, as axis angle {v:.3f}")
    for n in (1, 127, 128, 129):     # the block tail
        T.check_rot6d(g[:n], run_rot("acr_b200_rot6d_to_aa", g[:n], n, 3))


def test_rodrigues_every_element():
    rng = np.random.default_rng(6)
    ax = rng.standard_normal((64, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.concatenate([[0, 1e-9, 1e-8, 1e-7, 1e-4, 1, math.pi, 2 * math.pi], np.linspace(3, 100 * math.pi, 56)])
    aa = np.concatenate([ax * ang[:, None], rng.standard_normal((193, 3)), np.zeros((1, 3))]).astype(np.float32)
    worst = ortho = 0.0
    for n in (1, 255, 256, 257, aa.shape[0]):
        R = run_rot("acr_b200_rodrigues", aa[:n], n, 9).astype(np.float64)
        r = np.abs(R - T.rodrigues64(aa[:n]).reshape(n, 9)) / T.rodrigues_bound(aa[:n])[:, None]
        assert r.max() <= 1, (n, np.unravel_index(np.argmax(r), r.shape), r.max())
        M = R.reshape(n, 3, 3)
        o = np.abs(M @ M.transpose(0, 2, 1) - np.eye(3)).max()
        assert o <= T.ORTHO_BOUND
        worst, ortho = max(worst, r.max()), max(ortho, o / T.ORTHO_BOUND)
    print(f"\nrodrigues: worst err/bound {worst:.3f}, orthogonality {ortho:.3f}")


# ------------------------------------------------------------------------------------------------ camera translation
def run_cam_trans(j3d, pj2d, n_dev, focal, size):
    n = j3d.shape[0]
    out = Win(n, 3)
    keep = [dev(j3d), dev(pj2d), None if n_dev is None else dev([n_dev], np.int32)]
    rc = L.load().acr_b200_cam_trans(L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2]), n, float(focal), float(size), out.ptr,
                                     stream())
    torch.cuda.synchronize()
    assert rc == L.OK
    return out.read(n if n_dev is None else min(n, n_dev))


def test_cam_trans_validity_and_masks(models):
    st = Stats()
    n = 129
    poses, betas, cam, offs = make_hands(n, 700)
    cam[40:60, 1:] *= 4                                    # hands projected far off-centre
    rc, w = run_mano(models, poses, betas, side_pattern("alternate", n), 1, None, 9, cam, None)
    j3d, pj = w["joints"].read(n).copy(), w["pj2d"].read(n).copy()
    usable = {}
    for row, k in ((10, 5), (11, 4), (12, 3), (13, 0)):   # unusable by depth
        j3d[row, k:, 2] = -2.0
        usable[row] = k
    for row, k in ((20, 5), (21, 4), (22, 3), (23, 0)):   # unusable by pixel row: v == -2 exactly at 512, below at 256
        pj[row, k:, 1] = -1.0078125 if row % 2 else -1.5
        usable[row] = k
    for focal, size in ((1265.0, 512.0), (500.0, 256.0), (5000.0, 512.0), (1265.0, 256.0)):
        exp, b = T.cam_trans64(j3d, pj, focal, size)
        for row, k in usable.items():
            if size == 512.0 or row not in (21, 23):
                assert ((exp[row] == -1).all() and (b[row] == 0).all()) == (k < 4), (row, k)
        for m, nd in ((1, None), (128, None), (129, None), (129, 0), (129, 100), (129, 140)):
            got = run_cam_trans(j3d[:m], pj[:m], nd, focal, size)
            k = got.shape[0]
            if k:
                st.within(f"f={focal:.0f} size={size:.0f}", got, exp[:k], b[:k] + 1e-45)
    st.show("cam_trans")


# --------------------------------------------------------------------------------------------------------- smoothing
def smooth_sequence(frames, seed):
    """Seeded random-walk poses / betas for two hands; hand 0's root turns about a slowly moving axis from 2.7 rad
    through pi to 3.6 rad; detection drops out per side."""
    rng = np.random.default_rng(seed)
    poses = np.cumsum(rng.standard_normal((frames, 2, 48)) * 0.03, 0) + rng.standard_normal((1, 2, 48)) * 0.4
    betas = np.cumsum(rng.standard_normal((frames, 2, 10)) * 0.01, 0) + rng.standard_normal((1, 2, 10))
    ax = np.array([0.3, 1.0, -0.5]) + np.cumsum(rng.standard_normal((frames, 3)) * 0.005, 0)
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    poses[:, 0, :3] = ax * np.linspace(2.7, 3.6, frames)[:, None]
    det = (rng.random((frames, 2)) > 0.15).astype(np.float32)
    det[0] = (1, 0)                                        # hand 1 starts later than hand 0
    return poses.astype(np.float32), betas.astype(np.float32), det


class SmoothRig:
    """poses (2,48), betas (2,10) and the state, each a guarded window the kernel updates in place."""

    def __init__(self, rows=2):
        self.nstate = int(L.load().acr_b200_one_euro_state_floats())
        self.p, self.b, self.s = Win(rows, 48), Win(rows, 10), Win(self.nstate)
        self.s.buf[NG:NG + self.nstate] = 0

    def load(self, poses, betas):
        self.p.buf[NG:NG + self.p.numel] = dev(poses).view(torch.int32).flatten()
        self.b.buf[NG:NG + self.b.numel] = dev(betas).view(torch.int32).flatten()

    def run(self, coeff, hand_type=None, det=None, n_dev=None, rows=2):
        keep = [dev(hand_type, np.int32), dev(det), None if n_dev is None else dev([n_dev], np.int32)]
        rc = L.load().acr_b200_one_euro_smooth(self.p.ptr, self.b.ptr, L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2]), rows,
                                               self.s.ptr, float(coeff), stream())
        torch.cuda.synchronize()
        return rc

    def get(self):
        return self.p.bits().view(np.float32).copy(), self.b.bits().view(np.float32).copy(), self.s.bits().copy()


@pytest.mark.parametrize("coeff", [0.5, 4.0, 30.0])
def test_one_euro_every_frame(coeff):
    st = Stats()
    frames = 300
    poses, betas, det = smooth_sequence(frames, 800)
    rig, banks, seen = SmoothRig(), [T.OneEuro64(coeff), T.OneEuro64(coeff)], [False, False]
    bank = rig.nstate // 2
    ht = np.array([0, 1])
    for t in range(frames):
        rig.load(poses[t], betas[t])
        _, _, s0 = rig.get()
        assert rig.run(coeff, ht, det[t]) == L.OK
        p, b, s1 = rig.get()
        for h in range(2):
            pin, bin_ = poses[t, h].view(np.int32), betas[t, h].view(np.int32)
            if not det[t, h] > 0:      # an undetected hand: its row and its bank are untouched
                assert (p[h].view(np.int32) == pin).all() and (b[h].view(np.int32) == bin_).all()
                assert (s1[h * bank:(h + 1) * bank] == s0[h * bank:(h + 1) * bank]).all()
                continue
            r = banks[h].process(poses[t, h], betas[t, h])
            if not seen[h]:            # a first frame passes pose and betas through bit for bit
                assert (p[h, 3:].view(np.int32) == pin[3:]).all() and (b[h].view(np.int32) == bin_).all()
                seen[h] = True
            st.within("pose", p[h, 3:], r["pose"], r["b_pose"] + 1e-45)
            st.within("betas", b[h], r["betas"], r["b_betas"] + 1e-45)
            assert np.isfinite(p[h, :3]).all()
            e = np.linalg.norm(T.aa_to_rotmat64(p[h, :3])[0] - T.aa_to_rotmat64(r["aa"])[0])
            st.within("root (as a rotation)", np.array([e]), np.zeros(1),
                      np.array([T.smoothed_root_bound(r["b_M"], r["qnorm"])]))
    assert all(seen)
    st.show(f"one_euro_smooth smooth_coeff={coeff}, {frames} frames")


def test_one_euro_banks_masks_and_reset():
    poses, betas, _ = smooth_sequence(12, 801)
    a, b = SmoothRig(), SmoothRig()
    for t in range(6):     # hand_type NULL: bank = row, the same as hand_type [0, 1]
        for rig, ht in ((a, None), (b, np.array([0, 1]))):
            rig.load(poses[t], betas[t])
            assert rig.run(4.0, ht) == L.OK
        for x, y in zip(a.get(), b.get()):
            assert (x.view(np.int32) == y.view(np.int32)).all()
    # n_dev = 1 filters row 0 only
    a.load(poses[6], betas[6])
    _, _, s0 = a.get()
    assert a.run(4.0, None, None, n_dev=1) == L.OK
    p, bb, s1 = a.get()
    half = a.nstate // 2
    assert (p[1].view(np.int32) == poses[6, 1].view(np.int32)).all() and (bb[1].view(np.int32) == betas[6, 1].view(np.int32)).all()
    assert (s1[half:] == s0[half:]).all() and (s1[:half] != s0[:half]).any()
    assert (p[0, 3:] != poses[6, 0, 3:]).any()
    # a zeroed state (OneEuroState.reset) makes the next frame a first frame
    from acr_b200 import ops
    state = ops.OneEuroState("cuda")
    for t in range(3):
        pt, bt = dev(poses[t]), dev(betas[t])
        ops.one_euro_smooth(pt, bt, state, 4.0)
    assert (pt[:, 3:].cpu().numpy() != poses[2][:, 3:]).any()
    state.reset()
    pt, bt = dev(poses[3]), dev(betas[3])
    ops.one_euro_smooth(pt, bt, state, 4.0)
    assert (pt[:, 3:].cpu().numpy().view(np.int32) == poses[3][:, 3:].view(np.int32)).all()
    assert (bt.cpu().numpy().view(np.int32) == betas[3].view(np.int32)).all()


def test_one_euro_rejects_more_rows_than_banks():
    """The state has one bank per hand type: n_max > 2 is an argument error before any launch.  Every buffer here
    holds three rows and hand_type names existing banks only, so the call stays inside its buffers in any case."""
    from acr_b200 import ops
    rig = SmoothRig(rows=3)
    rng = np.random.default_rng(9)
    poses, betas = rng.standard_normal((3, 48)).astype(np.float32), rng.standard_normal((3, 10)).astype(np.float32)
    rig.load(poses, betas)
    before = rig.get()
    assert rig.run(4.0, np.array([0, 1, 0]), rows=3) == -1          # ACR_B200_EINVAL
    assert b"one_euro_smooth" in L.load().acr_b200_last_error()
    for x, y in zip(before, rig.get()):
        assert (x.view(np.int32) == y.view(np.int32)).all()
    with pytest.raises(L.AcrB200Error):
        ops.one_euro_smooth(dev(poses), dev(betas), ops.OneEuroState("cuda"), 4.0, hand_type=dev([0, 1, 0], np.int32))

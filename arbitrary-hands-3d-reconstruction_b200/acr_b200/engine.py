"""Launch-plan builder: NetSpec + state-dict -> packed weight blob, activation arena, C op list.

Host-side counterpart of csrc/plan.cu.  Built once per (weights, batch size, dtype); running it is a
single C call (``acr_b200_plan_run``) that issues every kernel of the backbone + heads.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import lib as L
from .netspec import BN_EPS, NetSpec, Op, Tensor, build_acr_spec, conv_flops_per_image

ALIGN = 1024          # arena / blob alignment (TMA global address needs 16 B; generous for swizzle)
POOL_CHUNKS = 16
POOL_PART_FLOATS = 256 * 32 + 64


def _pow2(v):
    return v > 0 and (v & (v - 1)) == 0


def _rup(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class _Blob:
    """Append-only byte blob with aligned sub-allocations (the packed weights)."""

    def __init__(self):
        self.parts: List[bytes] = []
        self.size = 0

    def add(self, arr: np.ndarray) -> int:
        off = _rup(self.size, 256)
        if off > self.size:
            self.parts.append(b"\0" * (off - self.size))
        b = np.ascontiguousarray(arr).tobytes()
        self.parts.append(b)
        self.size = off + len(b)
        return off

    def tobytes(self) -> bytes:
        return b"".join(self.parts)


class _Arena:
    """First-fit interval allocator over op indices (tensor liveness) -> byte offsets."""

    def __init__(self):
        self.free: List[Tuple[int, int]] = []   # (offset, size) sorted by offset
        self.top = 0

    def alloc(self, size: int) -> int:
        size = _rup(size, ALIGN)
        for i, (off, sz) in enumerate(self.free):
            if sz >= size:
                if sz == size:
                    self.free.pop(i)
                else:
                    self.free[i] = (off + size, sz - size)
                return off
        off = self.top
        self.top += size
        return off

    def release(self, off: int, size: int) -> None:
        size = _rup(size, ALIGN)
        self.free.append((off, size))
        self.free.sort()
        merged: List[Tuple[int, int]] = []
        for o, s in self.free:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1] = (merged[-1][0], merged[-1][1] + s)
            else:
                merged.append((o, s))
        # give the tail back to the bump pointer
        if merged and merged[-1][0] + merged[-1][1] == self.top:
            self.top = merged[-1][0]
            merged.pop()
        self.free = merged


def deconv_parity_weights(w: np.ndarray) -> np.ndarray:
    """ConvTranspose2d(k4, s2, p1) weight (cin, cout, 4, 4) -> the four 2x2 convs it is made of, (4, cout, cin, 2, 2) OIHW.
    Output pixel (2m+py, 2n+px) = sum over taps (ty, tx) of x[m + py + ty - 1, n + px + tx - 1] . w[:, :, 3-py-2ty, 3-px-2tx]:
    parity p = py*2 + px, tap (ty, tx) reads the input at offset (py + ty - 1, px + tx - 1)."""
    cin, cout = w.shape[:2]
    out = np.zeros((4, cout, cin, 2, 2), np.float32)
    for py in range(2):
        for px in range(2):
            for ty in range(2):
                for tx in range(2):
                    out[py * 2 + px, :, :, ty, tx] = w[:, :, 3 - py - 2 * ty, 3 - px - 2 * tx].T
    return out


class Engine:
    """The backbone + heads of ACR as one precompiled CUDA launch plan.

    ``state_dict`` uses the reference's key names (checkpoint compatible).  ``act_dtype`` is
    torch.bfloat16 or torch.float16 (storage of activations/weights; accumulation is fp32) -- the
    product path on the tensor cores -- or torch.float32: the VALIDATION plan (fp32 storage, fp64
    accumulation on the CUDA cores, csrc/validate_f32.cu), which is what the reference's default
    ``model_precision='fp32'`` maps to and what pins the whole pipeline at 1e-4.
    ``tf32=True`` (with act_dtype torch.float32): the TF32 plan, ``model_precision='tf32'`` -- what the reference's fp32
    model runs on Ampere / Hopper under cuDNN's default ``allow_tf32``.  The validation plan's op list and arena (fp32
    storage, no x-pair / stride-2 pair packing, no fused blocks, CUDA-core stem), but every conv on the wgmma tensor cores
    with tf32 operands and fp32 accumulation, its weights packed as DT_TF32 (BN folded, rounded to the nearest tf32).
    ``debug_ref_conv`` swaps the wgmma conv for the CUDA-core reference kernel (tests only).
    ``head_only`` builds the plan of ``ACR.head_forward`` (/root/reference/acr/model.py:47-65): the ops
    after the trunk, fed by an external (B,32,H/4,W/4) feature through ``run_heads``.
    ``weights`` re-uses the packed weight blob of another engine of the same dtype / flags (the blob does
    not depend on the batch size).
    ``backbone``: "hrnet" (HRNet-W32, or the trunk ``widths`` names) or "resnet50" (netspec.build_acr_spec): the
    ResNet-50 trunk runs on the tensor cores only (7x7 stem, max-pool, 1x1 stride-2 and transposed convs have no fp32
    validation or CUDA-core form), so fp32, ``tf32`` and ``debug_ref_conv`` raise AcrB200Error for it.
    """

    def __init__(self, state_dict: Dict[str, torch.Tensor], batch: int, device, act_dtype=torch.bfloat16,
                 input_size: int = 512, debug_ref_conv: bool = False, reuse_memory: bool = True,
                 dry_run: bool = False, keep_extra=(), stem_on_tensor_cores: bool = True,
                 head_only: bool = False, weights: Optional[torch.Tensor] = None, widths=None,
                 backbone: str = "hrnet", tf32: bool = False):
        self.keep_extra = tuple(keep_extra)   # extra tensor names kept alive after the run (tests)
        self.dry_run = dry_run      # layout only (arena size, op list); used by CPU tests
        if not dry_run and not torch.cuda.is_available():
            raise L.AcrB200Error("Engine needs a CUDA device; there is no CPU fallback on the product path")
        self.lib = L.load()
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.batch = int(batch)
        self.act_dtype = act_dtype
        self.dt = {torch.bfloat16: L.DT_BF16, torch.float16: L.DT_F16, torch.float32: L.DT_F32}[act_dtype]
        self.f32 = act_dtype == torch.float32
        if tf32 and not self.f32:
            raise L.AcrB200Error("Engine: tf32=True is the TF32 plan of fp32 storage: pass act_dtype=torch.float32")
        self.tf32 = bool(tf32)
        self.plan_dt = L.DT_TF32 if self.tf32 else self.dt   # act_dtype of the plan and the weight packer
        self.esz = 4 if self.f32 else 2
        self.npw = np.float32 if self.f32 else np.uint16      # numpy type of one packed weight
        if backbone == "resnet50" and (self.f32 or debug_ref_conv):
            raise L.AcrB200Error("Engine: the ResNet-50 trunk runs on the tensor cores only (no fp32 validation or TF32 "
                                 "plan, no debug_ref_conv): use act_dtype torch.bfloat16 or torch.float16")
        self.backbone = backbone
        self.stem_on_tensor_cores = stem_on_tensor_cores and not self.f32
        self.head_only = head_only
        from .netspec import WIDTHS
        # Folding the coarse fuse sums into the producing conv (ACR_B200_FOLD_FUSE=1) is an opt-in: it trades the fuse
        # kernels for extra latency-bound loads in the conv epilogue.  Tensor-core plans only.
        self.spec: NetSpec = build_acr_spec(input_size, widths=tuple(widths) if widths else WIDTHS,
                                            fold_fuse=(os.environ.get("ACR_B200_FOLD_FUSE", "0") != "0"
                                                       and act_dtype != torch.float32 and not debug_ref_conv),
                                            backbone=backbone)
        self.input_size = input_size
        self.flops_per_image = conv_flops_per_image(self.spec)
        self.debug_ref_conv = debug_ref_conv or (self.f32 and not self.tf32)
        self.run_count = 0          # bumped by every run(): lazily read outputs check it (acr/model.py)
        sd = {k: v.detach().float().cpu().numpy() for k, v in (state_dict or {}).items()
              if v.dtype.is_floating_point}
        self._build(sd, reuse_memory, weights)

    # ------------------------------------------------------------------ weights
    def _pack_conv(self, sd, blob: _Blob, wkey: str, bnkey: Optional[str], has_bias: bool, cin_pad: int,
                   cout_pad: int, pair: bool = False, s2x: bool = False) -> Tuple[int, int]:
        w = np.ascontiguousarray(sd[wkey + ".weight"], np.float32)
        cb = np.ascontiguousarray(sd[wkey + ".bias"], np.float32) if has_bias else None
        bn = [np.ascontiguousarray(sd[f"{bnkey}.{n}"], np.float32) for n in
              ("weight", "bias", "running_mean", "running_var")] if bnkey else [None] * 4
        if s2x:
            # stride-2 conv of a dense 32-channel tensor read as x-pairs (row = even pixel's channels | odd pixel's): tap
            # (ky,kx) reads the even half for kx = 1 and the odd half for kx = 0 (pair ox-1) / kx = 2 (pair ox)
            co, ci = w.shape[:2]
            w2 = np.zeros((co, 2 * ci, 3, 3), np.float32)
            for kx in range(3):
                off = 0 if kx == 1 else ci
                w2[:, off:off + ci, :, kx] = w[:, :, :, kx]
            w = w2
        if pair:
            # x-paired grid: channel index = dx*32 + c.  Output pixel x_out = 2j+dxo reads input pixel
            # x_in = 2(j+pt-1)+dxi through the original tap kx = x_in - x_out + 1 (zero block if outside 0..2)
            co, ci = w.shape[:2]
            w2 = np.zeros((2 * co, 2 * ci, 3, 3), np.float32)
            for dxo in range(2):
                for dxi in range(2):
                    for pt in range(3):
                        kx = 2 * (pt - 1) + dxi - dxo + 1
                        if 0 <= kx <= 2:
                            w2[dxo * co:(dxo + 1) * co, dxi * ci:(dxi + 1) * ci, :, pt] = w[:, :, :, kx]
            w = w2
            cb = None if cb is None else np.tile(cb, 2)
            bn = [None if b is None else np.tile(b, 2) for b in bn]
        cout, cin, k, _ = w.shape
        wp = np.zeros((cout_pad, k * k, cin_pad), self.npw)
        bias = np.zeros(cout_pad, np.float32)
        p = lambda a: None if a is None else a.ctypes.data
        L.check(self.lib.acr_b200_pack_conv(p(w), p(cb), p(bn[0]), p(bn[1]), p(bn[2]), p(bn[3]), BN_EPS, cout, cin, k,
                                            cout_pad, cin_pad, self.plan_dt, wp.ctypes.data, bias.ctypes.data),
                "pack_conv " + wkey)
        return blob.add(wp), blob.add(bias)

    def _pack_deconv(self, sd, blob: _Blob, wkey: str, bnkey: str, cin_pad: int, cout_pad: int) -> Tuple[int, int]:
        """ConvTranspose2d + BN -> [4 parities][cout_pad][4 taps][cin_pad] 16-bit (BN folded by pack_conv, parity by
        parity) + fp32 bias[cout_pad] (csrc/conv_tc.cuh MODE_DECONV)."""
        par = deconv_parity_weights(np.ascontiguousarray(sd[wkey + ".weight"], np.float32))
        bn = [np.ascontiguousarray(sd[f"{bnkey}.{n}"], np.float32) for n in ("weight", "bias", "running_mean", "running_var")]
        cout, cin = par.shape[1:3]
        wp = np.zeros((4, cout_pad, 4, cin_pad), self.npw)
        bias = np.zeros(cout_pad, np.float32)
        for p in range(4):
            w = np.ascontiguousarray(par[p])
            L.check(self.lib.acr_b200_pack_conv(w.ctypes.data, None, *(b.ctypes.data for b in bn), BN_EPS, cout, cin, 2,
                                                cout_pad, cin_pad, self.plan_dt, wp[p].ctypes.data, bias.ctypes.data),
                    "pack_conv " + wkey)
        return blob.add(wp), blob.add(bias)

    def _pack_raw(self, blob: _Blob, w: np.ndarray, cin_pad: int, cout_pad: int) -> int:
        cout, cin, k, _ = w.shape
        wp = np.zeros((cout_pad, k * k, cin_pad), self.npw)
        bias = np.zeros(cout_pad, np.float32)
        w = np.ascontiguousarray(w, np.float32)
        L.check(self.lib.acr_b200_pack_conv(w.ctypes.data, None, None, None, None, None, BN_EPS, cout, cin, k,
                                            cout_pad, cin_pad, self.plan_dt, wp.ctypes.data, bias.ctypes.data), "pack_conv")
        return blob.add(wp)

    def _pack_stem(self, sd, blob: _Blob, wkey: str, bnkey: str, kch: int) -> Tuple[int, int]:
        """Stem conv (64,3,k,k) OIHW + BN as a (64, kch, 1, 1) GEMM with input channel (ky*k+kx)*3+ci (BN folded by
        pack_conv): kch = 32 for the 3x3 stem (27 taps), 160 for the 7x7 one (147 taps)."""
        w = np.ascontiguousarray(sd[wkey + ".weight"], np.float32)
        ks = w.shape[-1]
        w1 = np.zeros((64, kch, 1, 1), np.float32)
        w1[:, :3 * ks * ks, 0, 0] = w.transpose(0, 2, 3, 1).reshape(64, 3 * ks * ks)
        sd_stem = {"stem.weight": w1}
        for nme in ("weight", "bias", "running_mean", "running_var"):
            sd_stem[f"stembn.{nme}"] = np.ascontiguousarray(sd[f"{bnkey}.{nme}"], np.float32)
        return self._pack_conv(sd_stem, blob, "stem", "stembn", False, kch, 64)

    def _pack_merged(self, sd, blob: _Blob, wkeys, bnkeys, has_bias: bool, k: int, cin_pad: int, each: int) -> Tuple[int, int]:
        """Convs of identical geometry on the same input as one wide conv: weights / biases concatenated along cout."""
        wps, bs = [], []
        for wk, bk in zip(wkeys, bnkeys):
            tmp = _Blob()
            self._pack_conv(sd, tmp, wk, bk, has_bias, cin_pad, each)
            raw = tmp.tobytes()
            nw = each * k * k * cin_pad * np.dtype(self.npw).itemsize
            wps.append(np.frombuffer(raw[:nw], self.npw))
            boff = _rup(nw, 256)
            bs.append(np.frombuffer(raw[boff: boff + each * 4], np.float32))
        return blob.add(np.concatenate(wps)), blob.add(np.concatenate(bs))

    @staticmethod
    def fold_weights(sd, side: str) -> np.ndarray:
        """contact_layers[4|5] (109, 218) folded onto the 128-wide head tensor: out = W[:, :109].pm + W[:, 109:112].pm[:3]
        + (b + W[:, 112:].pare), pm = [cam3 | params106] (acr/model.py:158-164); input channel order of the 128-wide
        tensor: params at 0..105, cam at 112..114.  -> (109, 128, 1, 1) fp32."""
        W = np.ascontiguousarray(sd[f"contact_layers.{4 if side == 'l' else 5}.weight"], np.float32).reshape(109, 218)
        weff = np.zeros((109, 128, 1, 1), np.float32)
        weff[:, :106, 0, 0] = W[:, 3:109]
        weff[:, 112:115, 0, 0] = W[:, 0:3] + W[:, 109:112]
        return weff

    # --------------------------------------------------------------------- plan
    def _build(self, sd, reuse_memory: bool, shared_weights: Optional[torch.Tensor] = None) -> None:
        spec, B = self.spec, self.batch
        blob = _Blob()
        ops = spec.ops
        if self.head_only:   # ACR.head_forward: everything after the trunk; feat32 (channels 0..31 of xcat) is external
            first = next(i for i, op in enumerate(ops) if op.kind == "coordcat")
            ops = ops[first:]

        # ---- memory geometry of every tensor
        geo: Dict[str, dict] = {}

        def geom(t: Tensor) -> dict:
            root = t.base or t
            if root.name not in geo:
                if root.dtype == "u8":
                    g = dict(stride=root.C, esz=1, dt=L.DT_U8)
                elif root.dtype == "f32":
                    g = dict(stride=_rup(root.C, 16), esz=4, dt=L.DT_F32)
                else:
                    g = dict(stride=_rup(root.C, 16), esz=self.esz, dt=self.dt)
                g["bytes"] = B * root.H * root.W * g["stride"] * g["esz"]
                g["offset"] = None
                geo[root.name] = g
            return geo[root.name]

        # flat fp32 scratch tensors of the part branch
        part = Tensor("pool_part", POOL_CHUNKS * POOL_PART_FLOATS, 1, 1, "f32")
        pooled = spec.tensors["pooled"]
        pooled.C, pooled.H, pooled.W = 256 * 32, 1, 1
        bias_img = {s: Tensor(f"{s}_bias_img", 112, 1, 1, "f32") for s in "lr"}
        pare = {s: Tensor(f"{s}_pare", 106, 1, 1, "f32") for s in "lr"}
        for t in [part] + list(bias_img.values()) + list(pare.values()):
            spec.tensors[t.name] = t

        # ---- expand the spec ops into launch records (python dicts first)
        recs: List[dict] = []
        for op in ops:
            if op.kind == "pool":
                recs.append(dict(kind=L.OP_POOL, out=part, ins=[op.ins[0], op.ins[1]]))
            elif op.kind == "parthead":
                if op.attrs["side"] == "l":   # one launch serves both sides
                    recs.append(dict(kind=L.OP_PARTHEAD, out=pooled, ins=[part],
                                     aux=[bias_img["l"], bias_img["r"], pare["l"], pare["r"]]))
                s = op.attrs["side"]   # folded contact_layers[4|5]: 1x1 conv 128 -> 109 with a per-image bias
                recs.append(dict(kind=L.OP_CONV_REF if self.debug_ref_conv else L.OP_CONV, out=op.out,
                                 ins=[op.ins[1]], aux=[bias_img[s]],
                                 attrs=dict(k=1, s=1, relu=False, residual=False, pow11=False, fold_side=s)))
            elif op.kind == "stem" and op.attrs.get("k") == 7:
                # ResNet conv1 7x7 s2 + bn1 + relu: the same shared-memory-operand GEMM with K = 147 taps + bias (160)
                if not (_pow2(op.out.W // 16) and _pow2(op.out.H // 16)):
                    raise L.AcrB200Error(f"Engine: the 7x7 stem needs power-of-two tile counts, input {self.input_size} "
                                         "is not a power-of-two multiple of 512")
                recs.append(dict(kind=L.OP_STEM_TC, out=op.out, ins=[op.ins[0]], attrs=dict(stem=op.attrs)))
            elif op.kind == "maxpool":
                recs.append(dict(kind=L.OP_MAXPOOL, out=op.out, ins=[op.ins[0]]))
            elif op.kind == "deconv":
                recs.append(dict(kind=L.OP_CONV, out=op.out, ins=[op.ins[0]], attrs=op.attrs))
            elif op.kind == "stem" and self.stem_on_tensor_cores and not self.debug_ref_conv \
                    and os.environ.get("ACR_B200_STEM_FUSED", "1") != "0" and _pow2(op.out.W // 16) and _pow2(op.out.H // 16):
                # conv1 + bn1 + relu as ONE wgmma GEMM whose im2col operand is built in shared memory (csrc/stem_tc.cu)
                recs.append(dict(kind=L.OP_STEM_TC, out=op.out, ins=[op.ins[0]], attrs=dict(stem=op.attrs)))
            elif op.kind == "stem" and self.stem_on_tensor_cores:
                # conv1 + bn1 + relu as im2col (27 normalised taps -> 32 channels) + a 1x1 wgmma conv
                cols = Tensor("stem_im2col", 32, op.out.H, op.out.W, "act")
                spec.tensors[cols.name] = cols
                recs.append(dict(kind=L.OP_IM2COL_STEM, out=cols, ins=[op.ins[0]]))
                recs.append(dict(kind=L.OP_CONV_REF if self.debug_ref_conv else L.OP_CONV, out=op.out, ins=[cols],
                                 attrs=dict(k=1, s=1, relu=True, residual=False, pow11=False, stem=op.attrs)))
            elif op.kind == "coordcat":
                recs.append(dict(kind=L.OP_COORD, out=op.out, ins=[op.ins[0]]))
            else:
                kind = {"stem": L.OP_STEM, "conv": L.OP_CONV_REF if self.debug_ref_conv else L.OP_CONV,
                        "fuse": L.OP_FUSE, "bilinear2x": L.OP_BILINEAR2X}[op.kind]
                recs.append(dict(kind=kind, out=op.out, ins=list(op.ins), attrs=op.attrs))
        self.recs = recs

        # ---- liveness (by root tensor) and arena offsets
        keep = {"segms", "l_center_map", "r_center_map", "l_prior_maps", "r_prior_maps", "l_params_maps",
                "r_params_maps", "pooled", "l_pare", "r_pare"}
        keep |= set(self.keep_extra)
        keep_roots = {(spec.tensors[k].base or spec.tensors[k]).name for k in keep}
        last_use: Dict[str, int] = {}
        for i, r in enumerate(recs):
            for t in r["ins"] + [r["out"]] + r.get("aux", []):
                last_use[(t.base or t).name] = i
        arena = _Arena()
        if self.head_only:      # the external feature is copied into the coord-concat buffer before the run
            xcat = spec.tensors["feat32"].base
            geom(xcat)["offset"] = arena.alloc(geom(xcat)["bytes"])
            keep_roots.add(xcat.name)
        for i, r in enumerate(recs):
            for t in [r["out"]] + r.get("aux", []):
                g = geom(t)
                if g["offset"] is None:
                    g["offset"] = arena.alloc(g["bytes"])
            for t in r["ins"]:
                g = geom(t)
                if t.dtype != "u8":
                    assert g["offset"] is not None, f"{t.name} read before written"
            if reuse_memory:
                for name, lu in last_use.items():
                    if lu == i and name not in keep_roots and name != "image" and geo[name]["offset"] is not None \
                            and not geo[name].get("freed"):
                        arena.release(geo[name]["offset"], geo[name]["bytes"])
                        geo[name]["freed"] = True
        self.arena_bytes = max(arena.top, ALIGN)
        for g in geo.values():
            if g["offset"] is not None:
                self.arena_bytes = max(self.arena_bytes, g["offset"] + _rup(g["bytes"], ALIGN))
        self.geo = geo
        self.n_ops = len(recs)

        def pairable(r) -> bool:
            """3x3 stride-1 32->32 convs on dense tensors run as 64->64 convs on the x-paired grid: same
            bytes in memory, but 128-byte operand rows (SWIZZLE_128B) instead of 64-byte ones."""
            a = r.get("attrs", {})
            if self.f32 or r["kind"] not in (L.OP_CONV, L.OP_CONV_REF) or "fold_side" in a or a.get("k") != 3 or a.get("s") != 1:
                return False
            ts = r["ins"] + [r["out"]]
            return all(t.C == 32 and t.base is None and t.dtype == "act" and t.W % 32 == 0 for t in ts)

        def block_pair(i) -> bool:
            """recs i, i + 1 are one BasicBlock that the fused kernel takes (csrc/conv_block.cuh): conv3x3-BN-ReLU, then
            conv3x3-BN + the block input, ReLU, both 64 -> 64 or both x-paired 32 -> 32, and nothing else reads the
            intermediate."""
            if self.f32 or i + 1 >= len(recs):
                return False
            r1, r2 = recs[i], recs[i + 1]
            if r1["kind"] != L.OP_CONV or r2["kind"] != L.OP_CONV:
                return False
            a1, a2 = r1.get("attrs", {}), r2.get("attrs", {})
            special = ("extra", "merged", "fold_side", "stem", "deconv", "pow11")
            if any(a.get(k) for a in (a1, a2) for k in special):
                return False
            if not all(a.get("k") == 3 and a.get("s") == 1 and a.get("relu") for a in (a1, a2)):
                return False
            x, y = r1["ins"][0], r1["out"]
            if a1.get("residual") or not a2.get("residual") or len(r2["ins"]) != 2 \
                    or r2["ins"][0] is not y or r2["ins"][1] is not x:
                return False
            if y.base is not None or last_use[y.name] != i + 1:
                return False
            if pairable(r1) and pairable(r2):
                return True
            return x.C == y.C == r2["out"].C == 64 and x.dtype == y.dtype == r2["out"].dtype == "act"

        # BasicBlocks run as one launch each; the records stay one per spec op
        self.block_starts = [i for i in range(len(recs)) if block_pair(i)]
        for i in self.block_starts:
            recs[i]["block"] = True
            recs[i]["block_mid"] = not reuse_memory or recs[i]["out"].name in keep_roots

        def bottleneck_triple(i) -> bool:
            """recs i .. i + 2 are one Bottleneck that the fused kernel takes (csrc/conv_bottleneck.cuh): 1x1 C_in -> 64
            (C_in 64 or 256), 3x3 64 -> 64, 1x1 64 -> 256 + residual, stride 1, ReLU on all three; the residual is the
            block input or a downsample's output; and neither intermediate is observable (reuse_memory=False keeps
            every tensor, keep_extra may name one): those triples stay three launches."""
            if self.f32 or not reuse_memory or i + 2 >= len(recs):
                return False
            rs = recs[i: i + 3]
            if any(r["kind"] != L.OP_CONV for r in rs):
                return False
            at = [r.get("attrs", {}) for r in rs]
            special = ("extra", "merged", "fold_side", "stem", "deconv", "pow11")
            if any(a.get(k) for a in at for k in special):
                return False
            if [(a.get("k"), a.get("s"), bool(a.get("relu")), bool(a.get("residual"))) for a in at] != \
                    [(1, 1, True, False), (3, 1, True, False), (1, 1, True, True)]:
                return False
            x, y1, y2, out = rs[0]["ins"][0], rs[0]["out"], rs[1]["out"], rs[2]["out"]
            if len(rs[1]["ins"]) != 1 or rs[1]["ins"][0] is not y1 or len(rs[2]["ins"]) != 2 or rs[2]["ins"][0] is not y2:
                return False
            res = rs[2]["ins"][1]
            downsample = any(r["kind"] == L.OP_CONV and r["out"] is res and r["ins"][0] is x for r in recs[:i])
            if res is not x and not downsample:
                return False
            ts = (x, y1, y2, out, res)
            if not (x.C in (64, 256) and y1.C == y2.C == 64 and out.C == res.C == 256 and
                    all(t.base is None and t.dtype == "act" for t in ts)):
                return False
            return all(y.name not in keep_roots and last_use[y.name] == j for y, j in ((y1, i + 1), (y2, i + 2)))

        # Bottlenecks run as one launch each, kept apart from the BasicBlocks
        self.bottleneck_starts = [i for i in range(len(recs)) if bottleneck_triple(i)]
        for i in self.bottleneck_starts:
            recs[i]["bottleneck"] = True

        if self.dry_run:
            return

        def ctensor(t: Tensor, pair: bool = False) -> L.Tensor:
            g = geom(t)
            ct = L.Tensor()
            ext = t.dtype == "u8"
            ct.offset = 0 if ext else g["offset"] + (t.c_off * g["esz"] if t.base is not None else 0)
            ct.C, ct.H, ct.W = t.C, t.H, t.W
            ct.pix_stride, ct.dtype, ct.external = g["stride"], g["dt"], int(ext)
            if pair:   # dense 32-channel NHWC seen as (H, W/2, 64): two x-adjacent pixels form one 128-byte row
                assert t.base is None and g["stride"] == t.C == 32 and t.W % 2 == 0 and not self.f32
                ct.C, ct.W, ct.pix_stride = 64, t.W // 2, 64
            return ct

        def s2x_able(r) -> bool:
            """3x3 stride-2 convs of a DENSE 32-channel tensor read it as x-pairs (H, W/2, 64): two boxes per tile with
            128-byte rows instead of nine 64-byte-row boxes of four parity views (csrc/conv_tc.cu MODE_S2X)."""
            a = r.get("attrs", {})
            if self.f32 or r["kind"] != L.OP_CONV or a.get("k") != 3 or a.get("s") != 2 or a.get("merged") or "stem" in a:
                return False
            x, y = r["ins"][0], r["out"]
            return x.C == 32 and x.base is None and x.dtype == "act" and x.W % 32 == 0 and y.H % 16 == 0 and y.W % 16 == 0

        # ---- weights + C op records
        f32 = lambda k: np.ascontiguousarray(sd[k], np.float32)
        cops = (L.Op * len(recs))()
        for i, r in enumerate(recs):
            o = cops[i]
            o.kind = r["kind"]
            pair = pairable(r)
            s2x = s2x_able(r)
            o.out = ctensor(r["out"], pair)
            o.n_in = len(r["ins"])
            for j, t in enumerate(r["ins"]):
                o.in_[j] = ctensor(t, pair or (s2x and j == 0))
            for j, t in enumerate(r.get("aux", [])):
                o.aux[j] = ctensor(t)
            a = r.get("attrs", {})
            if r["kind"] in (L.OP_CONV, L.OP_CONV_REF):
                x = r["ins"][0]
                o.k, o.stride, o.relu, o.has_residual = a["k"], a["s"], int(a["relu"]), int(a["residual"])
                # K per tap: 33/34-channel inputs are padded to ONE 64-channel chunk (TMA zero-fills the
                # channels beyond the 48-wide buffer) instead of three 16-channel chunks: a TMA box costs
                # ~620 clk whatever its size, so fewer, fatter boxes win (tools/tma_bench.cu)
                # (same rule for the wider trunks: 48 -> 64, 96 -> 128 with zero-filled tails)
                o.cin_pad = _rup(x.C, 64) if x.C > 32 else _rup(x.C, 16)
                o.cout_pad = _rup(r["out"].C, 16)
                if a.get("extra"):
                    o.shift[0] |= L.CONV_EXTRA
                    for q, (_, sh) in enumerate(a["extra"]):
                        o.shift[1 + q] = sh
                if a.get("deconv"):
                    o.cin_pad = _rup(x.C, 64)
                    o.w_offset[0], o.w_offset[1] = self._pack_deconv(sd, blob, a["w"], a["bn"], o.cin_pad, o.cout_pad)
                    o.shift[0] |= L.CONV_DECONV
                elif "stem" in a:
                    o.cin_pad, o.cout_pad = 32, 64
                    o.w_offset[0], o.w_offset[1] = self._pack_stem(sd, blob, a["stem"]["w"], a["stem"]["bn"], 32)
                elif "fold_side" in a:
                    o.cin_pad = 128
                    o.w_offset[0] = self._pack_raw(blob, self.fold_weights(sd, a["fold_side"]), o.cin_pad, o.cout_pad)
                    o.shift[0] |= L.CONV_BIAS_PER_IMAGE   # aux[0] = bias_img from the part head
                elif s2x:
                    o.cin_pad = 64
                    o.w_offset[0], o.w_offset[1] = self._pack_conv(sd, blob, a["w"], a["bn"], a["bias"], 64, o.cout_pad, s2x=True)
                    o.shift[0] |= L.CONV_S2X
                elif pair:
                    o.cin_pad = o.cout_pad = 64
                    o.w_offset[0], o.w_offset[1] = self._pack_conv(sd, blob, a["w"], a["bn"], a["bias"], 64, 64, pair=True)
                    o.shift[0] |= L.CONV_XPAIR
                elif a.get("merged"):
                    o.w_offset[0], o.w_offset[1] = self._pack_merged(sd, blob, a["w"], a["bn"], a["bias"], a["k"], o.cin_pad,
                                                                     a["merged"])
                else:
                    o.w_offset[0], o.w_offset[1] = self._pack_conv(sd, blob, a["w"], a["bn"], a["bias"], o.cin_pad, o.cout_pad)
                    if a.get("pow11"):
                        o.shift[0] |= L.CONV_POW11_CH0
                if r.get("block"):
                    o.shift[0] |= L.CONV_BLOCK | (L.CONV_BLOCK_MID if r["block_mid"] else 0)
                if r.get("bottleneck"):
                    o.shift[0] |= L.CONV_BOTTLENECK
            elif r["kind"] == L.OP_STEM_TC:
                ks = sd[a["stem"]["w"] + ".weight"].shape[-1]
                o.w_offset[0], o.w_offset[1] = self._pack_stem(sd, blob, a["stem"]["w"], a["stem"]["bn"], 32 if ks == 3 else 160)
                if ks == 7:   # k = 7 in the op
                    o.k = 7
            elif r["kind"] == L.OP_STEM:
                w = f32(a["w"] + ".weight")                                   # (64,3,3,3) OIHW
                g_, b_, m_, v_ = (f32(f"{a['bn']}.{n}") for n in ("weight", "bias", "running_mean", "running_var"))
                sc = g_ / np.sqrt(v_ + BN_EPS)
                wt = (w * sc[:, None, None, None]).transpose(2, 3, 1, 0).reshape(27, 64)  # [(ky,kx,ci)][co]
                o.w_offset[0] = blob.add(wt.astype(np.float32))
                o.w_offset[1] = blob.add((b_ - m_ * sc).astype(np.float32))
            elif r["kind"] == L.OP_FUSE:
                o.relu = int(a["relu"])
                for j, sh in enumerate(a["shifts"]):
                    o.shift[j] = sh
            elif r["kind"] == L.OP_PARTHEAD:
                keys = ["contact_layers.2.weight", "contact_layers.3.weight", "cam_shape_layers.1.0.weight",
                        "cam_shape_layers.1.0.bias", "cam_shape_layers.2.weight", "cam_shape_layers.3.weight",
                        "cam_shape_layers.2.bias", "cam_shape_layers.3.bias", "contact_layers.4.weight",
                        "contact_layers.5.weight", "contact_layers.4.bias", "contact_layers.5.bias"]
                for j, k in enumerate(keys):
                    o.w_offset[j] = blob.add(f32(k).reshape(-1))
        self.n_ops = len(recs)
        self._cops = cops
        if shared_weights is not None:     # same dtype / flags => byte-identical blob (packing is deterministic)
            if shared_weights.numel() != blob.size or shared_weights.device != self.device:
                raise L.AcrB200Error("Engine: the shared weight blob does not match this plan")
            self.weights = shared_weights
        else:
            self.weights = torch.frombuffer(bytearray(blob.tobytes()), dtype=torch.uint8).to(self.device)
        with torch.cuda.device(self.device):
            self.arena = torch.zeros(self.arena_bytes, dtype=torch.uint8, device=self.device)
            plan = C.c_void_p()
            L.check(self.lib.acr_b200_plan_create(cops, len(recs), B, self.arena.data_ptr(), self.arena_bytes,
                                                  self.weights.data_ptr(), self.weights.numel(), self.plan_dt, C.byref(plan)),
                    "plan_create")
        self.plan = plan

    def __del__(self):
        try:
            if getattr(self, "plan", None):
                self.lib.acr_b200_plan_destroy(self.plan)
                self.plan = None
        except Exception:
            pass

    # ---------------------------------------------------------------------- run
    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def run(self, image: torch.Tensor) -> None:
        """image: uint8 CUDA tensor (B, S, S, 3) RGB on this engine's device.  Asynchronous on that device's
        current stream.  Outputs (``view`` / ``map_nchw`` / ``parse_inputs``) alias the arena: they are valid
        until the next ``run`` on this engine."""
        if self.head_only:
            raise L.AcrB200Error("Engine.run: this is a heads-only plan, use run_heads(x)")
        if not (image.is_cuda and image.dtype == torch.uint8 and image.is_contiguous()):
            raise L.AcrB200Error("Engine.run expects a contiguous uint8 CUDA tensor (B,H,W,3)")
        if image.device != self.device:
            raise L.AcrB200Error(f"Engine.run: image lives on {image.device}, the plan on {self.device}")
        if tuple(image.shape) != (self.batch, self.input_size, self.input_size, 3):
            raise L.AcrB200Error(f"Engine.run: expected {(self.batch, self.input_size, self.input_size, 3)}, got {tuple(image.shape)}")
        with torch.cuda.device(self.device):
            self.run_count += 1
            L.check(self.lib.acr_b200_plan_run(self.plan, image.data_ptr(), self._stream()), "plan_run")

    def run_heads(self, x: torch.Tensor) -> None:
        """x: (B,32,S/4,S/4) backbone feature (any float dtype, NCHW like the reference's head_forward input).
        Copied (and rounded to the storage type) into channels 0..31 of the coord-concat buffer, then the
        heads-only plan runs."""
        if not self.head_only:
            raise L.AcrB200Error("Engine.run_heads needs an engine built with head_only=True")
        F = self.input_size // 4
        if tuple(x.shape) != (self.batch, 32, F, F) or not x.is_cuda or x.device != self.device:
            raise L.AcrB200Error(f"Engine.run_heads: expected a CUDA tensor {(self.batch, 32, F, F)} on {self.device}")
        with torch.cuda.device(self.device):
            self.run_count += 1
            self.view("feat32")[..., :32].copy_(x.permute(0, 2, 3, 1))
            L.check(self.lib.acr_b200_plan_run(self.plan, None, self._stream()), "plan_run")

    def profile(self, image: torch.Tensor) -> Dict[int, Tuple[float, int]]:
        """One serialised, event-bracketed pass: {op kind: (device ms, launches)}."""
        ms = np.zeros(16, np.float32)
        cnt = np.zeros(16, np.int32)
        with torch.cuda.device(self.device):
            L.check(self.lib.acr_b200_plan_profile(self.plan, image.data_ptr(), self._stream(), ms.ctypes.data,
                                                   cnt.ctypes.data), "plan_profile")
        return {k: (float(ms[k]), int(cnt[k])) for k in range(16) if cnt[k]}

    def profile_ops(self, image: torch.Tensor) -> np.ndarray:
        """One serialised, event-bracketed pass: device ms of every record, in the order of ``recs``.  The two convs of a
        fused BasicBlock (or the three of a fused Bottleneck) are one launch: its time is on the first, the others read 0
        (``launch_of_rec``)."""
        ms = np.zeros(self.n_ops, np.float32)
        with torch.cuda.device(self.device):
            L.check(self.lib.acr_b200_plan_profile_ops(self.plan, image.data_ptr(), self._stream(), ms.ctypes.data),
                    "plan_profile_ops")
        return ms

    @property
    def num_launches(self) -> int:
        return int(self.lib.acr_b200_plan_num_launches(self.plan))

    def launch_of_rec(self) -> np.ndarray:
        """Index of the launch that computes each record (the convs of a fused BasicBlock or Bottleneck share one)."""
        out = np.zeros(self.n_ops, np.int32)
        L.check(self.lib.acr_b200_plan_op_launch(self.plan, out.ctypes.data), "plan_op_launch")
        return out

    # ------------------------------------------------------------------ outputs
    def view(self, name) -> torch.Tensor:
        """NHWC view of a tensor (name or netspec.Tensor) inside the arena, no copy: (B,H,W,stride - c_off)
        starting at the tensor's first channel (channel slices of a wider buffer start at their c_off)."""
        t = self.spec.tensors[name] if isinstance(name, str) else name
        g = self.geo[(t.base or t).name]
        if g["offset"] is None:
            raise L.AcrB200Error(f"tensor {t.name} is not part of this plan")
        tdt = {L.DT_F32: torch.float32, L.DT_BF16: torch.bfloat16, L.DT_F16: torch.float16}[g["dt"]]
        n = self.batch * t.H * t.W * g["stride"]
        off = g["offset"]
        flat = self.arena[off: off + n * g["esz"]].view(tdt)
        v = flat.view(self.batch, t.H, t.W, g["stride"])
        return v[..., t.c_off:] if t.base is not None and t.c_off else v

    def map_nchw(self, name) -> torch.Tensor:
        """fp32 NCHW copy of a tensor with its logical channel count (the reference's layout)."""
        t = self.spec.tensors[name] if isinstance(name, str) else name
        return self.view(t)[..., : t.C].permute(0, 3, 1, 2).float().contiguous()

    def parse_inputs(self) -> Dict[str, tuple]:
        out = {}
        for s in "lr":
            out[f"{s}_center"] = (self.view(f"{s}_center_map"), 16)
            out[f"{s}_params"] = (self.view(f"{s}_params_maps"), 112)
            out[f"{s}_prior"] = (self.view(f"{s}_prior_maps"), 112)
        return out

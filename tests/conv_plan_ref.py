"""Restatement of the wgmma conv's launch plan (test infrastructure): conv_tc_prepare (csrc/conv_tc.cu) and launch_mode /
launch_inst (csrc/conv_tc.cuh), in their order, so that a test can say which kernel instance and which runtime branches
a conv reaches without a GPU.

``prepare(ConvArgs(...), num_sms)`` -> ``Plan``: the instance key (T, CK, MODE, NT) of conv_tc_kernel, the plan fields
the kernel branches on (patch1, nsplit, nsub, b_resident, SB, SA, pingpong, tma_out, plain), the grid and the dynamic
shared memory in bytes.  Arguments conv_tc_prepare or launch_mode reject raise ``Rejected``.
``compiled_instances()``: every (T, CK, MODE, NT) launch_mode can launch, i.e. every template instance it compiles.
``combination(plan)``: what one op-level case of tests/test_gpu_conv_instances.py must reach, per instance: the
instance, ping-pong teams, the short epilogue, the TMA-store epilogue, fp32 output, an N split.

Units: cin_pad / cout_pad / in_stride / out_stride are channels of the tensors' own type (fp32 for the TF32 plan), as in
ConvArgs; the plan itself counts 16-bit words (an fp32 channel is two), as conv_tc_prepare does.
"""
from dataclasses import dataclass

DT_BF16, DT_F16, DT_TF32 = 0, 1, 4          # act_dtype (acr_b200.lib.DT_*)
T_NAME = {DT_BF16: "__nv_bfloat16", DT_F16: "__half", DT_TF32: "float"}   # the kernel's T, as a demangled name spells it

# csrc/conv_tc.cuh
TILE_Y = TILE_X = 16
HALF_X = 8
MAX_NSUB = 128
SMEM_BUDGET = 224 * 1024
P1_PITCH = 24
MODE_PATCH, MODE_RESIDENT, MODE_XPAIR, MODE_P1, MODE_S2X, MODE_DECONV = 1, 2, 4, 16, 32, 64
H100_SMS = 132


class Rejected(ValueError):
    """conv_tc_prepare or launch_mode returns an error for these arguments."""


def _check(ok, what):
    if not ok:
        raise Rejected(what)


@dataclass(frozen=True)
class ConvArgs:
    """The ConvArgs fields the plan reads (csrc/ops.cuh), for act_dtype ``dt``.  in_H / in_W are the input record's
    spatial size (the x-paired forms: pairs, W / 2 of the dense tensor), out_H / out_W the output's."""
    dt: int
    batch: int
    in_H: int
    in_W: int
    out_H: int
    out_W: int
    cin_pad: int
    cout_pad: int
    in_stride: int
    out_stride: int
    k: int = 3
    stride: int = 1
    residual: bool = False
    out_f32: bool = False
    bias_per_image: bool = False
    pow11: bool = False
    n_ext: int = 0
    xpair: bool = False
    s2x: bool = False
    deconv: bool = False
    tma_env: bool = False          # ACR_B200_TMA_OUT=1 at plan creation
    out_aligned16: bool = True     # the output pointer is 16-byte aligned
    in_C: int = None               # the input record's channel count (the x-paired stride-2 form checks it); None: in_stride


@dataclass(frozen=True)
class Plan:
    key: tuple          # (T, CK, MODE, NT) of conv_tc_kernel
    patch_mode: int
    patch1: int
    nsplit: int
    nsub: int
    b_resident: int
    SB: int
    SA: int
    pingpong: int
    tma_out: int
    plain: int          # the short epilogue loop runs (16-bit T only: the fp32 kernel has no such branch)
    out_f32: int
    grid: int
    smem: int           # dynamic shared memory of the launch
    nA: int             # A loads per super-tile
    a_room: int         # SMEM_BUDGET - fixed - B region: the bytes SA is cut from


def prepare(a: ConvArgs, num_sms: int = H100_SMS) -> Plan:
    """conv_tc_prepare, then launch_mode's choice of instance."""
    _check(a.out_H % TILE_Y == 0 and a.out_W % TILE_X == 0, "output is not a multiple of the 16x16 super-tile")
    _check(a.in_stride % 8 == 0 and a.cin_pad % 16 == 0 and a.cout_pad % 16 == 0 and a.cout_pad <= 2048 and a.cin_pad <= 2048,
           "channel alignment")
    tf32 = a.dt == DT_TF32
    ew = 2 if tf32 else 1
    # (input dtype == act_dtype, fp32 for TF32: implied by ConvArgs.dt)
    _check(not tf32 or (a.out_f32 and not a.xpair and not a.s2x and not a.deconv and a.n_ext == 0),
           "the tf32 conv reads and writes fp32 tensors and has no x-paired, transposed or extra-term form")
    cin_pad, in_stride = a.cin_pad * ew, a.in_stride * ew
    _check(not a.deconv or (a.k == 4 and a.stride == 2 and a.cin_pad % 64 == 0 and not a.residual and a.n_ext == 0 and
                            not a.xpair and not a.s2x and not a.bias_per_image and not a.pow11 and
                            a.out_H == 2 * a.in_H and a.out_W == 2 * a.in_W and a.in_H % TILE_Y == 0 and a.in_W % TILE_X == 0),
           "the transposed conv is k4 s2 p1 over whole 16x16 input tiles, 64-channel K chunks, no residual")
    _check(a.deconv or a.k in (1, 3), "kernel size")
    _check(not a.xpair or (a.k == 3 and a.stride == 1 and a.cin_pad == 64 and a.cout_pad == 64 and a.in_stride >= 64),
           "the x-paired form is a 3x3 stride-1 64->64 conv")
    in_C = a.in_stride if a.in_C is None else a.in_C
    _check(not a.s2x or (a.k == 3 and a.stride == 2 and a.cin_pad == 64 and a.in_stride == 64 and in_C == 64 and not a.xpair and
                         a.in_H == 2 * a.out_H and a.in_W == a.out_W),
           "the x-paired stride-2 form reads a dense 32-channel tensor as (H, W/2, 64)")
    _check(a.out_stride % 2 == 0, "output / residual rows must hold channel pairs")   # (residual rows: cout_pad wide here)
    ck = 64 if cin_pad % 64 == 0 else (32 if cin_pad % 32 == 0 else 16)
    patch_mode = 1 if (a.k == 3 and a.stride == 1) else 0
    patch1 = 1 if (patch_mode and ck == 64 and not a.xpair) else 0
    s2x, deconv = int(a.s2x), int(a.deconv)
    box_rows = TILE_Y + 1 if s2x else (TILE_Y + 2 if (patch_mode or deconv) else TILE_Y)
    box_cols = P1_PITCH if (patch1 or s2x or deconv) else TILE_X
    # (tensor maps: encoded on the device side of the call; nothing here decides the instance)
    nsplit = (a.cout_pad + MAX_NSUB - 1) // MAX_NSUB
    nsub = ((a.cout_pad + nsplit - 1) // nsplit + 15) // 16 * 16
    _check(a.n_ext == 0 or not a.out_f32, "extra terms must be 16-bit tensors")
    tma_out = 1 if (a.tma_env and not deconv and not a.out_f32 and nsub % 64 == 0 and a.out_aligned16 and
                    a.out_stride % 8 == 0) else 0
    stage_out_bytes = 4 * 8192 if tma_out else 0
    taps = 4 if deconv else a.k * a.k
    cchunks = cin_pad // ck
    nt = 64 if nsub <= 64 else 128
    grid_h, grid_w = (a.in_H, a.in_W) if deconv else (a.out_H, a.out_W)
    tiles_per_img = (grid_w // TILE_X) * (grid_h // TILE_Y)
    total_tiles = tiles_per_img * a.batch
    npar = 4 if deconv else 1
    # shared-memory plan
    a_stage_bytes = box_rows * box_cols * ck * 2
    b_total = taps * cchunks * a.cout_pad * ck * 2 if (a.cout_pad <= 256 and not deconv) else 1 << 40
    bias_bytes = (a.cout_pad * 4 + 1023) & ~1023
    fixed = 1024 + bias_bytes + 512 + stage_out_bytes
    nA = cchunks if deconv else (2 if s2x else (cchunks if patch1 else (cchunks * 3 if patch_mode else taps * cchunks)))
    min_a = (3 if (patch_mode and not patch1) else 2) * a_stage_bytes
    b_resident = 1 if b_total + min_a + fixed <= SMEM_BUDGET else 0
    b_block_bytes = (a.cout_pad if b_resident else nt) * ck * 2
    if b_resident:
        last_row = (nsplit - 1) * nsub + nt
        over = (last_row - a.cout_pad if last_row > a.cout_pad else 0) * ck * 2
        b_region_bytes = (b_total + over + 1023) & ~1023
        SB = 0
    else:
        SB = 4
        while SB > 2 and SB * b_block_bytes + min_a + fixed > SMEM_BUDGET:
            SB -= 1
        b_region_bytes = (SB * b_block_bytes + 1023) & ~1023
    # (size_t in C++: a negative numerator would wrap; tests/test_cpu_conv_plan.py asserts it never is)
    a_room = SMEM_BUDGET - fixed - b_region_bytes
    SA = a_room // a_stage_bytes
    if SA > 8:
        SA = 8
    if SA > 2 * nA and not patch1:
        SA = 2 * nA
    if (patch1 or s2x or deconv) and SA > 4:
        SA = 4
    _check(SA >= 2, "shared memory plan does not fit")
    pingpong = 1 if (b_resident and nA <= SA) else 0
    smem = fixed + b_region_bytes + SA * a_stage_bytes
    nvt = total_tiles * nsplit * npar
    grid = nvt if nvt < num_sms else num_sms
    # the kernel's epilogue choice (conv_tc_kernel: `plain`; its short loop exists for 16-bit T only)
    plain = 1 if (not tf32 and not tma_out and not a.residual and not a.pow11 and a.n_ext == 0) else 0
    key = launch_mode(a.dt, ck, patch_mode, b_resident, patch1, s2x, deconv, int(a.xpair), nt)
    return Plan(key=key, patch_mode=patch_mode, patch1=patch1, nsplit=nsplit, nsub=nsub, b_resident=b_resident, SB=SB,
                SA=SA, pingpong=pingpong, tma_out=tma_out, plain=plain, out_f32=int(a.out_f32), grid=grid, smem=smem, nA=nA,
                a_room=a_room)


def launch_mode(dt, ck, patch_mode, b_resident, patch1, s2x, deconv, xpair, nt):
    """conv_tc_launch -> conv_tc_launch_{64_bf16, 64_f16, 32, 16, tf32} -> launch_mode<CK, T> -> launch_inst -> (T, CK,
    MODE, NT).  The TF32 plan has CK 64 and 32 only (its fp32 channel is two 16-bit words: conv_tc_launch_tf32)."""
    T = T_NAME[dt]
    mode = (MODE_PATCH if patch_mode else 0) | (MODE_RESIDENT if b_resident else 0)

    def inst(m):       # launch_inst: x-paired convs are NT = 64 only
        return (T, ck, m, 64 if m & MODE_XPAIR else nt)

    if dt == DT_TF32:
        _check(ck in (64, 32), "no tf32 instance of this chunk width")
        _check(not (deconv or s2x or xpair), "no tf32 form of the transposed or x-paired convs")
        if ck == 64 and patch1:
            return inst(MODE_PATCH | MODE_RESIDENT | MODE_P1 if b_resident else MODE_PATCH | MODE_P1)
    elif ck == 64:
        if deconv:
            return inst(MODE_DECONV)
        if s2x:
            return inst(MODE_RESIDENT | MODE_S2X if b_resident else MODE_S2X)
        if patch1:
            return inst(MODE_PATCH | MODE_RESIDENT | MODE_P1 if b_resident else MODE_PATCH | MODE_P1)
        if xpair:
            _check(mode == MODE_PATCH | MODE_RESIDENT, "x-paired conv needs resident weights")
            return inst(MODE_PATCH | MODE_RESIDENT | MODE_XPAIR)
    if ck == 64:
        _check(not patch_mode, "no three-box form of a 64-channel-chunk conv")
        return inst(MODE_RESIDENT if b_resident else 0)
    return inst(mode)


def compiled_instances():
    """Every (T, CK, MODE, NT) launch_mode can launch: its branches over every input, whether or not conv_tc_prepare
    can produce that input."""
    out = set()
    for dt in (DT_BF16, DT_F16, DT_TF32):
        for ck in ((64, 32) if dt == DT_TF32 else (64, 32, 16)):
            for bits in range(1 << 6):
                flags = [(bits >> i) & 1 for i in range(6)]
                for nt in (64, 128):
                    try:
                        out.add(launch_mode(dt, ck, *flags, nt))
                    except Rejected:
                        pass
    return out


def mode_name(mode):
    """MODE bits -> 'PATCH|RESIDENT|P1' etc. ('plain' for 0)."""
    names = [(MODE_PATCH, "PATCH"), (MODE_RESIDENT, "RESIDENT"), (MODE_XPAIR, "XPAIR"), (MODE_P1, "P1"),
             (MODE_S2X, "S2X"), (MODE_DECONV, "DECONV")]
    return "|".join(n for b, n in names if mode & b) or "plain"


def kernel_name(key):
    """The demangled template-argument list of an instance, as tools/sass_audit.py and the CUDA trace spell it."""
    T, ck, mode, nt = key
    return f"conv_tc_kernel<{ck}, {T}, {mode}, {nt}>"


def combination(plan: Plan):
    """(instance, pingpong, plain, tma_out, out_f32, nsplit > 1): the runtime branches of one launch."""
    return (plan.key, plan.pingpong, plan.plain, plan.tma_out, plan.out_f32, int(plan.nsplit > 1))


def sweep(num_sms: int = H100_SMS):
    """Every argument set conv_tc_prepare accepts, up to what does not change the plan (the spatial size and batch only
    move the grid, in_stride only the K tail's zero fill): cin_pad and cout_pad in steps of 16 up to 2048; k 1 and 3 at
    stride 1 and 2, the x-paired, stride-2 x-paired and transposed forms with their own preconditions; the epilogue
    terms (residual, 1.1 ** channel 0, per-image bias, extra terms) on and off; fp32 output on and off; TMA store on and
    off; all three types.  Yields (ConvArgs, Plan) for the accepted ones.

    The epilogue terms only decide `plain` and what the argument checks accept: once an argument set has given plain = 0
    its further epilogues would repeat that plan, so they are not evaluated."""
    forms = [dict(k=1, stride=1), dict(k=1, stride=2), dict(k=3, stride=1), dict(k=3, stride=2),
             dict(k=3, stride=1, xpair=True), dict(k=3, stride=2, s2x=True), dict(k=4, stride=2, deconv=True)]
    epilogues = [dict(), dict(bias_per_image=True), dict(residual=True), dict(pow11=True), dict(n_ext=1),
                 dict(residual=True, pow11=True, bias_per_image=True)]
    chans = range(16, 2049, 16)
    for dt in (DT_BF16, DT_F16, DT_TF32):
        for f in forms:
            for cin_pad in chans:
                for cout_pad in chans:
                    if f.get("xpair") and (cin_pad != 64 or cout_pad != 64):
                        continue
                    if f.get("s2x") and cin_pad != 64:
                        continue
                    if f.get("deconv") and cin_pad % 64:
                        continue
                    if f.get("deconv"):
                        geo = dict(in_H=16, in_W=16, out_H=32, out_W=32)
                    elif f.get("s2x") or f["stride"] == 2:
                        geo = dict(in_H=32, in_W=16 if f.get("s2x") else 32, out_H=16, out_W=16)
                    else:
                        geo = dict(in_H=16, in_W=16, out_H=16, out_W=16)
                    for out_f32 in (False, True):
                        for tma in (False, True):
                            seen_plain = set()
                            for e in epilogues:
                                if len(seen_plain) == 2 or (e and 0 in seen_plain):
                                    break      # every further epilogue gives plain = 0 again, with the same plan
                                a = ConvArgs(dt=dt, batch=1, cin_pad=cin_pad, cout_pad=cout_pad, in_stride=cin_pad,
                                             out_stride=cout_pad, out_f32=out_f32, tma_env=tma, **geo, **f, **e)
                                try:
                                    p = prepare(a, num_sms)
                                except Rejected:
                                    continue
                                seen_plain.add(p.plain)
                                yield a, p

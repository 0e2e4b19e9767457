"""GPU: ragged pre-processing -- frames of any sizes in one launch, and the CUDA graph from raw frames.

* acr_b200_cubic_tables == preprocess.cubic_tables bit for bit (every side 1..4096 at 512, a sample at 1024);
* one ragged batch == oracle/preprocess_ref.img_preprocess per frame, bit for bit, offsets included;
* a list of equal-size frames == the 4-D path; numpy / CPU / CUDA / non-contiguous inputs agree;
* img_preprocess(list) + batch_forward == batch_forward on the per-frame results, bit for bit;
* capture_frames_graph replays == the eager ragged path + fused_forward, bit for bit, on two size mixes.
"""
import numpy as np
import pytest
import torch

from acr_b200 import lib as L
from acr_b200.preprocess import FRAME_DTYPE, RaggedFrames, cubic_tables, preprocess_frames

pytestmark = pytest.mark.gpu

# upscaled (64x48, 1x7), odd (513x511, 37x1001), 720p, 1080p portrait and landscape, 2160x3840, and a few more
SIZES = [(64, 48), (1, 7), (513, 511), (37, 1001), (720, 1280), (1920, 1080), (1080, 1920), (2160, 3840),
         (600, 600), (7, 1), (480, 640), (1, 1)]


def _frames(shapes, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]


def _dev_tables(n_src, S):
    sides = torch.tensor(n_src, dtype=torch.int32, device="cuda")
    coef = torch.empty(len(n_src), S, 4, dtype=torch.int16, device="cuda")
    ofs = torch.empty(len(n_src), S, dtype=torch.int32, device="cuda")
    L.check(L.load().acr_b200_cubic_tables(L.ptr(sides), len(n_src), S, L.ptr(coef), L.ptr(ofs), L.current_stream()),
            "cubic_tables")
    return coef.cpu().numpy(), ofs.cpu().numpy()


def test_cubic_tables_on_device_equal_the_host_tables():
    n_src = list(range(1, 4097))
    coef, ofs = _dev_tables(n_src, 512)
    bad = [n for i, n in enumerate(n_src)
           if not (np.array_equal(coef[i], cubic_tables(n, 512)[0]) and np.array_equal(ofs[i], cubic_tables(n, 512)[1]))]
    assert not bad, f"{len(bad)} sides differ, first {bad[:8]}"
    sample = [1, 2, 3, 7, 511, 512, 513, 1000, 1023, 1024, 1025, 1080, 1920, 2160, 3840, 4096]
    coef, ofs = _dev_tables(sample, 1024)
    for i, n in enumerate(sample):
        c, o = cubic_tables(n, 1024)
        assert np.array_equal(coef[i], c) and np.array_equal(ofs[i], o), n


def test_ragged_batch_bit_exact_vs_oracle():
    from oracle import preprocess_ref
    frames = _frames(SIZES, seed=1)
    out, offs = preprocess_frames(frames)
    assert out.shape == (len(SIZES), 512, 512, 3) and offs.shape == (len(SIZES), 10)
    total = sum(h * w * 3 for h, w in SIZES)
    rf = RaggedFrames(len(SIZES), total)                 # the device-written offsets vectors
    rf.load(frames)
    out2, offs_dev = rf.launch()
    out, out2, offs_dev = out.cpu().numpy(), out2.cpu().numpy(), offs_dev.cpu().numpy()
    assert np.array_equal(out, out2)
    for i, f in enumerate(frames):
        ref, o = preprocess_ref.img_preprocess(f)
        assert np.array_equal(out[i], ref), SIZES[i]
        assert np.array_equal(offs[i].numpy(), o) and np.array_equal(offs_dev[i], o), SIZES[i]


def test_equal_sizes_match_the_4d_path_and_every_input_form():
    frames = _frames([(360, 640)] * 3, seed=2)
    ref, ref_offs = preprocess_frames(torch.from_numpy(np.stack(frames)).cuda())
    ref = ref.cpu()
    big = [np.ascontiguousarray(np.repeat(np.repeat(f, 2, 0), 2, 1)) for f in frames]     # f == big[::2, ::2]
    forms = {
        "numpy": frames,
        "cpu": [torch.from_numpy(f) for f in frames],
        "cuda": [torch.from_numpy(f).cuda() for f in frames],
        "tuple": tuple(frames),
        "numpy-strided": [b[::2, ::2] for b in big],
        "cpu-strided": [torch.from_numpy(b)[::2, ::2] for b in big],
        "cuda-strided": [torch.from_numpy(b).cuda()[::2, ::2] for b in big],
    }
    for name, fs in forms.items():
        out, offs = preprocess_frames(fs)
        assert torch.equal(out.cpu(), ref), name
        assert torch.equal(offs, ref_offs), name


def test_bad_descriptor_gives_a_zero_frame_and_leaves_the_others():
    """Descriptors are device data, so the kernel checks them: a frame with side != max(H, W) reads nothing."""
    frames = _frames([(40, 60), (50, 30), (20, 20)], seed=3)
    rf = RaggedFrames(3, sum(f.size for f in frames))
    rf.load(frames)
    good, good_offs = (t.clone() for t in rf.launch())
    desc = np.frombuffer(rf.desc.cpu().numpy().tobytes(), FRAME_DTYPE).copy()
    desc[1]["side"] = 10 ** 6
    rf.desc.copy_(torch.from_numpy(desc.view(np.uint8)))
    out, offs = rf.launch()
    assert not out[1].any() and not offs[1].any()
    assert torch.equal(out[0], good[0]) and torch.equal(out[2], good[2]) and torch.equal(offs[2], good_offs[2])
    with pytest.raises(L.AcrB200Error):
        L.check(L.load().acr_b200_preprocess_ragged(L.ptr(rf.packed), rf.max_bytes, L.ptr(rf.desc), 0, L.ptr(rf.coef),
                                                    L.ptr(rf.ofs), 512, L.ptr(rf.out), None, L.current_stream()))


# ------------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def app():
    from acr.main import ACR
    from acr_b200.synth import load_bn_calibration, make_synthetic_mano, synth_state_dict
    assets = {"left": make_synthetic_mano("left"), "right": make_synthetic_mano("right")}
    a = ACR(state_dict=synth_state_dict(0, bn_stats=load_bn_calibration(0)), mano_assets=assets)
    yield a
    del a
    torch.cuda.empty_cache()


def test_img_preprocess_list_then_batch_forward(app):
    from acr.utils import convert_kp2d_from_input_to_orgimg, img_preprocess, reorganize_results
    shapes = [(720, 1280), (1920, 1080), (64, 48), (513, 511)]
    frames = _frames(shapes, seed=4)
    paths = [f"/frames/{i:06d}.jpg" for i in range(len(frames))]
    meta = img_preprocess(frames, paths)
    assert meta["imgpath"] == paths and meta["name"] == [p.split("/")[-1] for p in paths]
    out = app.batch_forward(meta["image"], meta["offsets"])
    singles = [img_preprocess(f) for f in frames]
    ref = app.batch_forward(torch.stack([m["image"] for m in singles]), torch.stack([m["offsets"] for m in singles]))
    torch.cuda.synchronize()
    for k in ("reorganize_idx", "detection_flag", "params_pred", "verts", "j3d", "pj2d", "pj2d_org", "cam_trans"):
        assert torch.equal(out[k], ref[k]), k
    for k in ("cam", "poses", "betas"):
        assert torch.equal(out["params_dict"][k], ref["params_dict"][k]), k
    idx = out["reorganize_idx"].long().cpu()
    assert len(idx) > 0
    exp = convert_kp2d_from_input_to_orgimg(out["pj2d"], meta["offsets"][idx])
    torch.testing.assert_close(out["pj2d_org"], exp, rtol=1e-6, atol=1e-3)
    reorg = idx.numpy()
    res = reorganize_results(out, [paths[i] for i in reorg], reorg)
    assert sorted(res) == sorted({paths[i] for i in reorg})
    for p, hands in res.items():
        assert len(hands) == int((reorg == paths.index(p)).sum())


def test_frames_graph_replays_equal_eager(app):
    mix_a = _frames([(720, 1280), (64, 48), (1080, 1920), (37, 1001)], seed=5)
    mix_b = [torch.from_numpy(f).cuda() for f in _frames([(1920, 1080), (1, 7), (480, 640), (513, 511)], seed=6)]
    cap = max(sum(f.shape[0] * f.shape[1] * 3 for f in m) for m in (mix_a, mix_b))
    replay = app.capture_frames_graph(4, cap)

    def eager(fs):
        img, offs = preprocess_frames(fs)
        bufs, mano = app.fused_forward(img, offs.cuda())
        torch.cuda.synchronize()
        n = int(bufs.counts[2])
        return (bufs.counts.clone(), bufs.params_pred[:n].clone(), bufs.offsets_out[:n].clone(),
                mano["verts"][:n].clone(), mano["pj2d_org"][:n].clone())

    def graphed(fs):
        bufs, mano = replay(fs)
        torch.cuda.synchronize()
        n = int(bufs.counts[2])
        return bufs.counts, bufs.params_pred[:n], bufs.offsets_out[:n], mano["verts"][:n], mano["pj2d_org"][:n]

    names = ("counts", "params_pred", "offsets_out", "verts", "pj2d_org")
    for mix in (mix_a, mix_b):
        exp = eager(mix)
        for name, g, e in zip(names, graphed(mix), exp):
            assert torch.equal(g, e), name
    too_big = _frames([(720, 1280), (64, 48), (1080, 1920), (1200, 1000)], seed=7)
    with pytest.raises(ValueError, match="capacity"):
        replay(too_big)
    with pytest.raises(ValueError, match="exactly"):
        replay(mix_a[:3])
    exp = eager(mix_a)
    for name, g, e in zip(names, graphed(mix_a), exp):
        assert torch.equal(g, e), name

"""YUV 4:2:0 input on the device: cp_preprocess_yuv420 against cp_preprocess_ragged on cv2.cvtColor of the same frames,
bit for bit, in both layouts (every (Y, U, V) triple, the Objectron frame sizes under fix_res, keep_res, rotated,
anisotropic and up-scaling affines, a ragged batch at unaligned byte offsets); and every entry point that takes
pixel_format -- both forms of run_batch (dla_34 and res_18, tf32x3), slot tracking, the multi-category detector and
tracker, BatchPipeline and TrackPipeline -- against the same call on the cv2-converted BGR frames."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import synth
from centerpose_b200.detector import affine_from_center_scale
from tests import yuv_ref
from tests.test_gpu_streams import _rotated_crop, _seed_dets
from tests.test_gpu_tracker import _tracking_detector

pytestmark = pytest.mark.gpu
FORMATS = ("nv12", "i420")
OPT = cpb.default_opt("dla_34")


def to_bgr(f, fmt):
    import cv2
    return cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12 if fmt == "nv12" else cv2.COLOR_YUV2BGR_I420)


def from_bgr(bgr, fmt):
    """A BGR frame encoded as YUV 4:2:0 by cv2 (I420), re-packed as NV12 when asked."""
    import cv2
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    if fmt == "i420":
        return i420
    H, W = bgr.shape[:2]
    c = i420[H:].reshape(-1)
    n = H * W // 4
    return np.concatenate([i420[:H], np.stack([c[:n], c[n:]], axis=-1).reshape(H // 2, W)])


def synthetic_yuv(n, h, w, fmt, seed):
    return [from_bgr(f, fmt) for f in synth.synthetic_frames(n, h, w, seed=seed)]


def random_yuv(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


def _pack(frames, gaps=None):
    """Frames into one CUDA byte buffer, frame b after gaps[b] filler bytes -> (buffer, offsets)."""
    gaps = gaps or [0] * len(frames)
    parts, offs, off = [], [], 0
    for f, g in zip(frames, gaps):
        parts += [np.full(g, 0xA5, np.uint8), f.reshape(-1)]
        off += g
        offs.append(off)
        off += f.size
    return torch.from_numpy(np.concatenate(parts)).cuda(), np.array(offs, np.int64)


def _yuv_and_bgr(frames, fmt, dst_h, dst_w, trans=None, gaps=None):
    """(cp_preprocess_yuv420 of the frames, cp_preprocess_ragged of their cv2 conversion) as host arrays."""
    hw = np.array([(f.shape[0] * 2 // 3, f.shape[1]) for f in frames], np.int32)
    buf, offs = _pack(frames, gaps)
    got = cpb.preprocess_yuv420(buf, offs, hw, fmt, dst_h, dst_w, OPT.mean, OPT.std, trans_input=trans)
    bbuf, boffs = _pack([to_bgr(f, fmt) for f in frames])
    want = cpb.preprocess_ragged(bbuf, boffs, hw, dst_h, dst_w, OPT.mean, OPT.std, trans_input=trans)
    return got.cpu().numpy(), want.cpu().numpy()


def _same(got, want, what):
    assert got.shape == want.shape, what
    bad = np.argwhere(got != want)
    assert bad.size == 0, (what, bad[:8])


# ---- the kernel --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_every_yuv_triple(fmt, cplib):
    f = yuv_ref.exhaustive_yuv420(fmt)
    # scale 1: every output pixel is one source pixel with weight 2^15, so all 2^24 triples are converted
    got, want = _yuv_and_bgr([f], fmt, 4096, 4096, trans=np.eye(2, 3)[None])
    _same(got, want, "identity")
    # and the identity output is the normalised conversion itself
    mean, std = np.array(OPT.mean, np.float32).reshape(3, 1, 1), np.array(OPT.std, np.float32).reshape(3, 1, 1)
    bgr = yuv_ref.yuv420_to_bgr(f, fmt)[::61].transpose(2, 0, 1)
    assert np.array_equal(got[0][:, ::61], ((bgr / 255. - mean) / std).astype(np.float32))
    got, want = _yuv_and_bgr([f], fmt, 512, 512)
    _same(got, want, "fix_res")


def _affines(h, w):
    """name -> (dst_h, dst_w, forward affine or None for the kernel's own fix_res)."""
    kh, kw = (h | 31) + 1, (w | 31) + 1
    keep = affine_from_center_scale(np.array([w // 2, h // 2], np.float32), float(kw), kw, kh)
    aniso = np.array([[0.47, 0.06, 3.3], [-0.03, 0.71, -20.7]]) * np.array([[512. / w], [512. / h]]) * 1.3
    up = np.array([[3.3, 0.0, -3.3 * (w - 97.4)], [0.0, 3.1, -3.1 * 11.6]])      # crosses the right border, 3x up
    return {"fix_res": (512, 512, None), "keep_res": (kh, kw, keep), "rotated": (512, 512, _rotated_crop(h, w, 512)),
            "anisotropic": (512, 512, aniso), "upscale": (512, 512, up)}


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("h, w", [(480, 640), (600, 800), (1080, 1920), (1440, 1920)])
def test_frame_sizes_and_affines(fmt, h, w, cplib):
    f = random_yuv(h, w, seed=h + w)
    for name, (dh, dw, M) in _affines(h, w).items():
        got, want = _yuv_and_bgr([f], fmt, dh, dw, trans=None if M is None else M[None])
        _same(got, want, name)
    # the same frames cut from natural-looking content, where neighbouring chroma blocks differ gently
    g = synthetic_yuv(1, h, w, fmt, seed=h)[0]
    got, want = _yuv_and_bgr([g], fmt, 512, 512, trans=_rotated_crop(h, w, 512)[None])
    _same(got, want, "synthetic rotated")


@pytest.mark.parametrize("fmt", FORMATS)
def test_ragged_batch_at_unaligned_offsets(fmt, cplib):
    sizes = [(480, 640), (2, 2), (600, 800), (1080, 1920), (1440, 1920), (376, 500)]
    frames = [random_yuv(h, w, seed=7 * i + 1) for i, (h, w) in enumerate(sizes)]
    gaps = [1, 2, 4, 2, 6, 2]             # frames are an even number of bytes: every frame starts at an odd offset
    got, want = _yuv_and_bgr(frames, fmt, 512, 512, gaps=gaps)
    _, offs = _pack(frames, gaps)
    assert all(o % 2 for o in offs)
    _same(got, want, "fix_res")
    # frame by frame, alone: the ragged call is B single-frame calls
    for b, f in enumerate(frames):
        one, _ = _yuv_and_bgr([f], fmt, 512, 512)
        _same(got[b:b + 1], one, sizes[b])
    trans = np.stack([_affines(h, w)["anisotropic"][2] for h, w in sizes])
    got, want = _yuv_and_bgr(frames, fmt, 512, 512, trans=trans, gaps=gaps)
    _same(got, want, "anisotropic")


def test_refusals_reach_python(cplib):
    buf = torch.zeros(1000, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="needs even sizes"):
        cpb.preprocess_yuv420(buf, [0], [(9, 10)], "nv12", 64, 64, OPT.mean, OPT.std)
    with pytest.raises(RuntimeError, match="lies outside the 1000-byte buffer"):
        cpb.preprocess_yuv420(buf, [0], [(30, 30)], "i420", 64, 64, OPT.mean, OPT.std)
    with pytest.raises(ValueError, match="'nv12' or 'i420'"):
        cpb.preprocess_yuv420(buf, [0], [(10, 10)], "bgr", 64, 64, OPT.mean, OPT.std)


# ---- run_batch ---------------------------------------------------------------------------------------------------------
def _cam(h, w):
    return synth.default_camera(w, h)


def _detector(arch, frames_bgr):
    """A seeded tf32x3 detector whose heat-map biases are calibrated on the network inputs of these BGR frames (about
    4 objects per frame)."""
    opt = cpb.default_opt(arch)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=21, offset_std=0.3))
    m = m.cuda().eval()
    buf, offs = _pack(frames_bgr)
    hw = np.array([f.shape[:2] for f in frames_bgr], np.int32)
    x = cpb.preprocess_ragged(buf, offs, hw, opt.input_h, opt.input_w, opt.mean, opt.std)
    with torch.no_grad():
        synth.calibrate_head_bias(m, m(x)[-1], target=4)
    return cpb.ObjectPoseDetector(opt, model=m), opt


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("arch", ("dla_34", "res_18"))
def test_run_batch_matches_bgr(arch, fmt, cplib):
    arr = np.stack(synthetic_yuv(3, 480, 640, fmt, seed=11))
    sizes = [(480, 640), (600, 800), (720, 960), (512, 512)]
    lst = [synthetic_yuv(1, h, w, fmt, seed=20 + i)[0] for i, (h, w) in enumerate(sizes)]
    det, opt = _detector(arch, [to_bgr(f, fmt) for f in list(arr) + lst])
    assert det.model.precision == "tf32x3"
    # the array form: uint8 [B,3H/2,W] -- numpy, pinned and CUDA
    bgr = np.stack([to_bgr(f, fmt) for f in arr])
    cam = _cam(480, 640)
    wp, wn = det.run_batch(bgr, cam)
    assert wn.sum() > 0
    for src in (arr, torch.from_numpy(arr).pin_memory(), torch.from_numpy(arr).cuda()):
        gp, gn = det.run_batch(src, cam, pixel_format=fmt)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # the list form: mixed sizes, numpy / pinned / CUDA frames, one camera per frame
    cams = np.stack([_cam(h, w) for h, w in sizes])
    wp, wn = det.run_batch([to_bgr(f, fmt) for f in lst], cams)
    assert wn.sum() > 0
    mixed = [lst[0], torch.from_numpy(lst[1]).pin_memory(), torch.from_numpy(lst[2]).cuda(), torch.from_numpy(lst[3])]
    gp, gn = det.run_batch(mixed, cams, pixel_format=fmt)
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


SLOTS = [(480, 640), (600, 800), (512, 512)]
# per step: per slot True (a frame), None (idle), "new" (a new video starts in the slot)
SCHEDULE = [["new", "new", "new"], [True, True, None], ["new", True, True]]


def _slot_steps(fmt):
    vids = [[synthetic_yuv(1, h, w, fmt, seed=300 + 10 * s + k)[0] for k in range(len(SCHEDULE))]
            for s, (h, w) in enumerate(SLOTS)]
    steps = []
    for k, row in enumerate(SCHEDULE):
        frames = [vids[s][k] if e is not None else None for s, e in enumerate(row)]
        steps.append((frames, [e == "new" for e in row]))
    return steps


def _track_runs(det, fmt, pre):
    """The slot schedule through run_batch(list, track=True), then two array steps, on YUV frames and on their cv2
    conversion: per step (tracks, n_tracks) of both runs."""
    cams = np.stack([_cam(h, w) for h, w in SLOTS])
    arr = [np.stack(synthetic_yuv(3, 512, 512, fmt, seed=400 + k)) for k in range(2)]
    runs = []
    for yuv in (True, False):
        det.reset_tracking()
        out = []
        for k, (frames, new) in enumerate(_slot_steps(fmt)):
            pre_dets = [pre if (k == 0 and s == 1) else None for s in range(3)]
            if not yuv:
                frames = [to_bgr(f, fmt) if f is not None else None for f in frames]
            out.append(det.run_batch(frames, cams, track=True, new_video=new, pre_dets=pre_dets,
                                     **({"pixel_format": fmt} if yuv else {})))
        for a in arr:
            a = a if yuv else np.stack([to_bgr(f, fmt) for f in a])
            out.append(det.run_batch(a, _cam(512, 512), track=True, **({"pixel_format": fmt} if yuv else {})))
        runs.append(out)
    return runs


@pytest.mark.parametrize("fmt", FORMATS)
def test_slot_tracking_matches_bgr(fmt, cplib):
    det, opt = _tracking_detector()
    pre = _seed_dets(det, synth.synthetic_frames(1, 512, 512, seed=5)[0], _cam(512, 512))
    got, want = _track_runs(det, fmt, pre)
    assert sum(int(n.sum()) for _, n in want) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(got, want)):
        assert np.array_equal(gn, wn), k
        assert np.array_equal(gt, wt), (k, np.argwhere(gt != wt)[:8])
    assert int(got[1][1][2]) == 0 and not got[1][0][2].any()          # the idle slot


# ---- several categories ------------------------------------------------------------------------------------------------
def _category_checkpoints(tmp_path, tracking):
    opt = cpb.default_opt("dla_34", tracking_task=tracking)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=5))).cuda()
    paths = {}
    for c, s in (("chair", 3), ("cup", 4)):
        m.load_state_dict(synth.seeded_state_dict(m, seed=s, offset_std=0.3))
        if tracking:
            z = torch.zeros((2, 1, 512, 512), device="cuda")
            heads = m(x, x, z, z.repeat(1, 8, 1, 1))[-1]
        else:
            heads = m(x)[-1]
        synth.calibrate_head_bias(m, heads, target=4)
        paths[c] = str(tmp_path / (c + ".pth"))
        cpb.save_model(paths[c], 1, m)
    return opt, paths


@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_category_detector_matches_bgr(fmt, tmp_path, cplib):
    opt, paths = _category_checkpoints(tmp_path, False)
    det = cpb.MultiCategoryDetector(opt, paths)
    arr = np.stack(synthetic_yuv(2, 512, 512, fmt, seed=5))
    lst = [arr[0], synthetic_yuv(1, 600, 800, fmt, seed=6)[0]]
    cam = _cam(512, 512)
    for frames in (arr, lst):
        bgr = [to_bgr(f, fmt) for f in frames]
        wp, wn = det.run_batch(np.stack(bgr) if frames is arr else bgr, cam)
        gp, gn = det.run_batch(frames, cam, pixel_format=fmt)
        assert wn.shape == (2, 2) and (wn.sum(axis=1) > 0).all()
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_category_tracker_matches_bgr(fmt, tmp_path, cplib):
    opt, paths = _category_checkpoints(tmp_path, True)
    det = cpb.MultiCategoryTracker(opt, paths)
    cams = np.stack([_cam(h, w) for h, w in SLOTS])
    arr = np.stack(synthetic_yuv(3, 512, 512, fmt, seed=500))
    runs = []
    for yuv in (True, False):
        det.reset_tracking()
        kw = {"pixel_format": fmt} if yuv else {}
        out = []
        for frames, new in _slot_steps(fmt):
            if not yuv:
                frames = [to_bgr(f, fmt) if f is not None else None for f in frames]
            out.append(det.run_batch(frames, cams, new_video=new, **kw))
        out.append(det.run_batch(arr if yuv else np.stack([to_bgr(f, fmt) for f in arr]), _cam(512, 512), **kw))
        runs.append(out)
    assert sum(int(n.sum()) for _, n in runs[1]) > 0
    for k, ((gt, gn), (wt, wn)) in enumerate(zip(*runs)):
        assert gn.shape == (2, 3)
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt), k


# ---- pipelines ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_batch_pipeline_matches_bgr(fmt, cplib):
    batches = [np.stack(synthetic_yuv(2, 480, 640, fmt, seed=600 + k)) for k in range(3)]
    det, opt = _detector("dla_34", [to_bgr(f, fmt) for b in batches for f in b])
    cam = _cam(480, 640)
    outs = []
    for pf in (fmt, "bgr"):
        pipe = cpb.BatchPipeline(det, batch=2, height=480, width=640, camera_matrix=cam, pixel_format=pf)
        assert pipe.slots[0].u8.shape == ((2, 720, 640) if pf != "bgr" else (2, 480, 640, 3))
        got = []
        for k, b in enumerate(batches):
            if pf == "bgr":
                b = np.stack([to_bgr(f, fmt) for f in b])
            if pipe.in_flight == pipe.depth:
                got.append([a.copy() for a in pipe.collect()])
            pipe.submit(torch.from_numpy(b).pin_memory() if k % 2 else b)
        while pipe.in_flight:
            got.append([a.copy() for a in pipe.collect()])
        outs.append(got)
        with pytest.raises(ValueError, match="expected uint8 frames of shape"):
            pipe.submit(np.zeros((2, 480, 640, 3) if pf != "bgr" else (2, 720, 640), np.uint8))
    assert sum(int(n.sum()) for _, n in outs[1]) > 0
    for (gp, gn), (wp, wn) in zip(*outs):
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


@pytest.mark.parametrize("fmt", FORMATS)
def test_track_pipeline_matches_bgr(fmt, cplib):
    det, opt = _tracking_detector()
    cams = np.stack([_cam(h, w) for h, w in SLOTS])
    outs = []
    for pf in (fmt, "bgr"):
        det.reset_tracking()
        pipe = cpb.TrackPipeline(det, slots=3, camera_matrix=cams, pixel_format=pf)
        got = []
        for k, (frames, new) in enumerate(_slot_steps(fmt)):
            if pf == "bgr":
                frames = [to_bgr(f, fmt) if f is not None else None for f in frames]
            if k % 2:
                frames = [torch.from_numpy(f).pin_memory() if f is not None else None for f in frames]
            if pipe.in_flight == pipe.depth:
                got.append(pipe.collect())
            pipe.submit(frames, new_video=new)
        while pipe.in_flight:
            got.append(pipe.collect())
        outs.append(got)
    assert sum(int(n.sum()) for _, n in outs[1]) > 0
    for (gt, gn), (wt, wn) in zip(*outs):
        assert np.array_equal(gn, wn) and np.array_equal(gt, wt)

"""run()'s device pre-process on the GPU: cp_preprocess_resize_affine against cv2.resize -> cv2.warpAffine -> normalise,
bit for bit; the network input and meta run() builds on the device against pre_process in all three modes and at the
test scales; and run()'s results, at one and several scales and through a CenterPoseTrack sequence, against the same
detector's host pre_process."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import synth
from centerpose_b200.engine import preprocess
from oracle import make_golden_tracker_gt as mgt
from oracle import preprocess_ref
from tests.test_meta_geometry import MODES, _detector as _shell_detector

pytestmark = pytest.mark.gpu

OPT = cpb.default_opt("dla_34")
MEAN = np.array(OPT.mean, np.float32).reshape(1, 1, 3)
STD = np.array(OPT.std, np.float32).reshape(1, 1, 3)
CAM = np.array([[663.0287679036459, 0, 300.2775065104167], [0, 663.0287679036459, 395.00066121419275], [0, 0, 1]])


def _cv2_chain(f, T, rw, rh, dw, dh):
    import cv2
    inp = cv2.warpAffine(cv2.resize(f, (rw, rh)), T, (dw, dh), flags=cv2.INTER_LINEAR)
    return ((inp / 255. - MEAN) / STD).astype(np.float32).transpose(2, 0, 1)


def _rotated(h, w, dh, dw):
    import cv2
    M = cv2.getRotationMatrix2D((w * 0.4, h * 0.55), 30.0, min(dh, dw) / (0.6 * max(h, w)))
    M[:, 2] += np.array([dw / 2. - w * 0.4, dh / 2. - h * 0.55])
    return M


# (B, frame h x w, resized h x w, output h x w, affine)
CASES = [(1, 1440, 1920, 1080, 1440, 512, 512, "fix_res"),      # 0.75
         (3, 480, 640, 600, 800, 512, 512, "fix_res"),          # 1.25
         (1, 600, 800, 300, 400, 512, 512, "fix_res"),          # exactly one half
         (3, 481, 643, 360, 482, 256, 320, "rotated"),          # odd sizes
         (1, 61, 83, 122, 166, 96, 64, "rotated"),              # 2x
         (3, 7, 9, 16, 21, 24, 24, "rotated"),                  # tiny upscale
         (1, 3, 3, 1, 2, 8, 8, "fix_res"),                      # tiny downscale
         (3, 1, 1, 3, 2, 4, 4, "fix_res")]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d-%dx%d-to-%dx%d-%s" % (c[0], c[1], c[2], c[3], c[4], c[7]))
def test_resize_entry_is_cv2(case, cplib):
    B, sh, sw, rh, rw, dh, dw, kind = case
    frames = np.random.default_rng(sh * sw + rh).integers(0, 256, (B, sh, sw, 3), dtype=np.uint8)
    T = preprocess_ref.fix_res_affine(rh, rw, dw, dh) if kind == "fix_res" else _rotated(rh, rw, dh, dw)
    dev = torch.from_numpy(frames).cuda()
    out = torch.full((B, 3, dh, dw), float("nan"), device="cuda")
    preprocess(dev, dh, dw, OPT.mean, OPT.std, out=out, trans_input=T, resize_hw=(rh, rw))
    got = out.cpu().numpy()
    for b in range(B):
        assert np.array_equal(got[b], _cv2_chain(frames[b], T, rw, rh, dw, dh)), b
    # the frame's own size: the launch of the call without resize_hw
    same = preprocess(dev, dh, dw, OPT.mean, OPT.std, trans_input=T, resize_hw=(sh, sw))
    assert torch.equal(same, preprocess(dev, dh, dw, OPT.mean, OPT.std, trans_input=T))


def test_resize_entry_needs_the_affine(cplib):
    with pytest.raises(ValueError, match="resize_hw needs the trans_input"):
        preprocess(torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda"), 8, 8, OPT.mean, OPT.std,
                   resize_hw=(4, 4))


@pytest.mark.parametrize("h, w", [(1440, 1920), (480, 640), (800, 600), (481, 643)])
@pytest.mark.parametrize("mode", list(MODES))
def test_run_network_input_is_pre_process(mode, h, w, cplib):
    """The device input and meta of every test scale equal pre_process's, bit for bit."""
    det = _shell_detector(mode)
    det.opt.device = torch.device("cuda")
    det.scales, det._stage = [1.0, 0.75, 0.5, 1.25], None
    img = synth.synthetic_frames(1, h, w, seed=h + w)[0]
    inp = {"camera_matrix": CAM, "id": 4, "pre_dets": [{"score": 0.5}]}
    frame = det._device_frame(img)
    for scale in det.scales:
        got_x, got = det._device_pre_process(frame, scale, inp)
        want_x, want = det.pre_process(img, scale, inp)
        assert got_x.is_cuda and got_x.dtype == torch.float32
        assert np.array_equal(got_x.cpu().numpy(), want_x.numpy()), (mode, h, w, scale)
        assert list(got) == list(want)
        for k in want:
            if k == "pre_dets":
                assert got[k] is want[k]
            else:
                g, r = np.asarray(got[k]), np.asarray(want[k])
                assert g.shape == r.shape and g.dtype == r.dtype and np.array_equal(g, r), (mode, h, w, scale, k)


def _calibrated(tracking=False, seed=21, frame=None):
    """A seeded dla_34 detector whose heat-map biases put a handful of distinct peaks on `frame` at scales 0.75 and 1
    (setup only, as in bench.py), or on synthetic 512 x 512 frames."""
    opt = cpb.default_opt("dla_34", tracking_task=tracking)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed, offset_std=0.3, head_gain=1.0))
    det = cpb.ObjectPoseDetector(opt, model=m)
    if frame is not None:
        x = torch.cat([det.pre_process(frame, sc, {})[0] for sc in (0.75, 1.0)]).cuda()
    else:
        x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(2, 512, 512, seed=500))).cuda()
    with torch.no_grad():
        if tracking:
            z1, z8 = torch.zeros((2, 1, 512, 512), device="cuda"), torch.zeros((2, 8, 512, 512), device="cuda")
            synth.calibrate_head_bias(det.model, det.model(x, x, z1, z8)[-1], target=6)
        else:
            synth.calibrate_head_bias(det.model, det.model(x)[-1], target=6)
    return det, opt


def _host_run(det):
    """det.run() with the host pre_process (pre_process -> upload -> process), as before the device path."""
    det._device_frame = lambda image: None
    return det


def _same_bits(a, b):
    """The same values bit for bit (NaN fields included)."""
    if isinstance(b, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _assert_same_results(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert sorted(a) == sorted(b)
        for k in b:
            assert _same_bits(a[k], b[k]), k


def _assert_same_run(got, want):
    _assert_same_results(got["results"], want["results"])
    assert len(got["boxes"]) == len(want["boxes"])
    for a, b in zip(got["boxes"], want["boxes"]):
        for i in range(4):
            assert _same_bits(a[i], b[i])
    assert sorted(got["output"]) == sorted(want["output"])
    for k, v in want["output"].items():
        assert (v is None and got["output"][k] is None) or _same_bits(got["output"][k], v), k


@pytest.mark.parametrize("scales", [[1.0], [0.75], [0.75, 1.0]])
def test_run_results_are_those_of_the_host_chain(scales, cplib):
    img = synth.synthetic_frames(1, 600, 800, seed=3)[0]
    det, opt = _calibrated(frame=img)
    opt.test_scales = det.scales = scales
    opt.nms = False
    got = det.run(img, meta_inp={"camera_matrix": CAM})
    got_last = det._last
    want = _host_run(det).run(img, meta_inp={"camera_matrix": CAM})
    assert len(want["results"]) > 0
    _assert_same_run(got, want)
    assert _same_bits(got_last[0], det._last[0]) and _same_bits(got_last[1], det._last[1])
    assert got["pre"] > 0


def test_run_tracking_sequence_is_that_of_the_host_chain(cplib):
    """Five frames of CenterPoseTrack seeded from pre_dets on frame 0 (opt.gt_pre_hm_hmhp_first): the device and host
    pre-process give the same tracks, bit for bit."""
    from oracle import make_golden_tracker as mg
    dets = []
    for _ in range(2):
        det, opt = _calibrated(tracking=True, seed=31)
        opt.gt_pre_hm_hmhp_first = True               # seeded, with ground-truth heat maps, on frame 0 only
        dets.append(det)
    dev_det, host_det = dets[0], _host_run(dets[1])
    _, seq = mg.make_sequence()
    frames = synth.synthetic_frames(5, 480, 640, seed=77)
    pre = mgt.gt_list(seq[0], width=640, height=480)
    n_tracks = 0
    for f in range(5):
        meta = {"camera_matrix": CAM, "id": f, "pre_dets": pre}
        got = dev_det.run(frames[f], meta_inp=meta)
        want = host_det.run(frames[f], meta_inp=meta)
        _assert_same_run(got, want)
        assert torch.equal(dev_det.pre_images, host_det.pre_images)
        n_tracks += len(got["results"])
    assert n_tracks > 0

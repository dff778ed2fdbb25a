"""The meta row and the pre-process in all three input modes (fix_res, keep_res, fix_short), without a GPU.

In the keep_res and fix_short modes pre_process returns s as the (w, h) pair, as the reference does; the affine uses
only its width (image.py:44-45), and so must the meta row the decode and the tracker read.  `make_meta` takes a 1-D s
as one scale per image, so a (w, h) pair handed to it unreduced used to fail to broadcast at batch 1 and was read as
s = w for image 0 and s = h for image 1 at batch 2."""
import types

import numpy as np
import pytest

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import ObjectPoseDetector
from oracle import ref_shims

CAM = np.array([[600.0, 0, 300.5], [0, 610.0, 400.25], [0, 0, 1]])
# (h, w) frames: the four geometries of tests/test_gpu_plan_geometry.py and two Objectron-like ones
FRAMES = [(800, 600), (1920, 1440), (1080, 1920), (720, 1280), (480, 640), (375, 500)]
MODES = {"fix_res": dict(fix_res=True, fix_short=-1), "keep_res": dict(fix_res=False, fix_short=-1),
         "fix_short": dict(fix_res=True, fix_short=512)}


def _detector(mode):
    """An ObjectPoseDetector that only pre-processes (no model, no device)."""
    opt = cpb.default_opt("dla_34")
    for k, v in MODES[mode].items():
        setattr(opt, k, v)
    det = ObjectPoseDetector.__new__(ObjectPoseDetector)
    det.opt = opt
    det.mean = np.array(opt.mean, dtype=np.float32).reshape(1, 1, 3)
    det.std = np.array(opt.std, dtype=np.float32).reshape(1, 1, 3)
    return det


def test_make_meta_scale_forms():
    c = np.array([300., 400.], np.float32)
    one = cpb.make_meta(1, c, 608.0, 600, 800, CAM).numpy()
    assert one.shape == (1, L.CP_META_DOUBLES)
    assert list(one[0, :5]) == [300., 400., 608., 600., 800.]
    assert np.array_equal(one[0, 5:14], CAM.reshape(9))
    two = cpb.make_meta(2, c, 608.0, 600, 800, CAM).numpy()
    assert np.array_equal(two[:, 2], [608., 608.])
    per = cpb.make_meta(2, np.stack([c, c + 1]), np.array([608., 512.]), 600, 800, CAM).numpy()
    assert np.array_equal(per[:, 2], [608., 512.]) and np.array_equal(per[1, :2], [301., 401.])
    pairs = cpb.make_meta(2, c, np.array([[608., 832.], [512., 704.]]), 600, 800, CAM).numpy()
    assert np.array_equal(pairs[:, 2], [608., 512.])
    # a 1-D s of the wrong length is neither broadcast nor reinterpreted
    with pytest.raises(ValueError):
        cpb.make_meta(1, c, np.array([608., 832.]), 600, 800, CAM)
    with pytest.raises(ValueError):
        cpb.make_meta(3, c, np.array([608., 832.]), 600, 800, CAM)
    with pytest.raises(ValueError):
        cpb.make_meta(1, c, np.array([608., 832., 1.]), 600, 800, CAM)


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("mode", list(MODES))
def test_meta_tensor_of_pre_process_takes_the_width(mode, batch):
    det = _detector(mode)
    img = synth.synthetic_frames(1, 800, 600, seed=5)[0]
    _, meta = det.pre_process(img, 1.0, {"camera_matrix": CAM})
    if mode == "fix_res":
        assert meta["s"] == 800.0
    else:
        assert isinstance(meta["s"], np.ndarray) and meta["s"].shape == (2,)
    m = det._meta_tensor(meta, batch).numpy()
    want_s = {"fix_res": 800.0, "keep_res": 608.0, "fix_short": 600.0}[mode]
    assert m.shape == (batch, L.CP_META_DOUBLES)
    for b in range(batch):
        assert m[b, 2] == want_s, (mode, m[b, 2])
        assert np.array_equal(m[b, 0:2], meta["c"]) and m[b, 3] == 600 and m[b, 4] == 800
        assert np.array_equal(m[b, 5:14], CAM.reshape(9))
    # the same width the input affine was built from
    want_trans = cpb.detector.affine_from_center_scale(meta["c"], want_s, meta["inp_width"], meta["inp_height"])
    assert np.array_equal(meta["trans_input"], want_trans)


def test_pre_process_geometry():
    """The network input sizes the GPU geometry tests are built on."""
    want = {("keep_res", 800, 600): (832, 608), ("fix_short", 1920, 1440): (704, 512),
            ("fix_short", 1080, 1920): (512, 960), ("keep_res", 720, 1280): (736, 1312),
            ("fix_res", 720, 1280): (512, 512)}
    for (mode, h, w), (ih, iw) in want.items():
        x, meta = _detector(mode).pre_process(synth.synthetic_frames(1, h, w, seed=1)[0], 1.0)
        assert tuple(x.shape) == (1, 3, ih, iw) and (meta["inp_height"], meta["inp_width"]) == (ih, iw), (mode, h, w)
        assert (meta["out_height"], meta["out_width"]) == (ih // 4, iw // 4)


@pytest.mark.skipif(not ref_shims.reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("mode", list(MODES))
def test_pre_process_matches_reference(mode):
    """ObjectPoseDetector.pre_process == the unmodified BaseDetector.pre_process (base_detector.py:91-148): the image
    bit for bit and every meta entry, in each mode, frame size and at a test scale below 1."""
    extra = {"fix_res": [], "keep_res": ["--keep_res"], "fix_short": ["--fix_short", "512"]}[mode]
    ref_opt = ref_shims.make_opt("dla_34", extra_args=extra)
    from lib.detectors.base_detector import BaseDetector
    det = _detector(mode)
    assert (ref_opt.fix_res, ref_opt.fix_short, ref_opt.pad, ref_opt.down_ratio) == \
        (det.opt.fix_res, det.opt.fix_short, det.opt.pad, det.opt.down_ratio)
    assert (ref_opt.input_h, ref_opt.input_w) == (det.opt.input_h, det.opt.input_w)
    stub = types.SimpleNamespace(opt=ref_opt, mean=np.array(ref_opt.mean, np.float32).reshape(1, 1, 3),
                                 std=np.array(ref_opt.std, np.float32).reshape(1, 1, 3))
    for i, (h, w) in enumerate(FRAMES):
        img = synth.synthetic_frames(1, h, w, seed=30 + i)[0]
        for scale in ((1.0, 0.75) if i < 2 else (1.0,)):
            inp = {"camera_matrix": CAM, "id": 3}
            want_x, want = BaseDetector.pre_process(stub, img, scale, inp)
            got_x, got = det.pre_process(img, scale, inp)
            assert got_x.dtype == want_x.dtype and np.array_equal(got_x.numpy(), want_x.numpy()), (mode, h, w, scale)
            assert sorted(got) == sorted(want)
            for k in want:
                g, r = np.asarray(got[k]), np.asarray(want[k])
                assert g.shape == r.shape and g.dtype == r.dtype and np.array_equal(g, r), (mode, h, w, scale, k)

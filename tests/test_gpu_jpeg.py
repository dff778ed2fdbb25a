"""JPEG decoding on the device: cp_jpeg_decode on one mixed batch equals cv2.imdecode bit for bit at the default and at
small subsequence lengths; a corrupt stream sets only its frame's error word; run(path) and run(bytes) give what
run(cv2.imread(path)) gives, in every pre-process mode and at two test scales, over a tracking sequence and in the demo
flow; and run_batch(list, pixel_format="jpeg") equals run_batch on the cv2-decoded frames, for detection, slot
tracking, per-frame format lists, a distorted camera and several categories."""
import json
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib
from centerpose_b200 import synth
from centerpose_b200.engine import jpeg_decode, jpeg_parse
from tests import jpeg_craft as jc
from tests.test_gpu_run_preprocess import CAM, _assert_same_run, _calibrated
from tests.test_meta_geometry import MODES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frame(h, w, seed):
    import cv2
    base = cv2.imread(os.path.join(ROOT, "tests", "data", "frame_%d.png" % (seed % 2)))
    img = cv2.resize(base, (w, h), interpolation=cv2.INTER_LINEAR).astype(np.int16)
    img += np.random.default_rng(seed).integers(-6, 7, img.shape).astype(np.int16)
    return np.clip(img, 0, 255).astype(np.uint8)


def _variants():
    out = []
    sizes = [(1, 1), (5, 3), (17, 33), (37, 53), (480, 640), (640, 480)]
    for i, s in enumerate(jc.SAMPLINGS):
        for j, (h, w) in enumerate(sizes):
            q = (10, 50, 75, 95, 100)[(i + j) % 5]
            out.append(jc.encode(_frame(h, w, i * 7 + j), s, q, restart=(0, 1, 4)[(i + j) % 3]))
    img = _frame(233, 311, 3)
    out.append(jc.strip(jc.encode(img, "420", 80), 0xC4))                     # MJPEG: no DHT
    out.append(jc.encode(img, "422", 90, optimize=True))
    for o in (3, 6, 8):
        out.append(jc.with_orientation(jc.encode(img, "420", 85, restart=2), o, big_endian=o == 6))
    out.append(jc.encode(np.full((256, 256), 128, np.uint8), "gray", 75))     # a periodic symbol stream
    return out


def _decode(files, words=0):
    hs = [jpeg_parse(np.frombuffer(f, np.uint8)) for f in files]
    assert all(h.status == 0 for h in hs)
    offs = np.cumsum([0] + [len(f) for f in files[:-1]])
    dev = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).cuda()
    sizes = [h.out_h * h.out_w * 3 for h in hs]
    oo = np.cumsum([0] + sizes[:-1])
    out = torch.full((sum(sizes),), 77, dtype=torch.uint8, device="cuda")
    err = jpeg_decode(hs, dev, offs, out, oo, subseq_words=words).cpu().numpy()
    host = out.cpu().numpy()
    return [host[o:o + s].reshape(h.out_h, h.out_w, 3) for o, s, h in zip(oo, sizes, hs)], err


@pytest.mark.parametrize("words", [0, 1, 2, 5])
def test_decode_batch_is_cv2(words, cplib):
    files = _variants()
    got, err = _decode(files, words)
    assert not err.any()
    for k, (f, g) in enumerate(zip(files, got)):
        assert np.array_equal(g, jc.decode(f)), k
    if words == 1:
        assert cplib.cp_jpeg_last_rounds() >= 2


def _invalid_code(data):
    """32 one bits (four stuffed 0xFF bytes) in the middle of the scan: no Huffman code is all ones."""
    a, b = jc.scan_range(data)
    m = (a + b) // 2
    while data[m - 1] == 0xFF:
        m += 1
    return data[:m] + b"\xff\x00" * 4 + data[m:]


def _wrong_rst(data):
    i = data.index(b"\xff\xd1", jc.scan_range(data)[0])
    return data[:i + 1] + b"\xd3" + data[i + 2:]


def _truncated(data):
    a, b = jc.scan_range(data)
    cut = (a + b) // 2
    if data[cut - 1] == 0xFF:
        cut -= 1
    return data[:cut] + b"\xff\xd9"


def test_corrupt_frames_set_only_their_error_word(cplib):
    img = _frame(120, 160, 5)
    good = [jc.encode(img, "420", 90), jc.encode(img, "444", 70, restart=3), jc.encode(img, "gray", 60)]
    bad = {1: (_truncated(jc.encode(img, "420", 90)), _lib.JPEG_ERR_SHORT),
           3: (_invalid_code(jc.encode(img, "422", 90)), _lib.JPEG_ERR_CODE),
           5: (_wrong_rst(jc.encode(img, "420", 90, restart=2)), _lib.JPEG_ERR_RESTART)}
    files = [good[0], bad[1][0], good[1], bad[3][0], good[2], bad[5][0]]
    for words in (0, 1):
        got, err = _decode(files, words)
        for k in range(len(files)):
            if k in bad:
                assert err[k] & bad[k][1], (k, err[k])
            else:
                assert err[k] == 0 and np.array_equal(got[k], jc.decode(files[k])), k


def test_decode_refuses_bad_arguments(cplib):
    import ctypes
    data = jc.encode(_frame(16, 16, 1), "420", 90)
    hs = (_lib.CpJpegHeader * 1)(jpeg_parse(np.frombuffer(data, np.uint8)))
    bad = _lib.CpJpegHeader()
    bad.status = 3
    assert cplib.cp_jpeg_workspace_bytes((_lib.CpJpegHeader * 1)(bad), 1) == 0
    ws = cplib.cp_jpeg_workspace_bytes(hs, 1)            # the need at one word per subsequence, the most
    assert ws > 0
    src = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).cuda()
    out = torch.zeros(16 * 16 * 3, dtype=torch.uint8, device="cuda")
    work = torch.zeros(ws, dtype=torch.uint8, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    offs = (ctypes.c_int64 * 1)(0)
    args = (src.data_ptr(), offs, out.data_ptr(), offs, work.data_ptr())
    assert cplib.cp_jpeg_decode(hs, 1, *args, ws - 1, err.data_ptr(), 1, None) == -1
    assert cplib.cp_jpeg_decode(hs, 1, *args, ws, err.data_ptr(), -1, None) == -1
    assert cplib.cp_jpeg_decode(hs, 1, *args, ws, None, 0, None) == -1
    assert cplib.cp_jpeg_decode((_lib.CpJpegHeader * 1)(bad), 1, *args, ws, err.data_ptr(), 0, None) == -1
    assert int(out.sum()) == 0


# ---------------------------------------------------------------- run()
def _no_host_decode(monkeypatch):
    """cv2's decoders raise from here on: a run() that still returns went through the device decode."""
    import cv2

    def refuse(*a, **k):
        raise AssertionError("the host decoder was called")
    monkeypatch.setattr(cv2, "imread", refuse)
    monkeypatch.setattr(cv2, "imdecode", refuse)


def _write_jpegs(tmp_path, frames, **kw):
    paths = []
    for i, f in enumerate(frames):
        p = str(tmp_path / ("f%d.jpg" % i))
        open(p, "wb").write(jc.encode(f, **kw))
        paths.append(p)
    return paths


@pytest.mark.parametrize("scales", [[1.0], [0.75]])
@pytest.mark.parametrize("mode", list(MODES))
def test_run_path_and_bytes_are_run_of_imread(mode, scales, cplib, tmp_path, monkeypatch):
    import cv2
    img = synth.synthetic_frames(1, 600, 800, seed=3)[0]
    path = _write_jpegs(tmp_path, [img], sampling="420", quality=92)[0]
    det, opt = _calibrated(frame=cv2.imread(path))
    for k, v in MODES[mode].items():
        setattr(opt, k, v)
    opt.test_scales = det.scales = scales
    opt.nms = False
    want = det.run(cv2.imread(path), meta_inp={"camera_matrix": CAM})
    if mode == "fix_res":
        assert len(want["results"]) > 0
    srcs = (path, open(path, "rb").read(), np.fromfile(path, np.uint8))
    _no_host_decode(monkeypatch)
    for src in srcs:
        _assert_same_run(det.run(src, meta_inp={"camera_matrix": CAM}), want)
        _assert_same_run(det.run(src, filename="frame_0001", meta_inp={"camera_matrix": CAM}), want)


def test_run_tracking_sequence_from_jpeg_files(cplib, tmp_path, monkeypatch):
    import cv2
    from oracle import make_golden_tracker as mg
    from oracle import make_golden_tracker_gt as mgt
    dets = []
    for _ in range(2):
        det, opt = _calibrated(tracking=True, seed=31)
        opt.gt_pre_hm_hmhp_first = True
        dets.append(det)
    _, seq = mg.make_sequence()
    paths = _write_jpegs(tmp_path, synth.synthetic_frames(5, 480, 640, seed=77), sampling="422", quality=90)
    pre = mgt.gt_list(seq[0], width=640, height=480)
    imgs = [cv2.imread(p) for p in paths]
    _no_host_decode(monkeypatch)
    n = 0
    for f, p in enumerate(paths):
        meta = {"camera_matrix": CAM, "id": f, "pre_dets": pre}
        got = dets[0].run(p, meta_inp=meta)
        want = dets[1].run(imgs[f], meta_inp=meta)
        _assert_same_run(got, want)
        n += len(got["results"])
    assert n > 0


def test_run_host_fallbacks(cplib, tmp_path):
    """A progressive JPEG, a corrupt JPEG and a PNG take cv2.imread: the results are those of run(cv2.imread(path))."""
    import cv2
    img = synth.synthetic_frames(1, 480, 640, seed=8)[0]
    det, _ = _calibrated(frame=img)
    files = {"prog.jpg": jc.encode(img, "420", 90, progressive=True),
             "bad.jpg": _invalid_code(jc.encode(img, "420", 90))}
    for name, data in files.items():
        open(str(tmp_path / name), "wb").write(data)
    cv2.imwrite(str(tmp_path / "f.png"), img)
    assert jpeg_parse(np.frombuffer(files["prog.jpg"], np.uint8)).status == 3
    for name in ("prog.jpg", "bad.jpg", "f.png"):
        p = str(tmp_path / name)
        _assert_same_run(det.run(p, meta_inp={"camera_matrix": CAM}), det.run(cv2.imread(p),
                                                                               meta_inp={"camera_matrix": CAM}))


def test_run_bytes_host_fallbacks_decode_the_bytes(cplib, tmp_path):
    """Encoded input that the device does not decode (progressive, corrupt, PNG) is decoded by cv2.imdecode of those
    bytes, also when `filename` names something else: a label, or a file holding another image."""
    import cv2
    img = synth.synthetic_frames(1, 480, 640, seed=8)[0]
    other = synth.synthetic_frames(1, 480, 640, seed=9)[0]
    det, _ = _calibrated(frame=img)
    decoy = str(tmp_path / "decoy.jpg")
    open(decoy, "wb").write(jc.encode(other, "420", 90))
    data = [jc.encode(img, "420", 90, progressive=True), _invalid_code(jc.encode(img, "420", 90)),
            cv2.imencode(".png", img)[1].tobytes()]
    for d in data:
        want = det.run(cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_COLOR), filename="x",
                       meta_inp={"camera_matrix": CAM})
        for src in (d, np.frombuffer(d, np.uint8)):
            for name in ("nonexistent", decoy):
                _assert_same_run(det.run(src, filename=name, meta_inp={"camera_matrix": CAM}), want)


def test_demo_flow_on_jpeg_files(cplib, tmp_path, monkeypatch):
    """demo.py's flow (run(path) with --debug 4) on JPEG copies of tests/data writes the files the same flow writes
    with the host decode."""
    import cv2
    cam = np.array([[663.0287679036459, 0, 300.2775065104167], [0, 663.0287679036459, 395.00066121419275], [0, 0, 1]])
    src = tmp_path / "jpg"
    src.mkdir()
    for f in sorted(os.listdir(os.path.join(ROOT, "tests", "data"))):
        if f.endswith(".png"):
            img = cv2.imread(os.path.join(ROOT, "tests", "data", f))
            open(str(src / (f[:-4] + ".jpg")), "wb").write(jc.encode(img, "420", 90))
    outs = []
    for host in (False, True):
        opt = cpb.default_opt("dla_34", debug=4)
        m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
        m.load_state_dict(synth.seeded_state_dict(m, seed=9, offset_std=0.3, head_gain=6.0))
        ck = str(tmp_path / "chair_seeded.pth")
        cpb.save_model(ck, 1, m)
        opt.load_model = ck
        opt.demo = str(src)
        opt.demo_save = str(tmp_path / ("save_host" if host else "save_dev"))
        det = cpb.detector_factory["object_pose"](opt)
        det.pause = False
        if host:
            det._device_jpeg = lambda data, header: None
        with monkeypatch.context() as mp:
            if not host:
                _no_host_decode(mp)
            for f in sorted(os.listdir(opt.demo)):
                det.run(os.path.join(opt.demo, f), meta_inp={"camera_matrix": cam})
        outs.append(opt.demo_save)
    files = sorted(os.path.relpath(os.path.join(d, f), outs[0]) for d, _, fs in os.walk(outs[0]) for f in fs)
    assert files and files == sorted(os.path.relpath(os.path.join(d, f), outs[1]) for d, _, fs in os.walk(outs[1])
                                     for f in fs)
    for f in files:
        a, b = open(os.path.join(outs[0], f), "rb").read(), open(os.path.join(outs[1], f), "rb").read()
        if f.endswith(".json"):
            assert json.loads(a) == json.loads(b), f
        else:
            assert a == b, f


# ---------------------------------------------------------------- run_batch(list, pixel_format="jpeg")
SIZES = [(601, 803), (481, 640), (512, 512), (720, 1280)]


def _cam(h, w):
    return np.array([[600., 0, w / 2.], [0, 600., h / 2.], [0, 0, 1]])


def _files(seed, kinds=("420", "422", "444", "gray")):
    return [jc.encode(_frame(h, w, seed + i), kinds[i % len(kinds)], 90, restart=i % 2)
            for i, (h, w) in enumerate(SIZES)]


def _det():
    from tests.test_gpu_yuv_input import _detector
    return _detector("dla_34", [jc.decode(f) for f in _files(40)])[0]


def test_run_batch_jpeg_detection(cplib):
    det = _det()
    files = _files(40)
    cams = np.stack([_cam(h, w) for h, w in SIZES])
    wp, wn = det.run_batch([jc.decode(f) for f in files], cams)
    assert wn.sum() > 0
    forms = [files, [np.frombuffer(f, np.uint8) for f in files],
             [torch.from_numpy(np.frombuffer(f, np.uint8).copy()).pin_memory() for f in files]]
    for fr in forms:
        gp, gn = det.run_batch(fr, cams, pixel_format="jpeg")
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)
    # a per-frame list mixing "jpeg" with "nv12" and "bgr", and a distorted camera
    from tests.test_gpu_undistort import PLUMB
    from tests.test_gpu_pixel_formats import encode as colour_encode
    from tests.test_gpu_pixel_formats import to_bgr
    nv12 = colour_encode(_frame(480, 640, 9), "nv12", 0)
    mix = [files[0], nv12, jc.decode(files[2]), files[3]]
    fmts = ["jpeg", "nv12", "bgr", "jpeg"]
    cams4 = np.stack([_cam(601, 803), _cam(480, 640), _cam(512, 512), _cam(720, 1280)])
    conv = [jc.decode(files[0]), to_bgr(nv12, "nv12"), jc.decode(files[2]), jc.decode(files[3])]
    for dists in (None, [PLUMB, None, None, PLUMB]):
        wp, wn = det.run_batch(conv, cams4, distortion=dists)
        gp, gn = det.run_batch(mix, cams4, pixel_format=fmts, distortion=dists)
        assert np.array_equal(gn, wn) and np.array_equal(gp, wp)


def test_run_batch_jpeg_refusals(cplib):
    det = _det()
    files = _files(40)
    cams = np.stack([_cam(h, w) for h, w in SIZES])
    prog = jc.encode(_frame(64, 64, 1), "420", 90, progressive=True)
    with pytest.raises(ValueError, match="frame 2 is a JPEG the device decoder does not take: progressive"):
        det.run_batch(files[:2] + [prog] + files[3:], cams, pixel_format="jpeg")
    with pytest.raises(ValueError, match="frame 1 is a corrupt JPEG"):
        det.run_batch([files[0], _invalid_code(files[1])] + files[2:], cams, pixel_format="jpeg")


def test_run_batch_jpeg_slot_tracking(cplib):
    from tests.test_gpu_track_graph import _detector as _trk_detector
    det = _trk_detector()
    cams = np.stack([_cam(h, w) for h, w in SIZES])
    schedule = [[None, "new", "new", None], [True, True, None, "new"], ["new", True, True, True],
                [True, None, True, True]]
    runs = []
    for jpeg in (False, True):
        det.reset_tracking()
        out = []
        for k, row in enumerate(schedule):
            files = _files(100 + k)
            fs = [None if e is None else (f if jpeg else jc.decode(f)) for e, f in zip(row, files)]
            out.append(det.run_batch(fs, cams, track=True, new_video=[e == "new" for e in row],
                                     **({"pixel_format": "jpeg"} if jpeg else {})))
        runs.append(out)
    assert sum(int(n.sum()) for _, n in runs[1]) > 0
    for (a, na), (b, nb) in zip(*runs):
        assert np.array_equal(na, nb) and np.array_equal(a, b)


def test_multi_category_detector_jpeg(cplib, tmp_path):
    from tests.test_gpu_yuv_input import _category_checkpoints
    files = _files(60)
    cams = np.stack([_cam(h, w) for h, w in SIZES])
    det = cpb.MultiCategoryDetector(*_category_checkpoints(tmp_path, False))
    wp, wn = det.run_batch([jc.decode(f) for f in files], cams)
    gp, gn = det.run_batch(files, cams, pixel_format="jpeg")
    assert np.array_equal(gn, wn) and np.array_equal(gp, wp)

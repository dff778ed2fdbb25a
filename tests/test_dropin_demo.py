"""The demo flow of the reference's `src/demo.py` (demo.py:22-87) on this package: a detector built from a checkpoint
path, `run()` on image files with a camera matrix, and the `--debug 4` JSON files it writes (object_pose.py:357-414)."""
import json
import os

import numpy as np
import pytest

import centerpose_b200 as cpb
from centerpose_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJECT_KEYS = {"class", "ct", "bbox", "confidence", "kps_displacement_mean", "kps_heatmap_mean", "kps_heatmap_std",
               "kps_heatmap_height", "obj_scale", "location", "quaternion_xyzw", "kps_pnp", "kps_3d_cam"}


@pytest.mark.gpu
def test_demo_flow_on_gpu(cplib, tmp_path):
    """The demo flow (demo.py:22-87: Detector(opt) from a checkpoint path -> run(image path, meta_inp) per file ->
    --debug 4 JSON) with the real engine, on the committed sample frames."""
    opt = cpb.default_opt("dla_34", debug=4)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=9, offset_std=0.3, head_gain=6.0))
    ck = str(tmp_path / "chair_seeded.pth")
    cpb.save_model(ck, 1, m)
    opt.load_model = ck
    opt.demo = os.path.join(ROOT, "tests", "data")
    opt.demo_save = str(tmp_path / "save")
    cam = np.array([[663.0287679036459, 0, 300.2775065104167], [0, 663.0287679036459, 395.00066121419275], [0, 0, 1]])
    det = cpb.detector_factory["object_pose"](opt)
    det.pause = False
    names = sorted(f for f in os.listdir(opt.demo) if f.endswith(".png"))
    for f in names:
        ret = det.run(os.path.join(opt.demo, f), meta_inp={"camera_matrix": cam})
        assert set(ret) == {"results", "boxes", "output", "tot", "load", "pre", "net", "dec", "post", "merge", "pnp", "track"}
        j = json.load(open(os.path.join(opt.demo_save, "data", os.path.splitext(f)[0] + ".json")))
        assert set(j) == {"camera_data", "objects"} and len(j["objects"]) == len(ret["boxes"])
        for o in j["objects"]:
            assert set(o) == OBJECT_KEYS

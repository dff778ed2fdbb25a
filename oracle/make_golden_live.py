"""TEST INFRASTRUCTURE ONLY -- stores what the tests that compare with the UNMODIFIED reference compared against,
so that they run without the reference tree:

    python -m oracle.make_golden_live          # needs the reference tree (oracle/ref_shims.py)

Fixtures
  live_decode_scenes.npz    reference decode (candidates scoring above 0.05) + post-process + soft-NMS + PnP of three
                            planted scenes (one of them with the tracking heads)
  live_gpfit.npz            the reference's gpfit `moments` / `fitgaussian` on seeded heat-map windows
  live_model_api.json       the reference's heads and default options per configuration
It also checks that two committed fixtures are what the reference computes from its own default options: the head
logits of net_dla34_b2_96x128.npz and the state-dict keys / shapes of state_dict_keys.json.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shims          # noqa: E402
from centerpose_b200 import synth     # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

# (tracking, rep_mode, objects, keypoint disagreement in px, seed) of the planted decode scenes
DECODE_SCENES = ((False, 1, 5, 2.0, 77), (True, 1, 2, 0.5, 78), (False, 3, 3, 1.0, 79))
MODEL_CONFIGS = (("dla_34", False), ("dlav1_34", False), ("dla_34", True))
STATE_DICT_KEYS = {("dla_34", False): "dla_34_plain", ("dlav1_34", False): "dlav1_34_plain", ("dla_34", True): "dla_34_track"}
OPT_CONFIGS = (("dla_34", False, 1), ("dla_34", True, 1), ("dlav1_34", False, 0))
OPT_FIELDS = ("K", "rep_mode", "vis_thresh", "nms", "use_pnp", "head_conv", "down_ratio", "mean", "std", "c", "input_h",
              "input_w", "num_classes", "test_scales", "fix_res", "hm_hp", "reg_offset", "reg_hp_offset", "tracking_task",
              "hps_uncertainty", "obj_scale_uncertainty", "balance_coefficient")


def gpfit_windows(n=30, seed=3):
    rng = np.random.default_rng(seed)
    g = np.exp(-((np.arange(11)[:, None] - 5.3) ** 2 + (np.arange(11)[None] - 4.6) ** 2) / 6)
    return [rng.random((11, 11)) * g for _ in range(n)]


def jsonable(v):
    """Option values as JSON stores them (tuples and arrays become lists)."""
    if isinstance(v, np.ndarray):
        return v.tolist()
    if isinstance(v, (tuple, list)):
        return [jsonable(x) for x in v]
    if isinstance(v, dict):
        return {k: jsonable(x) for k, x in v.items()}
    if isinstance(v, np.generic):
        return v.item()
    return v


def check_net():
    import centerpose_b200 as cpb
    from lib.models.model import create_model as ref_create
    from tests.util import golden, net_case_inputs
    g = golden("net_dla34_b2_96x128")
    opt = cpb.default_opt("dla_34")
    sd = synth.seeded_state_dict(cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt), seed=int(g["wseed"]),
                                 offset_std=float(g["offset_std"]))
    ropt = ref_shims.make_opt("dla_34")
    ref = ref_create(ropt.arch, ropt.heads, ropt.head_conv, ropt).eval()
    ref.load_state_dict(sd, strict=True)
    x, _ = net_case_inputs(g)
    with torch.no_grad():
        out = ref(torch.from_numpy(x))[-1]
    for h, v in out.items():
        if not np.array_equal(v.numpy(), g["head_" + h]):
            raise SystemExit("net_dla34_b2_96x128.npz differs from the reference model built from its own options: " + h)


def make_decode():
    from oracle.make_golden import reference_pipeline
    arrays = {}
    for i, (trk, rep, nobj, dis, seed) in enumerate(DECODE_SCENES):
        opt = ref_shims.make_opt("dla_34", tracking_task=trk, rep_mode=rep)
        heads = synth.TRACKING_HEADS if trk else synth.DEFAULT_HEADS
        h, truth = synth.planted_heads(n_obj=nobj, seed=seed, heads=heads, disagree_px=dis)
        dets, recs = reference_pipeline(h, opt, truth["cam"], 512, 512, np.array([256., 256.], np.float32), 512.0)
        # candidates come out sorted by score; only the ones above 0.05 are compared (the tied tail is order-undefined)
        n = int((dets["scores"][0, :, 0] > 0.05).sum())
        assert (dets["scores"][0, :n, 0] > 0.05).all()
        for k, v in dets.items():
            arrays["scene%d_dets_%s" % (i, k)] = v[0][:n]
        arrays["scene%d_records" % i] = recs
    np.savez_compressed(os.path.join(GOLD, "live_decode_scenes.npz"), **arrays)


def make_gpfit():
    from lib.utils.gpfit import moments, fitgaussian
    w = gpfit_windows()
    np.savez_compressed(os.path.join(GOLD, "live_gpfit.npz"), moments=np.array([moments(a) for a in w], np.float64),
                        fitgaussian=np.array([fitgaussian(a) for a in w], np.float64))


def make_model_api():
    from lib.models.model import create_model as ref_create
    out = {"heads": {}, "opts": {}}
    keys = json.load(open(os.path.join(GOLD, "state_dict_keys.json")))
    for arch, trk in MODEL_CONFIGS:
        ropt = ref_shims.make_opt(arch, tracking_task=trk)
        r = ref_create(ropt.arch, ropt.heads, ropt.head_conv, ropt)
        out["heads"]["%s_%d" % (arch, trk)] = [[k, v] for k, v in ropt.heads.items()]
        if [[k, list(v.shape)] for k, v in r.state_dict().items()] != keys[STATE_DICT_KEYS[(arch, trk)]]:
            raise SystemExit("state_dict_keys.json differs from the reference model of %s tracking=%d" % (arch, trk))
    for arch, trk, rep in OPT_CONFIGS:
        r = ref_shims.make_opt(arch, tracking_task=trk, rep_mode=rep)
        out["opts"]["%s_%d_%d" % (arch, trk, rep)] = {f: jsonable(getattr(r, f)) for f in OPT_FIELDS}
    with open(os.path.join(GOLD, "live_model_api.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    if not ref_shims.reference_available():
        raise SystemExit("reference tree not present: these goldens can only be generated where it is")
    ref_shims.install()
    torch.set_num_threads(os.cpu_count() or 1)
    check_net()
    make_decode()
    make_gpfit()
    make_model_api()

"""`ObjectPoseDetector.run()` end to end in the keep_res and fix_short modes, whose network inputs are not 512 x 512
and whose pre_process returns s as the (w, h) pair: the records run() decodes vs the oracle chain net_ref (fp64, on the
device) -> decode_ref -> pnp_ref on the same pre-processed frame, with the meta the reference's pre_process gives."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import scale_width
from tests.test_gpu_bench_parity import E2E_BOUNDS, _match
from tests.util import oracle_records

pytestmark = pytest.mark.gpu

# (mode, frame h, frame w, opt overrides, network input h x w)
CASES = [("keep_res", 800, 600, dict(fix_res=False), (832, 608)),
         ("fix_short", 1920, 1440, dict(fix_short=512), (704, 512))]


def _detector(opt, sd, precision):
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.precision = precision
    if sd is None:
        sd = synth.seeded_state_dict(m, seed=0, offset_std=0.3)
    m.load_state_dict(sd)
    return cpb.ObjectPoseDetector(opt, model=m)


@pytest.mark.parametrize("mode,h,w,over,inp", CASES, ids=[c[0] for c in CASES])
def test_run_vs_oracle_chain(mode, h, w, over, inp, cplib):
    from oracle import decode_ref, net_ref
    opt = cpb.default_opt("dla_34")
    for k, v in over.items():
        setattr(opt, k, v)
    img = synth.synthetic_frames(1, h, w, seed=h + w)[0]
    cam = synth.default_camera(w, h)
    # setup: calibrated random weights (~4 centre peaks pass vis_thresh), as test_gpu_bench_parity._e2e_oracle
    det = _detector(opt, None, "fp32")
    x, meta = det.pre_process(img, 1.0, {"camera_matrix": cam})
    assert tuple(x.shape[2:]) == inp and isinstance(meta["s"], np.ndarray)
    with torch.no_grad():
        synth.calibrate_head_bias(det.model, det.model(x.cuda())[-1], target=4)
    sd = {k: v.detach().cpu().clone() for k, v in det.model.state_dict().items()}

    det = _detector(opt, sd, "tf32x3")
    ret = det.run(img, meta_inp={"camera_matrix": cam})
    poses, n_valid = det._last                       # the pose records run() unpacked (process() keeps them)
    got = poses[0, :n_valid[0]].astype(np.float64)
    assert len(ret["results"]) == got.shape[0]

    with torch.no_grad():
        sd64 = {k: v.double().cuda() if v.dtype.is_floating_point else v for k, v in sd.items()}
        heads = net_ref.forward(x.cuda().double(), sd64, opt.heads, "dla_34")
    prm = decode_ref.DecodeParams(rep_mode=opt.rep_mode, vis_thresh=opt.vis_thresh, category=opt.c)
    _, want = oracle_records({k: v[0].float().cpu().numpy() for k, v in heads.items()}, prm, cam, w, h, meta["c"],
                             scale_width(meta["s"]), L)

    bnd = E2E_BOUNDS["tf32x3"]
    margin = np.abs(want[:, L.P_SCORE] - opt.vis_thresh) > 2e-3 if want.shape[0] else np.zeros(0, bool)
    pairs = _match(got, want)
    n_want, n_pair, n_stable = int(margin.sum()), sum(1 for i, j in pairs if margin[j]), 0
    worst = dict(score=0.0, px=0.0, quat=0.0)
    for i, j in pairs:
        g, r = got[i], want[j]
        worst["score"] = max(worst["score"], abs(g[L.P_SCORE] - r[L.P_SCORE]))
        dk = np.abs(g[L.P_KPS:L.P_KPS + 16] - r[L.P_KPS:L.P_KPS + 16]).max()
        dh = np.abs(g[L.P_KPS_HM_MEAN:L.P_KPS_HM_MEAN + 16] - r[L.P_KPS_HM_MEAN:L.P_KPS_HM_MEAN + 16]).max()
        if max(dk, dh) > 2.0:              # a grouping gate flipped (regressed <-> heat-map peak): not a drift sample
            continue
        n_stable += 1
        dd = np.abs(g[L.P_KPS_DISP_MEAN:L.P_KPS_DISP_MEAN + 16] - r[L.P_KPS_DISP_MEAN:L.P_KPS_DISP_MEAN + 16]).max()
        worst["px"] = max(worst["px"], dk, dh, dd, np.abs(g[L.P_BBOX:L.P_BBOX + 4] - r[L.P_BBOX:L.P_BBOX + 4]).max())
        if int(g[L.P_STATUS]) in (L.PNP_OK, L.PNP_INVISIBLE) and int(r[L.P_STATUS]) in (L.PNP_OK, L.PNP_INVISIBLE):
            q1, q2 = r[L.P_QUAT:L.P_QUAT + 4], g[L.P_QUAT:L.P_QUAT + 4]
            worst["quat"] = max(worst["quat"], np.abs(q1 - (q2 if np.dot(q1, q2) >= 0 else -q2)).max())
    print("run() %s %dx%d -> %dx%d: oracle dets %d (away from the threshold), gpu dets %d, matched %d, same keypoint "
          "source %d; max drift: score %.2e, keypoints/boxes %.3e px, quaternion %.2e"
          % (mode, h, w, inp[0], inp[1], n_want, got.shape[0], n_pair, n_stable, worst["score"], worst["px"],
             worst["quat"]))
    assert n_want > 0
    assert n_pair == n_want, "a detection away from the score threshold is missing from run()"
    assert n_stable >= bnd["stable_frac"] * n_pair
    assert worst["score"] <= bnd["score"]
    assert worst["px"] <= bnd["px"]
    assert worst["quat"] <= bnd["quat"]

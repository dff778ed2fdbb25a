"""Decode / grouping / post-process / soft-NMS / PnP parity on the GPU: the
fused CUDA stage (through cp_decode_pnp) vs the reference's golden vectors, vs
the CPU oracle on fresh seeds, and size-independent properties at batch 32."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import dets_to_dict
from oracle import decode_ref
from tests.util import DETS_KEYS, compare_records, decode_case_geometry, decode_case_inputs, golden, oracle_records

pytestmark = pytest.mark.gpu

CASES = ["decode_rep1_3obj", "decode_rep1_10obj_noisy", "decode_rep0_3obj", "decode_rep4_2obj", "decode_rep4_5pts_epnp",
         "decode_track_rep1_3obj", "decode_rep1_3obj_modern_torch", "decode_cls3_rep1_6obj", "decode_scale075_rep1_3obj",
         "decode_scale125_rep0_nonms"]
C512 = np.array([256., 256.], np.float32)


def _run(hb, cam, rep_mode, tracking, category, c=C512, s=512.0, w=512, h=512, **over):
    B = hb["hm"].shape[0]
    prm = cpb.decode_params(None, rep_mode=rep_mode, tracking_task=tracking, c=category, **over)
    heads = {k: torch.from_numpy(v).cuda() for k, v in hb.items()}
    meta = cpb.make_meta(B, c, s, w, h, cam)
    dets, poses, n_valid = cpb.decode_pnp(heads, meta, prm, want_dets=True)
    torch.cuda.synchronize()
    return dets.cpu().numpy(), poses.cpu().numpy(), n_valid.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_matches_reference_golden(name, cplib):
    g = golden(name)
    hb, truths = decode_case_inputs(g)
    modern = bool(int(g["modern_bool"])) if "modern_bool" in g.files else False
    c, s, scales, nms = decode_case_geometry(g)
    dets, poses, n_valid = _run(hb, g["cam"], int(g["rep_mode"]), bool(int(g["tracking"])), str(g["category"]), c=c, s=s,
                                modern_bool_semantics=modern, num_classes=hb["hm"].shape[1], test_scales=scales, nms=nms)
    dd = dets_to_dict(dets)
    for b in range(int(g["batch"])):
        valid = g["dets%d_scores" % b][:, 0] > 0.05
        for k in DETS_KEYS:
            want = g["dets%d_%s" % (b, k)]
            assert np.abs(dd[k][b][valid] - want[valid]).max() <= (1e-3 if "std" in k or "unc" in k else 2e-5), (b, k)
        want = g["records%d" % b]
        assert n_valid[b] == want.shape[0], (b, n_valid[b], want.shape[0])
        got = poses[b, :n_valid[b]]
        assert (got[:, L.P_SRC_INDEX] == want[:, L.P_SRC_INDEX]).all()      # identical detection set and order
        compare_records(got, want, L)
        assert (poses[b, n_valid[b]:] == 0).all()


@pytest.mark.parametrize("rep,trk,nobj,dis,cat,seed", [(1, False, 6, 2.5, "chair", 301), (1, True, 4, 1.0, "cup", 302),
                                                       (3, False, 3, 1.0, "bike", 303), (0, False, 8, 3.0, "chair", 304)])
def test_matches_oracle_fresh_seeds(rep, trk, nobj, dis, cat, seed, cplib):
    heads = synth.TRACKING_HEADS if trk else synth.DEFAULT_HEADS
    B = 3
    hb, truths = synth.planted_batch(B, n_obj=nobj, seed=seed, heads=heads, disagree_px=dis)
    cam = truths[0]["cam"]
    dets, poses, n_valid = _run(hb, cam, rep, trk, cat)
    prm = decode_ref.DecodeParams(rep_mode=rep, use_moments=trk, vis_thresh=0.3, category=cat)
    for b in range(B):
        _, want = oracle_records({k: v[b] for k, v in hb.items()}, prm, cam, 512, 512, C512, 512.0, L)
        assert n_valid[b] == want.shape[0]
        got = poses[b, :n_valid[b]]
        assert (got[:, L.P_SRC_INDEX] == want[:, L.P_SRC_INDEX]).all()
        compare_records(got, want, L)


def test_non_square_image_affine(cplib):
    """600x800 Objectron frame (demo.py:143-144 intrinsics): c = (300, 400), s = 800."""
    hb, truths = synth.planted_batch(2, n_obj=3, seed=410, cam=synth.default_camera(512, 512))
    cam = np.array([[663.0287679036459, 0, 300.2775065104167], [0, 663.0287679036459, 395.00066121419275], [0, 0, 1]])
    c, s = np.array([300., 400.], np.float32), 800.0
    dets, poses, n_valid = _run(hb, cam, 1, False, "chair", c=c, s=s, w=600, h=800)
    prm = decode_ref.DecodeParams(rep_mode=1, vis_thresh=0.3, category="chair")
    for b in range(2):
        _, want = oracle_records({k: v[b] for k, v in hb.items()}, prm, cam, 600, 800, c, s, L)
        assert n_valid[b] == want.shape[0]
        compare_records(poses[b, :n_valid[b]], want, L)


@pytest.mark.parametrize("oh,ow,K,nobj", [(96, 128, 100, 3), (128, 128, 128, 5), (64, 64, 20, 2), (160, 96, 100, 3),
                                          (160, 160, 100, 3), (208, 152, 100, 4), (184, 328, 128, 5)])
def test_map_shapes_and_K(oh, ow, K, nobj, cplib):
    """Ragged shapes: non-square head maps (keep_res / fix_short inputs), K at CP_MAX_K and a small K, vs the oracle.
    160 x 160 is the largest map whose top-K runs in shared memory; the 208 x 152 (keep_res 832 x 608) and 184 x 328
    (keep_res 736 x 1312) maps keep the NMS-ed map in the workspace."""
    B = 2
    w, h = ow * 4, oh * 4
    hb, truths = synth.planted_batch(B, n_obj=nobj, seed=900 + K, out_h=oh, out_w=ow, disagree_px=0.5)
    cam = truths[0]["cam"]
    c, s = np.array([w / 2., h / 2.], np.float32), float(max(w, h))
    dets, poses, n_valid = _run(hb, cam, 1, False, "chair", c=c, s=s, w=w, h=h, K=K)
    assert poses.shape == (B, K, L.CP_POSE_RECORD)
    prm = decode_ref.DecodeParams(K=K, rep_mode=1, vis_thresh=0.3, category="chair")
    for b in range(B):
        _, want = oracle_records({k: v[b] for k, v in hb.items()}, prm, cam, w, h, c, s, L)
        assert n_valid[b] == want.shape[0] == len(truths[b]["R"])
        got = poses[b, :n_valid[b]]
        assert (got[:, L.P_SRC_INDEX] == want[:, L.P_SRC_INDEX]).all()
        compare_records(got, want, L)


def test_empty_scene_and_no_pnp(cplib):
    hb, _ = synth.planted_batch(2, n_obj=0, seed=500)
    dets, poses, n_valid = _run(hb, synth.default_camera(), 1, False, "chair")
    assert (n_valid == 0).all() and (poses == 0).all()
    hb, truths = synth.planted_batch(1, n_obj=2, seed=501)
    dets, poses, n_valid = _run(hb, truths[0]["cam"], 1, False, "chair", use_pnp=False)
    assert n_valid[0] == 2 and (poses[0, :2, L.P_STATUS] == L.PNP_NOT_RUN).all()


def test_topk_is_exact_and_sorted(cplib):
    """The top-K list must be the K largest NMS survivors, descending, ties by ascending index."""
    rng = np.random.default_rng(7)
    hb, _ = synth.planted_batch(2, n_obj=0, seed=600)
    hb["hm"] = rng.normal(-3, 1.5, size=hb["hm"].shape).astype(np.float32)       # dense random field
    dets, poses, n_valid = _run(hb, synth.default_camera(), 1, False, "chair")
    dd = dets_to_dict(dets)
    for b in range(2):
        sc = dd["scores"][b, :, 0]
        assert (np.diff(sc) <= 0).all()
        nms = decode_ref.nms3x3(decode_ref.sigmoid_f32(hb["hm"][b]))
        want, ind, _, _ = decode_ref.topk_channel(nms, 100)
        assert np.abs(sc - want[0]).max() <= 2e-6
        got_ind = dets[b, :, L.D_IND].astype(np.int64)
        same = sc == want[0]                       # identical where the two sigmoids round identically
        assert (got_ind[same] == ind[0][same]).mean() > 0.97


def test_batch32_properties(cplib):
    """BASELINE config 3 batch: every planted object is found, poses reproject onto the planted keypoints."""
    B, nobj = 32, 3
    hb, truths = synth.planted_batch(B, n_obj=nobj, seed=700)
    dets, poses, n_valid = _run(hb, truths[0]["cam"], 1, False, "chair", visible_thresh=0)
    for b in range(B):
        n_planted = len(truths[b]["R"])
        assert n_valid[b] == n_planted
        ok = poses[b, :n_valid[b], L.P_STATUS] == L.PNP_OK
        assert ok.all()
        # planted keypoints (output-map px * 4) are recovered by the PnP reprojection to < 0.05 px
        for i in range(n_valid[b]):
            proj = poses[b, i, L.P_PROJ_CUBOID:L.P_PROJ_CUBOID + 16].reshape(8, 2)
            d = [np.abs(proj - t * 4).max() for t in truths[b]["kps_map"]]
            assert min(d) < 0.05
    # the same frames processed alone give bit-identical records
    hb1 = {k: v[5:6] for k, v in hb.items()}
    _, p1, n1 = _run(hb1, truths[0]["cam"], 1, False, "chair", visible_thresh=0)
    assert n1[0] == n_valid[5] and np.array_equal(p1[0], poses[5])

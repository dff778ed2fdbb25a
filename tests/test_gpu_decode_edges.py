"""The CUDA decode's discrete decisions against the oracle on tied and boundary inputs (tests/decode_scenes.py):
exact top-K under ties and plateaus at every map-size edge, the class merge up to 80 classes, the nearest-peak argmin,
the decode.py gates and the soft-NMS on their boundaries, all three apply_sigmoid modes through the whole record, and
the measured distance of the device sigmoid from torch's.

Wherever equality is asserted the maps are decoded with apply_sigmoid = 0, so the kernel and the oracle select from
the same bits, and nothing is excused by a fraction.  The semantics asserted here are pinned on the oracle side by
tests/test_decode_select_ref.py."""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.detector import dets_to_dict
from oracle import decode_ref
from tests import decode_scenes as S
from tests.util import DETS_KEYS, compare_records, oracle_records

pytestmark = pytest.mark.gpu

F32 = np.float32
SENT = F32(decode_ref.SENT)
# bound on the distance of the device sigmoid (sigmoid_acc: 1 / (1 + expf(-x))) from torch.sigmoid on the CPU over
# logits in [-20, 20].  test_sigmoid_ulp_distance measured 4 ulp (H100 80GB HBM3, CUDA 12.9, torch 2.11 on an x86-64
# host; DESIGN.md section 5).  The CPU side is torch's vectorised sigmoid, whose last bits may depend on the host's
# SIMD path, so the bound leaves 2 ulp of headroom over the measurement; the test prints the value it sees.
SIGMOID_MAX_ULP = 6


def _decode(hb, K, apply_sigmoid, rep_mode=4, use_pnp=False, cam=None, **over):
    B, C, H, W = hb["hm"].shape
    prm = cpb.decode_params(None, rep_mode=rep_mode, K=K, num_classes=C, apply_sigmoid=apply_sigmoid,
                            use_pnp=use_pnp, **over)
    heads = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in hb.items()}
    w, h = 4 * W, 4 * H
    cam = synth.default_camera(w, h) if cam is None else cam
    meta = cpb.make_meta(B, np.array([w / 2., h / 2.], F32), float(max(w, h)), w, h, cam)
    dets, poses, n_valid = cpb.decode_pnp(heads, meta, prm, want_dets=True)
    torch.cuda.synchronize()
    return dets.cpu().numpy(), poses.cpu().numpy(), n_valid.cpu().numpy()


def _geometry(hb):
    H, W = hb["hm"].shape[2:]
    w, h = 4 * W, 4 * H
    return np.array([w / 2., h / 2.], F32), float(max(w, h)), w, h


def _frame(hb, b):
    return {k: v[b] for k, v in hb.items()}


def _assert_selection(dets, hb, K):
    """Score, index and class of every one of the K candidate rows equal the oracle's; zeros are reported as +0.0."""
    for b in range(hb["hm"].shape[0]):
        sc, ind, cls = S.oracle_selection(_frame(hb, b), K)
        got_sc = dets[b, :, L.D_SCORE]
        assert np.array_equal(dets[b, :, L.D_IND].astype(np.int64), ind), b
        assert np.array_equal(dets[b, :, L.D_CLS].astype(np.int64), cls), b
        assert np.array_equal(got_sc, sc), b
        assert not np.signbit(got_sc[got_sc == 0]).any(), b


@pytest.mark.parametrize("H,W,K,C", [
    (10, 10, 100, 1), (8, 16, 128, 1),                                 # HW == K
    (64, 64, 1, 1), (64, 64, 2, 2), (64, 64, 31, 7), (64, 64, 128, 7), (64, 64, 100, 80),
    (128, 128, 127, 1), (160, 160, 128, 1),                            # the largest map staged in shared memory
    (160, 161, 100, 1), (161, 160, 100, 2), (161, 160, 1, 1),          # the smallest maps kept in the workspace
    (208, 152, 128, 1)])
def test_selection_is_exact(H, W, K, C, cplib):
    """Six frames, one per map kind (quantised, constant, plateau + borders, raw negative with -0.0 maxima, raw mixed),
    rotated over the classes and the joints.  rep_mode 4 with zero hp_offset makes every record keypoint the chosen
    hm_hp peak (or the -10000 sentinel), so the per-joint top-K and the nearest-peak argmin are observable exactly."""
    B = len(S.KINDS)
    hb = S.selection_heads(B, C, H, W, seed=H * 1000 + W + K + C)
    dets, _, _ = _decode(hb, K, 0, rep_mode=4)
    _assert_selection(dets, hb, K)
    prm = decode_ref.DecodeParams(K=K, rep_mode=4)
    for b in range(B):
        want = decode_ref.decode(decode_ref.process_heads(_frame(hb, b), 0), prm)["kps"]
        assert np.array_equal(dets[b, :, L.D_KPS:L.D_KPS + 16], want), b


def test_mode1_selection_exact(cplib):
    """Logit maps (apply_sigmoid = 1) whose distinct values are far enough apart that both sigmoids keep them distinct
    and ordered: the selection is exact again, and the scores are within SIGMOID_MAX_ULP of torch's.  A constant-logit
    frame gives the first K indices of class 0."""
    B, C, H, W, K = 4, 2, 64, 64, 100
    rng = np.random.default_rng(41)
    hm = (rng.integers(-24, 25, size=(B, C, H, W)) / 4.0).astype(F32)
    hm[B - 1] = F32(0.5)
    hb = S.selection_heads(B, C, H, W, seed=42)
    hb["hm"] = hm
    vals = np.unique(decode_ref.sigmoid_f32(np.unique(hm)))
    assert vals.size == np.unique(hm).size                              # distinct and (np.unique) ordered on the CPU
    assert S.ulp_distance(vals[1:], vals[:-1]).min() > 2 * SIGMOID_MAX_ULP
    dets, _, _ = _decode(hb, K, 1, rep_mode=4)
    for b in range(B):
        sc, ind, cls = S.oracle_selection(_frame(hb, b), K, apply_sigmoid=1)
        assert np.array_equal(dets[b, :, L.D_IND].astype(np.int64), ind), b
        assert np.array_equal(dets[b, :, L.D_CLS].astype(np.int64), cls), b
        assert S.ulp_distance(dets[b, :, L.D_SCORE], sc).max() <= SIGMOID_MAX_ULP, b
    assert np.array_equal(dets[B - 1, :, L.D_IND], np.arange(K)) and (dets[B - 1, :, L.D_CLS] == 0).all()


def _mode_heads(mode, seed):
    """Planted scenes (cuboid projections, so the PnP is well posed) in the form each apply_sigmoid mode decodes:
    0 = both maps as probabilities, 1 = both as logits, 2 = hm a logit and hm_hp raw with a negative floor and
    exact -0.0 cells (an opt.mse_loss head)."""
    hb, truths = synth.planted_batch(2, n_obj=4, seed=seed, disagree_px=1.0)
    rng = np.random.default_rng(seed)
    if mode == 0:
        hb["hm"] = decode_ref.sigmoid_f32(hb["hm"])
        hb["hm_hp"] = decode_ref.sigmoid_f32(hb["hm_hp"])
    elif mode == 2:
        hp = decode_ref.sigmoid_f32(hb["hm_hp"]) - rng.uniform(0.0, 0.02, size=hb["hm_hp"].shape).astype(F32)
        zero = rng.random(hp.shape) < 0.002
        hp[zero & (hp < 0.01)] = F32(-0.0)
        hb["hm_hp"] = hp.astype(F32)
        assert (hb["hm_hp"] < 0).mean() > 0.5
    return hb, truths


@pytest.mark.parametrize("mode,moments", [(0, False), (0, True), (1, False), (1, True), (2, False), (2, True)])
def test_records_all_modes(mode, moments, cplib):
    """Every apply_sigmoid mode through the whole record against the oracle, with and without the moment window
    (mode 2 reads its raw hm_hp there and in the single-cell height): same detection set and order, the record
    tolerances of tests/util.compare_records, the dets fields at the tolerances of the reference goldens."""
    hb, truths = _mode_heads(mode, seed=1200 + mode)
    cam = truths[0]["cam"]
    c, s, w, h = _geometry(hb)
    dets, poses, n_valid = _decode(hb, 100, mode, rep_mode=1, use_pnp=True, cam=cam, use_moments=int(moments))
    dd = dets_to_dict(dets)
    prm = decode_ref.DecodeParams(rep_mode=1, use_moments=moments, vis_thresh=0.3)
    n_hm = 0
    for b in range(2):
        want_dets, want = oracle_records(_frame(hb, b), prm, cam, w, h, c, s, L, apply_sigmoid=mode)
        valid = want_dets["scores"][:, 0] > 0.05
        if mode == 0:                                   # same bits on both sides: every row is the oracle's
            _assert_selection(dets[b:b + 1], {"hm": hb["hm"][b:b + 1]}, 100)
        for k in DETS_KEYS:
            err = np.abs(dd[k][b][valid] - want_dets[k][valid]).max()
            assert err <= (1e-3 if "std" in k or "unc" in k else 2e-5), (b, k, err)
        assert n_valid[b] == want.shape[0] == len(truths[b]["R"])
        got = poses[b, :n_valid[b]]
        assert (got[:, L.P_SRC_INDEX] == want[:, L.P_SRC_INDEX]).all()
        compare_records(got, want, L)
        n_hm += int((want_dets["kps_heatmap_height"][valid] != SENT).sum())
    assert n_hm > 0                                     # the heat-map fields were reached, not only their sentinels


@pytest.mark.parametrize("rep_mode,moments", [(1, False), (1, True), (3, False), (4, False)])
def test_gate_boundaries(rep_mode, moments, cplib):
    """decode_scenes.gate_heads: joint peaks exactly on l / r / t / b, at exactly 0.3 * size and 0.5 * size, with a
    score of exactly 0.1f and just above, and equidistant pairs.  The keypoint source (peak or regressed), the
    kps_heatmap_* fields including their sentinels, the soft-NMS survivors and their order equal the oracle's."""
    heads, layout = S.gate_heads()
    K = 32
    dets, poses, n_valid = _decode(heads, K, 0, rep_mode=rep_mode, use_moments=int(moments))
    prm = decode_ref.DecodeParams(K=K, rep_mode=rep_mode, use_moments=moments, vis_thresh=0.3)
    c, s, _, _ = _geometry(heads)
    surv, want = S.oracle_survivors(_frame(heads, 0), prm, c, s)
    dd = dets_to_dict(dets)
    for k in ("scores", "bboxes", "kps", "kps_displacement_mean", "kps_heatmap_mean", "kps_heatmap_std",
              "kps_heatmap_height"):
        assert np.array_equal(dd[k][0], want[k]), k
    # a moment window holding two peaks has an empty centroid column (width 0 / 0): the reference raises there, both
    # sides write the -10000 sentinels
    assert not np.isnan(dets).any()
    assert n_valid[0] == len(surv) == len({i for i, _, _, _, _ in layout})
    assert np.array_equal(poses[0, :n_valid[0], L.P_SRC_INDEX], [k for k, _ in surv])
    assert np.abs(poses[0, :n_valid[0], L.P_SCORE] - np.array([v for _, v in surv])).max() <= 2e-6


@pytest.mark.parametrize("moments", [False, True])
def test_raw_moment_windows(moments, cplib):
    """apply_sigmoid = 2 on decode_scenes.raw_moment_heads: raw hm_hp windows with negative cells, non-positive totals
    and non-positive centroid row / column sums.  Where fitgaussian would reject the start point both sides write the
    -10000 sentinels (no NaN reaches the record); elsewhere the moments and the single-cell height equal the
    oracle's."""
    heads, _ = S.raw_moment_heads(seed=5)
    K = 32
    dets, _, _ = _decode(heads, K, 2, rep_mode=1, use_moments=int(moments))
    prm = decode_ref.DecodeParams(K=K, rep_mode=1, use_moments=moments, vis_thresh=0.3)
    want = decode_ref.decode(decode_ref.process_heads(_frame(heads, 0), 2), prm)
    dd = dets_to_dict(dets)
    assert not np.isnan(dets).any()
    assert np.array_equal(dets[0, :, L.D_IND], decode_ref.topk_classes(decode_ref.nms3x3(
        decode_ref.sigmoid_f32(heads["hm"][0])), K)[1])
    for k in ("kps", "kps_displacement_mean"):
        assert np.array_equal(dd[k][0], want[k]), k
    sent = want["kps_heatmap_height"] == SENT
    assert np.array_equal(dd["kps_heatmap_height"][0] == SENT, sent)
    assert 0 < sent[:9].sum() < sent[:9].size if moments else not sent[:9].any()
    for k in ("kps_heatmap_mean", "kps_heatmap_std", "kps_heatmap_height"):
        assert np.array_equal(dd[k][0] == SENT, want[k] == SENT), k
        assert np.allclose(dd[k][0], want[k], rtol=1e-6, atol=1e-6), k


def test_soft_nms_equal_scores(cplib):
    """Equal scores with identical and heavily overlapping boxes (decode_scenes.soft_nms_heads): the same survivors in
    the same order as the oracle's soft-NMS, ties going to the earlier candidate."""
    hb = S.soft_nms_heads()
    dets, poses, n_valid = _decode(hb, 16, 0, rep_mode=0)
    c, s, _, _ = _geometry(hb)
    surv, want = S.oracle_survivors(_frame(hb, 0), decode_ref.DecodeParams(K=16, rep_mode=0, vis_thresh=0.3), c, s)
    assert np.array_equal(dets[0, :, L.D_SCORE], want["scores"][:, 0])
    assert n_valid[0] == len(surv) == 8
    assert np.array_equal(poses[0, :n_valid[0], L.P_SRC_INDEX], [k for k, _ in surv])
    assert np.abs(poses[0, :n_valid[0], L.P_SCORE] - np.array([v for _, v in surv])).max() <= 2e-6


def test_sigmoid_ulp_distance(cplib):
    """64 frames of 128 single-cell logit peaks sweeping [-20, 20]: the decoded centre scores are the device sigmoid
    of known logits.  Prints and bounds their distance from torch.sigmoid on the CPU, in ulp."""
    hb = S.sigmoid_sweep_heads()
    B, K = hb["hm"].shape[0], 128
    dets, _, _ = _decode(hb, K, 1, rep_mode=0)
    ind = dets[:, :, L.D_IND].astype(np.int64)
    logits = np.take_along_axis(hb["hm"][:, 0].reshape(B, -1), ind, 1)
    assert np.array_equal(np.sort(logits.reshape(-1)), np.sort(np.linspace(-20, 20, B * K).astype(F32)))
    want = torch.sigmoid(torch.from_numpy(logits)).numpy()
    ulp = S.ulp_distance(dets[:, :, L.D_SCORE], want)
    worst = int(ulp.max())
    print("sigmoid_acc vs torch.sigmoid (CPU) over [-20, 20]: max %d ulp at logit %.4f, %.1f %% of %d logits "
          "bit-identical" % (worst, float(logits.reshape(-1)[ulp.argmax()]), 100.0 * (ulp == 0).mean(), ulp.size))
    assert worst <= SIGMOID_MAX_ULP

"""The oracle's selection helpers (oracle/decode_ref.py: nms3x3, topk_channel, topk_classes, the nearest-peak argmin
and process_heads) against their stated semantics, and the adversarial scenes of tests/decode_scenes.py against what
they claim to contain.  tests/test_gpu_decode_edges.py asserts the CUDA decode EQUAL to these helpers on tied and
boundary inputs, so this file has to hold on its own, without a GPU.

The rules: equality NMS keeps every cell equal to its 3x3 max (-inf padding), -0.0 compares equal to +0.0; top-K is
value descending, ties by ascending flat index; the class merge orders equal values by class * K + k; the nearest
heat-map peak is the first minimum in top-K order."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import decode_ref
from tests import decode_scenes as S

F32 = np.float32


def _torch_nms(heat):
    t = torch.from_numpy(heat)[None]
    hmax = F.max_pool2d(t, 3, stride=1, padding=1)
    return (t * (hmax == t).float())[0].numpy()


def _by_value_then_index(v, K):
    """Brute force: the K best of a flat vector, value descending, ties by ascending index (a stable sort)."""
    order = sorted(range(v.size), key=lambda i: (-float(v[i]), i))[:K]
    return np.asarray(order, np.int64)


@pytest.mark.parametrize("C,H,W,K", [(1, 16, 16, 10), (3, 33, 17, 40), (2, 64, 64, 100)])
def test_untied_matches_torch(C, H, W, K):
    """Continuous maps (no ties among the NMS survivors): max_pool2d equality NMS and torch.topk, bit for bit."""
    rng = np.random.default_rng(C * 1000 + H)
    heat = rng.uniform(0.1, 1.0, size=(C, H, W)).astype(F32)
    n = decode_ref.nms3x3(heat)
    assert np.array_equal(n, _torch_nms(heat))
    assert ((n > 0).reshape(C, -1).sum(1) >= K).all()          # the K-th value is a survivor, not a zero tie
    sc, ind, ys, xs = decode_ref.topk_channel(n, K)
    tv, ti = torch.topk(torch.from_numpy(n).reshape(C, -1), K)
    assert np.array_equal(sc, tv.numpy()) and np.array_equal(ind, ti.numpy())
    assert np.array_equal(ys, (ind // W).astype(F32)) and np.array_equal(xs, (ind % W).astype(F32))
    # decode.py:52-68 _topk: topk per class, then topk over the C*K candidates
    s2, i2, c2, _, _ = decode_ref.topk_classes(n, K)
    tv2, tk2 = torch.topk(tv.reshape(-1), K)
    assert np.array_equal(s2, tv2.numpy())
    assert np.array_equal(c2, (tk2 // K).numpy()) and np.array_equal(i2, ti.reshape(-1)[tk2].numpy())


@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("H,W,K", [(10, 10, 100), (8, 16, 128), (37, 23, 31), (64, 64, 1), (64, 64, 128)])
def test_ties_by_ascending_index(kind, H, W, K):
    rng = np.random.default_rng(H * W + K)
    heat = S.tie_map(kind, H, W, rng)[None]
    n = decode_ref.nms3x3(heat)
    assert np.array_equal(n, _torch_nms(heat))                  # same keep decisions as the reference, zeros included
    sc, ind, _, _ = decode_ref.topk_channel(n, K)
    want = _by_value_then_index(n.reshape(-1), K)
    assert np.array_equal(ind[0], want)
    assert np.array_equal(sc[0], n.reshape(-1)[want])
    if kind == "const":
        assert np.array_equal(ind[0], np.arange(K))             # every cell survives: the first K indices


def test_negative_zero_equals_positive_zero():
    """A -0.0 local maximum of a raw map ties with the +0.0 of suppressed cells, by index, in the NMS and the top-K."""
    heat = -np.random.default_rng(11).uniform(0.5, 1.0, size=(1, 5, 6)).astype(F32)
    heat[0, 2, 3] = F32(-0.0)             # local max among negatives: kept as -0.0
    heat[0, 4, 5] = F32(0.5)
    n = decode_ref.nms3x3(heat)
    assert n[0, 2, 3] == 0 and np.signbit(n[0, 2, 3])
    sc, ind, _, _ = decode_ref.topk_channel(n, 20)
    assert ind[0, 0] == 29 and sc[0, 0] == F32(0.5)
    # the suppressed cells (-0.0 from `heat * keep` on negatives) and the -0.0 maximum are one tie, in index order,
    # ahead of every negative maximum
    zeros = np.flatnonzero(n.reshape(-1) == 0)
    assert zeros.size >= 19 and 15 in zeros[:19]
    assert np.array_equal(ind[0, 1:], zeros[:19]) and (sc[0, 1:] == 0).all()
    # the same with the maximum and a suppressed zero swapped in sign: nothing changes
    heat2 = heat.copy()
    heat2[0, 2, 3] = F32(0.0)
    assert np.array_equal(decode_ref.topk_channel(decode_ref.nms3x3(heat2), 20)[1], ind)
    # -0.0 next to +0.0: both are maxima of their window
    pair = np.full((1, 3, 4), -2.0, F32)
    pair[0, 1, 1], pair[0, 1, 2] = F32(-0.0), F32(0.0)
    k = decode_ref.nms3x3(pair) == 0
    assert k[0, 1, 1] and k[0, 1, 2]
    assert np.array_equal(k, _torch_nms(pair) == 0)


def test_class_merge_ties_by_class_then_rank():
    """Equal values in several classes: class * K + k order (decode.py:52-68 on an index-ascending topk)."""
    K = 4
    sc = np.array([[0.9, 0.5, 0.5, 0.1], [0.5, 0.5, 0.2, 0.1], [0.9, 0.5, 0.0, 0.0]], F32)
    flat = sc.reshape(-1)
    want = _by_value_then_index(flat, K)
    assert list(want) == [0, 8, 1, 2]
    heat = np.zeros((3, 1, 16), F32)     # a 1 x 16 map per class whose NMS survivors are exactly these values
    for c in range(3):
        heat[c, 0, 0:2 * K:2] = sc[c]
    n = decode_ref.nms3x3(heat)
    s, ind, cls, _, _ = decode_ref.topk_classes(n, K)
    assert list(cls) == [0, 2, 0, 0] and list(ind) == [0, 0, 2, 4] and np.array_equal(s, flat[want])


@pytest.mark.parametrize("C", [2, 7, 80])
def test_class_merge_brute_force(C):
    """topk_classes on tie-heavy maps of 2, 7 and 80 classes equals a stable sort of every (class, cell)."""
    H, W, K = 24, 20, 100
    hb = S.selection_heads(1, C, H, W, seed=C)
    n = decode_ref.nms3x3(hb["hm"][0])
    s, ind, cls, _, _ = decode_ref.topk_classes(n, K)
    per = np.stack([_by_value_then_index(n[c].reshape(-1), K) for c in range(C)])
    vals = np.stack([n[c].reshape(-1)[per[c]] for c in range(C)])
    pick = _by_value_then_index(vals.reshape(-1), K)
    assert np.array_equal(cls, pick // K) and np.array_equal(ind, per.reshape(-1)[pick])
    assert np.array_equal(s, vals.reshape(-1)[pick])
    # the scene holds equal top values in more than one class
    assert len({float(v) for v in vals[:, 0]}) < C


def test_nearest_peak_first_minimum():
    """Two heat-map peaks equidistant from a regressed keypoint: decode() takes the first in top-K order."""
    heads, layout = S.gate_heads()
    prm = decode_ref.DecodeParams(K=32, rep_mode=4)
    dets = decode_ref.decode(decode_ref.process_heads({k: v[0] for k, v in heads.items()}, 0), prm)
    seen = set()
    for i, cx, cy, j, name in layout:
        kx, ky = dets["kps"][i, 2 * j], dets["kps"][i, 2 * j + 1]
        if name == "equidistant_x":         # equal scores: the lower index, (cx - 2, cy + 1)
            assert (kx, ky) == (cx - 2, cy + 1)
        elif name == "equidistant_d":       # scores 0.4 (lower index) and 0.6: the higher score is first in top-K order
            assert (kx, ky) == (cx + 3, cy + 1)
        seen.add(name)
    assert {"equidistant_x", "equidistant_d"} <= seen


def test_gate_scene_is_on_its_boundaries():
    """Every gate case of decode_scenes.gate_heads is decided ON its boundary in fp32, and the oracle takes the branch
    the case is named for (rep_mode 1: kps is the peak when no gate fails; the kps_heatmap_* fields need all seven)."""
    heads, layout = S.gate_heads()
    hb = {k: v[0] for k, v in heads.items()}
    prm = decode_ref.DecodeParams(K=32, rep_mode=1)
    dets = decode_ref.decode(decode_ref.process_heads(hb, 0), prm)
    assert F32(10) * F32(0.3) == F32(3) and F32(10) * F32(0.5) == F32(5)
    expect_peak = {"equidistant_x": True, "equidistant_d": True, "on_l": True, "on_r": True, "on_t": True,
                   "on_b": True, "at_0.3_size": True, "at_0.5_size": False, "score_0.1": False,
                   "score_above_0.1": True, "outside": False}
    expect_hm = dict(expect_peak)
    names = set()
    for i, cx, cy, j, name in layout:
        names.add(name)
        assert dets["scores"][i, 0] == F32(0.9 - 0.01 * i)
        bb = dets["bboxes"][i]
        assert list(bb) == [cx - 5, cy - 5, cx + 5, cy + 5]
        kx, ky = dets["kps"][i, 2 * j], dets["kps"][i, 2 * j + 1]
        rx, ry = dets["kps_displacement_mean"][i, 2 * j], dets["kps_displacement_mean"][i, 2 * j + 1]
        took_peak = (kx, ky) != (rx, ry)
        assert took_peak == expect_peak[name], (i, j, name)
        has_hm = dets["kps_heatmap_height"][i, j] != F32(decode_ref.SENT)
        assert has_hm == expect_hm[name], (i, j, name)
        if name.startswith("on_"):
            edge = {"on_l": kx == bb[0], "on_r": kx == bb[2], "on_t": ky == bb[1], "on_b": ky == bb[3]}[name]
            assert edge, (i, j, name)
    assert names == set(expect_peak)


def test_soft_nms_scene():
    """Identical boxes with equal scores: the first survives.  The decayed 0.7 moves behind the undecayed 0.6 ties, and
    the removal swaps the last live box into the removed slot, which puts the 0.5 pair in reverse index order."""
    hb = {k: v[0] for k, v in S.soft_nms_heads().items()}
    prm = decode_ref.DecodeParams(K=16, rep_mode=0, vis_thresh=0.3)
    surv, dets = S.oracle_survivors(hb, prm, np.array([32., 32.], F32), 64.0)
    sc = dets["scores"][:, 0]
    assert list(sc[:9]) == [F32(v) for v in (0.8, 0.8, 0.7, 0.7, 0.6, 0.6, 0.6, 0.5, 0.5)]
    ks = [k for k, _ in surv]
    assert ks == [0, 2, 4, 5, 6, 3, 8, 7], ks
    assert surv[5][1] < 0.6 and 0.3 < surv[-1][1] < 0.5


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_process_heads_modes(mode):
    rng = np.random.default_rng(3)
    h = {"hm": rng.normal(size=(1, 4, 4)).astype(F32), "hm_hp": rng.normal(size=(8, 4, 4)).astype(F32),
         "wh": rng.normal(size=(2, 4, 4)).astype(F32)}
    out = decode_ref.process_heads(h, mode)
    sig = decode_ref.sigmoid_f32
    assert np.array_equal(out["hm"], h["hm"] if mode == 0 else sig(h["hm"]))
    assert np.array_equal(out["hm_hp"], sig(h["hm_hp"]) if mode == 1 else h["hm_hp"])
    assert np.array_equal(out["wh"], h["wh"])
    if mode == 1:       # the default is the reference's own path
        d = decode_ref.process_heads(h)
        assert all(np.array_equal(d[k], out[k]) for k in h)
    with pytest.raises(ValueError):
        decode_ref.process_heads(h, 3)


def test_scenes_are_deterministic():
    a = S.selection_heads(2, 3, 16, 16, seed=9)
    b = S.selection_heads(2, 3, 16, 16, seed=9)
    assert all(np.array_equal(a[k], b[k]) and a[k].dtype == np.float32 for k in a)
    assert a["hm"].shape == (2, 3, 16, 16) and a["hm_hp"].shape == (2, 8, 16, 16)
    s = S.sigmoid_sweep_heads(B=2, K=8)
    n = decode_ref.nms3x3(decode_ref.sigmoid_f32(s["hm"][1]))
    _, ind, _, _ = decode_ref.topk_channel(n, 8)
    assert set(s["hm"][1, 0].reshape(-1)[ind[0]]) == set(np.linspace(-20, 20, 16).astype(F32)[8:])


def test_raw_moment_scene_reaches_the_rejected_start_points():
    """decode_scenes.raw_moment_heads holds windows fitgaussian fits with negative cells, and windows it rejects for a
    non-positive total and for a non-positive centroid row / column sum.  The oracle decode writes the -10000
    sentinels for the rejected ones and never a NaN; the same holds for the two-peak windows of the gate scene."""
    heads, peaks = S.raw_moment_heads(seed=5)
    hp = heads["hm_hp"][0]
    cats = {"fit_with_negatives": 0, "total_le_0": 0, "centroid_line_le_0": 0}
    for i, j, px, py in peaks:
        w = S.moment_window(hp[j], px, py)
        if decode_ref.fit_start(w) is not None:
            cats["fit_with_negatives"] += int((w < 0).any())
            continue
        t = w.sum()
        if t <= 0:
            cats["total_le_0"] += 1
            continue
        X, Y = np.indices(w.shape)
        x, y = (X * w).sum() / t, (Y * w).sum() / t
        assert 0 <= x <= 11 and 0 <= y <= 11
        assert w[:, int(y)].sum() <= 0 or w[int(x), :].sum() <= 0
        cats["centroid_line_le_0"] += 1
    assert min(cats.values()) >= 5, cats
    prm = decode_ref.DecodeParams(K=32, rep_mode=1, use_moments=True)
    for hb, mode in ((heads, 2), (S.gate_heads()[0], 0)):
        with np.errstate(all="raise"):           # fit_start screens the 0 / 0 and sqrt(negative) of rejected windows
            d = decode_ref.decode(decode_ref.process_heads({k: v[0] for k, v in hb.items()}, mode), prm)
        h = d["kps_heatmap_height"][:9]
        assert not any(np.isnan(v).any() for v in d.values())
        assert 0 < (h == F32(decode_ref.SENT)).sum() < h.size

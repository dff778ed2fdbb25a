"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference's
post-network path: sigmoid -> 3x3 NMS -> top-K -> keypoint/centre grouping
-> output-map-to-image affine -> score filter + Gaussian soft-NMS.

Never imported by the product path (`centerpose_b200/`).

Parity status: PINNED -- `tests/test_oracle_decode.py` checks every function
here against the unmodified reference functions (through `oracle/ref_shims.py`,
when `/root/reference` is present) and against the golden vectors in
`tests/golden/decode_*.npz` that `oracle/make_golden.py` produced by running
the reference itself.

Reference lines followed (relative to /root/reference/src/lib):
  detectors/object_pose.py:136-138   sigmoid on hm / hm_hp       -> process_heads
  models/decode.py:17-23             _nms                        -> nms3x3
  models/decode.py:40-68             _topk_channel / _topk       -> topk_channel / topk_classes
  models/utils.py:43-47              _transpose_and_gather_feat  -> gather
  models/decode.py:72-375            object_pose_decode(Inference=True) -> decode
  utils/gpfit.py:13-41               moments / fitgaussian(max_nfev=1) -> moments / fit_start
  utils/image.py:23-74               transform_preds / get_affine_transform -> map_to_image
  utils/post_process.py:12-68        object_pose_post_process    -> post_process
  detectors/object_pose.py:27-124    soft_nms_nvidia(method=2)   -> soft_nms
  detectors/object_pose.py:184-197   merge_outputs               -> merge_outputs
"""
import math

import numpy as np

SENT = -10000.0
F32 = np.float32


class DecodeParams(object):
    """The subset of the reference `opt` the decode path reads."""

    def __init__(self, K=100, rep_mode=1, use_moments=False, balance=2.0, vis_thresh=0.3,
                 nms=True, category="chair", num_scales=1, modern_bool=False):
        self.K = K
        self.rep_mode = rep_mode
        # opt.tracking_task or opt.refined_Kalman or rep_mode == 2  (decode.py:222)
        self.use_moments = bool(use_moments or rep_mode == 2)
        self.balance = balance          # opt.balance_coefficient[opt.c]  (opts.py:239-241)
        self.vis_thresh = vis_thresh
        self.nms = nms
        self.category = category
        self.num_scales = num_scales
        # False: torch==1.1.0 (pinned) semantics of `mask_2 == 7` (decode.py:183-188); True: torch >= 1.2, where the sum of
        # bools is a logical OR and the comparison with 7 is never true
        self.modern_bool = bool(modern_bool)


def sigmoid_f32(x):
    """fp32 logistic; uses torch's CPU kernel when present so that it is
    bit-identical with the reference's `sigmoid_()` (object_pose.py:136)."""
    x = np.ascontiguousarray(x, dtype=F32)
    try:
        import torch
        return torch.sigmoid(torch.from_numpy(x)).numpy()
    except ImportError:     # pragma: no cover
        return (F32(1) / (F32(1) + np.exp(-x))).astype(F32)


def nms3x3(heat):
    """heat [C,H,W] fp32 -> heat * (maxpool3x3(heat) == heat)."""
    C, H, W = heat.shape
    pad = np.full((C, H + 2, W + 2), -np.inf, dtype=F32)
    pad[:, 1:-1, 1:-1] = heat
    hmax = pad[:, 1:-1, 1:-1].copy()
    for dy in range(3):
        for dx in range(3):
            hmax = np.maximum(hmax, pad[:, dy:dy + H, dx:dx + W])
    keep = (hmax == heat).astype(F32)
    return heat * keep


def topk_channel(scores, K):
    """scores [C,H,W] -> (score[C,K], ind[C,K], ys[C,K], xs[C,K]); descending
    value, ties broken by ascending index (torch.topk leaves tie order
    implementation-defined; SURVEY.md 8d 'tie hazard')."""
    C, H, W = scores.shape
    flat = scores.reshape(C, -1)
    sc = np.zeros((C, K), F32)
    ind = np.zeros((C, K), np.int64)
    for c in range(C):
        order = np.lexsort((np.arange(flat.shape[1]), -flat[c].astype(np.float64)))[:K]
        ind[c] = order
        sc[c] = flat[c, order]
    ys = (ind // W).astype(F32)
    xs = (ind % W).astype(F32)
    return sc, ind, ys, xs


def topk_classes(scores, K):
    """decode.py:52-68 -- per-class top-K then top-K over classes."""
    sc, ind, ys, xs = topk_channel(scores, K)
    flat = sc.reshape(-1)
    order = np.lexsort((np.arange(flat.size), -flat.astype(np.float64)))[:K]
    clses = (order // K).astype(np.int64)
    return flat[order], ind.reshape(-1)[order], clses, ys.reshape(-1)[order], xs.reshape(-1)[order]


def gather(feat, ind):
    """feat [C,H,W], ind [N] -> [N,C]  (channel-last gather, utils.py:43-47)."""
    C = feat.shape[0]
    return feat.reshape(C, -1)[:, ind].T.astype(F32)


def moments(data):
    """utils/gpfit.py:13-26, float64.  Returns (height, x, y, width_x, width_y)
    with the file's own conventions: x is the ROW centroid, y the COLUMN
    centroid, width_x is computed from column int(y) with (i - y)^2 and
    width_y from row int(x) with (i - x)^2.  `fitgaussian` runs
    `least_squares(..., max_nfev=1)` which returns its (bounds-clipped) start
    point, so the fit is a no-op apart from the clip into
    [0, inf) x [0, rows] x [0, cols] x [0, inf)^2 made strictly feasible."""
    data = np.asarray(data, np.float64)
    total = data.sum()
    X, Y = np.indices(data.shape)
    x = (X * data).sum() / total
    y = (Y * data).sum() / total
    col = data[:, int(y)]
    width_x = np.sqrt(np.abs((np.arange(col.size) - y) ** 2 * col).sum() / col.sum())
    row = data[int(x), :]
    width_y = np.sqrt(np.abs((np.arange(row.size) - x) ** 2 * row).sum() / row.sum())
    height = data.max()
    return height, x, y, width_x, width_y


def fit_start(data):
    """What `fitgaussian` (gpfit.py:29-41) returns for a window, or None where the reference raises.  Raises are:
    `moments` indexing a row / column that does not exist (int(NaN), a centroid of exactly rows or cols), and
    least_squares rejecting the start point, because it is outside bounds=(0, [inf, rows, cols, inf, inf]) or NaN.
    Otherwise max_nfev=1 returns the start point; a zero width is made strictly feasible."""
    rows, cols = np.asarray(data).shape
    with np.errstate(divide="ignore", invalid="ignore"):
        try:
            height, x, y, width_x, width_y = moments(data)
        except (ValueError, IndexError, OverflowError):
            return None
    if not (height >= 0 and 0 <= x <= rows and 0 <= y <= cols and width_x >= 0 and width_y >= 0):
        return None
    # least_squares(max_nfev=1) only makes x0 strictly feasible
    width_x = max(width_x, 1e-10) if width_x == 0 else width_x
    width_y = max(width_y, 1e-10) if width_y == 0 else width_y
    return height, x, y, width_x, width_y


def process_heads(heads, apply_sigmoid=1):
    """object_pose.py:136-138 -- returns a copy with sigmoid applied as `cp_decode_params.apply_sigmoid` says:
    0 = hm and hm_hp are probabilities already (neither is touched), 1 = both are logits, 2 = only hm is a logit
    (opt.mse_loss: hm_hp is decoded raw, and the moment window and the height read see the raw values)."""
    if apply_sigmoid not in (0, 1, 2):
        raise ValueError("apply_sigmoid must be 0, 1 or 2")
    out = {k: np.ascontiguousarray(v, dtype=F32) for k, v in heads.items()}
    if apply_sigmoid != 0:
        out["hm"] = sigmoid_f32(out["hm"])
    if "hm_hp" in out and apply_sigmoid == 1:
        out["hm_hp"] = sigmoid_f32(out["hm_hp"])
    return out


def decode(heads, prm):
    """heads: dict of [C,H,W] fp32 arrays for ONE image, hm / hm_hp already
    sigmoid'ed (see process_heads).  Returns the 13 arrays of decode.py:348-361
    without the batch dimension."""
    K = prm.K
    heat = heads["hm"]
    H, W = heat.shape[1:]
    J = heads["hps"].shape[0] // 2
    th = F32(0.1)

    heat_n = nms3x3(heat)
    scores, inds, clses, ys, xs = topk_classes(heat_n, K)

    kps = gather(heads["hps"], inds)                       # [K,2J]
    kps[:, 0::2] += xs[:, None]
    kps[:, 1::2] += ys[:, None]
    if "reg" in heads:
        reg = gather(heads["reg"], inds)
        cx = xs + reg[:, 0]
        cy = ys + reg[:, 1]
    else:
        cx = xs + F32(0.5)
        cy = ys + F32(0.5)
    wh = gather(heads["wh"], inds)
    two = F32(2)
    bboxes = np.stack([cx - wh[:, 0] / two, cy - wh[:, 1] / two,
                       cx + wh[:, 0] / two, cy + wh[:, 1] / two], 1).astype(F32)

    kps_disp = kps.copy()
    hm_hp_copy = heads["hm_hp"]
    hm_hp = nms3x3(hm_hp_copy)
    hm_score, hm_inds, hm_ys, hm_xs = topk_channel(hm_hp, K)        # [J,K]
    if "hp_offset" in heads:
        off = gather(heads["hp_offset"], hm_inds.reshape(-1)).reshape(J, K, 2)
        hm_xs = hm_xs + off[:, :, 0]
        hm_ys = hm_ys + off[:, :, 1]
    else:
        hm_xs = hm_xs + F32(0.5)
        hm_ys = hm_ys + F32(0.5)
    m = (hm_score > th)
    hm_score = np.where(m, hm_score, F32(-1)).astype(F32)
    hm_ys = np.where(m, hm_ys, F32(SENT)).astype(F32)
    hm_xs = np.where(m, hm_xs, F32(SENT)).astype(F32)

    kps_out = kps.copy()
    hmean = np.full((K, 2 * J), SENT, F32)
    hstd = np.full((K, 2 * J), SENT, F32)
    hheight = np.full((K, J), SENT, F32)
    l, t, r, b = bboxes[:, 0], bboxes[:, 1], bboxes[:, 2], bboxes[:, 3]
    size = np.maximum(b - t, r - l)
    for j in range(J):
        rx = kps[:, 2 * j][:, None]
        ry = kps[:, 2 * j + 1][:, None]
        dx = rx - hm_xs[j][None, :]
        dy = ry - hm_ys[j][None, :]
        dist = np.sqrt((dx * dx + dy * dy).astype(F32)).astype(F32)   # [K centres, K peaks]
        mi = np.argmin(dist, 1)
        md = dist[np.arange(K), mi]
        sx = hm_xs[j][mi]
        sy = hm_ys[j][mi]
        ss = hm_score[j][mi]
        bad = (sx < l) | (sx > r) | (sy < t) | (sy > b) | (ss < th) | (md > size * F32(0.3))
        if prm.rep_mode == 3:
            pass
        elif prm.rep_mode == 4:
            kps_out[:, 2 * j] = sx
            kps_out[:, 2 * j + 1] = sy
        else:
            kps_out[:, 2 * j] = np.where(bad, kps[:, 2 * j], sx)
            kps_out[:, 2 * j + 1] = np.where(bad, kps[:, 2 * j + 1], sy)
        ok2 = (sx > F32(0.8) * l) & (sx < F32(1.2) * r) & (sy > F32(0.8) * t) & (sy < F32(1.2) * b) \
            & (ss > th) & (md < size * F32(0.5)) & (scores > th)
        if prm.modern_bool:
            ok2 = np.zeros_like(ok2)
        if prm.rep_mode in (1, 2):
            data = hm_hp_copy[j]
            for k in range(K):
                if not ok2[k]:
                    continue
                fx, fy = sx[k], sy[k]
                if fx == F32(SENT) or fy == F32(SENT):
                    continue
                ran = 5
                if prm.use_moments:
                    big = np.zeros((H + 2 * ran, W + 2 * ran))
                    big[ran:H + ran, ran:W + ran] = data
                    win = big[int(fy):int(fy + 2 * ran + 1), int(fx):int(fx + 2 * ran + 1)]
                    fit = fit_start(win)
                    if fit is None:         # the reference raises here; the -10000 sentinels stay (DESIGN.md 5)
                        continue
                    height, mu_x, mu_y, std_x, std_y = fit
                else:
                    mu_x = ran
                    mu_y = ran
                    height = data[int(fy), int(fx)]
                    std_x = 1
                    std_y = 1
                hmean[k, 2 * j] = F32(fx + mu_x - ran)
                hmean[k, 2 * j + 1] = F32(fy + mu_y - ran)
                hstd[k, 2 * j] = F32(std_x)
                hstd[k, 2 * j + 1] = F32(std_y)
                hheight[k, j] = F32(height)

    out = {
        "bboxes": bboxes, "scores": scores.reshape(K, 1).astype(F32), "kps": kps_out.astype(F32),
        "clses": clses.reshape(K, 1).astype(F32),
        "kps_displacement_mean": kps_disp.astype(F32),
        "kps_heatmap_mean": hmean, "kps_heatmap_std": hstd, "kps_heatmap_height": hheight,
    }
    if "hps_uncertainty" in heads:
        u = gather(heads["hps_uncertainty"], inds)
        out["kps_displacement_std"] = (np.sqrt(np.exp(u)) * F32(prm.balance)).astype(F32)
    else:
        out["kps_displacement_std"] = np.zeros((K, 2 * J), F32)
    out["obj_scale"] = gather(heads["scale"], inds) if "scale" in heads else np.zeros((K, 3), F32)
    if "scale_uncertainty" in heads:
        out["obj_scale_uncertainty"] = np.sqrt(np.exp(gather(heads["scale_uncertainty"], inds))).astype(F32)
    else:
        out["obj_scale_uncertainty"] = np.zeros((K, 3), F32)
    out["tracking"] = gather(heads["tracking"], inds) if "tracking" in heads else np.zeros((K, 2), F32)
    out["tracking_hp"] = gather(heads["tracking_hp"], inds) if "tracking_hp" in heads \
        else np.zeros((K, 2 * J), F32)
    return out


def map_to_image(pts, c, s, out_w, out_h):
    """utils/image.py:23-74 with rot=0.  The reference builds a 3-point affine
    and lets cv2.getAffineTransform solve it in float64; with rot=0 the
    solution is the isotropic map  p*a + (c - a*out/2),  a = src_w/dst_w,
    where the point pairs are first rounded to float32 (image.py:52-66)."""
    pts = np.asarray(pts, F32).reshape(-1, 2)
    src_w = F32(s[0]) if isinstance(s, (np.ndarray, list)) else F32(s)
    cx, cy = F32(c[0]), F32(c[1])
    dst_w, dst_h = F32(out_w), F32(out_h)
    # float32 control points exactly as the reference stores them
    d0 = np.array([dst_w * F32(0.5), dst_h * F32(0.5)], F32)
    d1 = d0 + np.array([0, dst_w * F32(-0.5)], F32)
    s0 = np.array([cx, cy], F32)
    s1 = (s0 + np.array([0, src_w * F32(-0.5)], F32)).astype(F32)
    a = (float(s0[1]) - float(s1[1])) / (float(d0[1]) - float(d1[1]))
    tx = float(s0[0]) - a * float(d0[0])
    ty = float(s0[1]) - a * float(d0[1])
    out = np.zeros(pts.shape, np.float64)
    for i in range(pts.shape[0]):
        if pts[i, 0] == F32(SENT) and pts[i, 1] == F32(SENT):
            out[i] = [SENT, SENT]
        else:
            out[i, 0] = a * float(pts[i, 0]) + tx
            out[i, 1] = a * float(pts[i, 1]) + ty
    return out


SCALED_KEYS = ("bbox", "kps", "kps_displacement_std", "tracking", "tracking_hp", "kps_displacement_mean", "kps_heatmap_mean")


def post_process(dets, c, s, out_h, out_w, scale=1):
    """utils/post_process.py:12-68 (Inference=True) for one image: list of K dicts, followed by the division of
    detectors/object_pose.py:171-177 when the pass ran at a test scale != 1 (`ct` and kps_heatmap_std stay as they are)."""
    coefficient = 0.32
    K = dets["scores"].shape[0]
    ssc = (F32(s[0]) if isinstance(s, (np.ndarray, list)) else s)
    # `s[i] / max(w, h)`: python/np scalar division, float64 unless s is np.float32
    ratio = ssc / max(out_w, out_h)
    preds = []
    for j in range(K):
        item = {}
        item["score"] = float(dets["scores"][j, 0])
        item["cls"] = int(dets["clses"][j, 0])
        item["obj_scale"] = dets["obj_scale"][j]
        item["obj_scale_uncertainty"] = dets["obj_scale_uncertainty"][j]
        item["kps_displacement_std"] = (dets["kps_displacement_std"][j] * ratio * coefficient).flatten()
        bbox = map_to_image(dets["bboxes"][j], c, s, out_w, out_h)
        item["bbox"] = bbox.reshape(-1)
        item["ct"] = [(item["bbox"][0] + item["bbox"][2]) / 2, (item["bbox"][1] + item["bbox"][3]) / 2]
        item["kps"] = map_to_image(dets["kps"][j], c, s, out_w, out_h).reshape(-1)
        item["tracking"] = (dets["tracking"][j] * ratio).flatten()
        item["tracking_hp"] = (dets["tracking_hp"][j] * ratio).flatten()
        item["kps_displacement_mean"] = map_to_image(dets["kps_displacement_mean"][j], c, s, out_w, out_h).reshape(-1)
        item["kps_heatmap_mean"] = map_to_image(dets["kps_heatmap_mean"][j], c, s, out_w, out_h).reshape(-1)
        item["kps_heatmap_std"] = (dets["kps_heatmap_std"][j] * ratio * coefficient).flatten()
        item["kps_heatmap_height"] = dets["kps_heatmap_height"][j]
        if scale != 1:
            for k in SCALED_KEYS:
                item[k] = (np.array(item[k], np.float32) / scale).tolist()
        preds.append(item)
    return preds


def soft_nms(boxes, sigma=0.5, threshold=0.001):
    """object_pose.py:27-124 with method=2 (Gaussian).  `boxes` is a list of
    dicts; it is permuted / rescored in place exactly like the reference and
    the surviving prefix length is returned."""
    N = len(boxes)
    i = 0
    while i < N:
        maxpos = i
        maxscore = boxes[i]["score"]
        for pos in range(i + 1, N):
            if maxscore < boxes[pos]["score"]:
                maxscore = boxes[pos]["score"]
                maxpos = pos
        boxes[i], boxes[maxpos] = boxes[maxpos], boxes[i]
        tx1, ty1, tx2, ty2 = [float(v) for v in boxes[i]["bbox"]]
        pos = i + 1
        while pos < N:
            x1, y1, x2, y2 = [float(v) for v in boxes[pos]["bbox"]]
            area = (x2 - x1 + 1) * (y2 - y1 + 1)
            iw = min(tx2, x2) - max(tx1, x1) + 1
            if iw > 0:
                ih = min(ty2, y2) - max(ty1, y1) + 1
                if ih > 0:
                    ua = float((tx2 - tx1 + 1) * (ty2 - ty1 + 1) + area - iw * ih)
                    ov = iw * ih / ua
                    weight = math.exp(-(ov * ov) / sigma)
                    boxes[pos]["score"] = weight * boxes[pos]["score"]
                    if boxes[pos]["score"] < threshold:
                        # pos takes (bbox, score) of the last live box and swaps the other keys
                        last = boxes[N - 1]
                        cur = boxes[pos]
                        lb, ls = last["bbox"], last["score"]
                        boxes[pos], boxes[N - 1] = last, cur
                        boxes[pos]["bbox"], boxes[pos]["score"] = lb, ls
                        N -= 1
                        pos -= 1
            pos += 1
        i += 1
    return N


def merge_outputs(preds, prm):
    """object_pose.py:184-197 for a single scale."""
    results = [dict(d) for d in preds if d["score"] > prm.vis_thresh]
    if prm.nms or prm.num_scales > 1:
        n = soft_nms(results, threshold=prm.vis_thresh)
        results = results[:n]
    return results

"""Decode scenes that hand chosen image points to the PnP.

The PnP of `cp_decode_pnp` (pnp_warp.cuh, called from phase G of decode.cu) only sees what the decode assembles: 8 or 16
image points, the `scale` head at the centre cell and the camera of the frame.  The builders here write head maps whose
decode yields points at chosen image positions, so that tests drive the product kernel -- its point assembly, the
warp loop over detections and the reuse of one scratch region per warp -- rather than a test-only entry point.

- rep_mode 0 (`rep0_scene`): one `hm` peak per object on its own centre cell, `hps` at that cell = target map position
  - cell, `hm_hp` zero (apply_sigmoid = 0: no joint peak passes 0.1, every keypoint is its regressed position).  Any
  position is reachable, including far outside the frame; a target below -5000 is a point `pnp_collect` drops.
- rep_mode 4 (`rep4_scene`): 0 - 8 valid points from `hm_hp` peaks at floor(target map position) with `hp_offset` =
  the fraction.  A joint without a peak decodes to the -10000 sentinel.  One object per image, because the nearest-peak
  match would hand a dropped joint another object's peak; `hp_offset` is one map for all joints, so two joints on one
  cell are refused.
- rep_mode 1 (`rep1_scene`): 16 points from `synth.planted_batch` (disagreeing displacement / heat-map means, dropped
  heat-map joints).

Every scene decodes with nms = 0 and vis_thresh 0.3, and its centre scores descend in placement order, so pose record i
of image b is object i of image b.  The intended points are only intended: the tests read the points the kernel used
back from `dets` and rebuild them in fp64 with `decode_ref.map_to_image` (`aff * (double)x + tx`, as decode.cu does).
"""
import numpy as np

from centerpose_b200 import synth
from oracle import decode_ref, pnp_ref

F32 = np.float32
J = 8
SENT = -10000.0
OK, INVISIBLE, BEHIND, FEW_POINTS, SOLVER_FAIL = 1, 2, 3, 4, 5
HAS_POSE = (OK, INVISIBLE)
VISIBLE = {0: "bike", 3: "cup", 6: "chair"}          # visible_thresh -> a category of the reference with that gate
VISIBLE_OF = {"book": 6, "chair": 6, "cereal_box": 6, "camera": 3, "bottle": 3, "cup": 3, "bike": 0, "laptop": 0,
              "shoe": 0}                             # category -> visible_thresh (cuboid_pnp_shell.py:59-66)
M_GL = np.array([[0, 1, 0], [1, 0, 0], [0, 0, -1.0]])  # OpenCV -> OpenGL frame change of cuboid_pnp_solver.py


class Scene(object):
    """One `cp_decode_pnp` call.  objs[b][i]: dict(pts [n_in,2] intended image points (SENT rows: not decoded),
    scale [3] fp32, npts intended valid count, want set of intended statuses or None, tag str)."""

    def __init__(self, cls, name, rep_mode, heads, objs, c, s, img_w, img_h, cam, visible_thresh=6, opencv_return=0,
                 apply_sigmoid=0, K=100):
        self.cls, self.name, self.rep_mode, self.heads, self.objs = cls, name, rep_mode, heads, objs
        self.c, self.s, self.img_w, self.img_h = np.asarray(c, F32), float(s), img_w, img_h
        self.cam = np.asarray(cam, np.float64)
        self.visible_thresh, self.opencv_return, self.apply_sigmoid, self.K = visible_thresh, opencv_return, \
            apply_sigmoid, K
        self.B, _, self.out_h, self.out_w = heads["hm"].shape

    @property
    def n_in(self):
        return 16 if self.rep_mode == 1 else 8

    def decode_kwargs(self):
        return dict(rep_mode=self.rep_mode, nms=False, K=self.K, visible_thresh=self.visible_thresh,
                    show_axes=bool(self.opencv_return), apply_sigmoid=self.apply_sigmoid, vis_thresh=0.3)

    def oracle_params(self):
        return decode_ref.DecodeParams(K=self.K, rep_mode=self.rep_mode, vis_thresh=0.3, nms=False,
                                       category=VISIBLE[self.visible_thresh])


def affine(c, s, out_w, out_h):
    """(a, tx, ty) of decode_ref.map_to_image: image = a * map + (tx, ty)."""
    p = decode_ref.map_to_image(np.array([[0.0, 0.0]], F32), c, s, out_w, out_h)[0]
    q = decode_ref.map_to_image(np.array([[1.0, 0.0]], F32), c, s, out_w, out_h)[0]
    return q[0] - p[0], p[0], p[1]


def used_points(dets_row, rep_mode, c, s, out_w, out_h, D):
    """The fp64 image points the kernel hands the PnP, rebuilt from one `dets` row (fp32 map coordinates)."""
    if rep_mode == 1:
        a = decode_ref.map_to_image(dets_row[D.D_KPS_DISP_MEAN:D.D_KPS_DISP_MEAN + 16], c, s, out_w, out_h)
        b = decode_ref.map_to_image(dets_row[D.D_KPS_HM_MEAN:D.D_KPS_HM_MEAN + 16], c, s, out_w, out_h)
        return np.hstack([a, b]).reshape(16, 2)
    return decode_ref.map_to_image(dets_row[D.D_KPS:D.D_KPS + 16], c, s, out_w, out_h)


def n_valid_points(pts):
    pts = np.asarray(pts, np.float64)
    return int((~((pts[:, 0] < -5000) | (pts[:, 1] < -5000))).sum())


def _blank(B, H, W):
    z = lambda ch: np.zeros((B, ch, H, W), F32)      # noqa: E731
    return {"hm": z(1), "wh": z(2), "hps": z(2 * J), "reg": z(2), "hm_hp": z(J), "hp_offset": z(2), "scale": z(3)}


def _score(i):
    return F32(0.9 - 0.003 * i)


def _cells(H, W, n, step=4):
    cells = [(x, y) for y in range(2, H - 1, step) for x in range(2, W - 1, step)]
    if n > len(cells):
        raise ValueError("%d objects do not fit a %dx%d map at spacing %d" % (n, H, W, step))
    return cells[:n]


def rep0_scene(cls, name, objs, out_h=128, out_w=128, img_w=512, img_h=512, c=None, s=None, cam=None, **kw):
    """objs[b][i]: dict(pts [8,2] image targets, scale [3]).  Targets below -5000 make points pnp_collect drops."""
    c = np.array([img_w / 2.0, img_h / 2.0], F32) if c is None else np.asarray(c, F32)
    s = float(max(img_w, img_h)) if s is None else s
    cam = synth.default_camera(img_w, img_h) if cam is None else cam
    a, tx, ty = affine(c, s, out_w, out_h)
    B = len(objs)
    h = _blank(B, out_h, out_w)
    for b, row in enumerate(objs):
        for i, (o, (cx, cy)) in enumerate(zip(row, _cells(out_h, out_w, len(row)))):
            h["hm"][b, 0, cy, cx] = _score(i)
            h["wh"][b, :, cy, cx] = 10.0
            h["scale"][b, :, cy, cx] = np.asarray(o["scale"], F32)
            m = (np.asarray(o["pts"], np.float64) - [tx, ty]) / a
            with np.errstate(over="ignore", invalid="ignore"):
                h["hps"][b, 0::2, cy, cx] = (m[:, 0] - cx).astype(F32)
                h["hps"][b, 1::2, cy, cx] = (m[:, 1] - cy).astype(F32)
            o.setdefault("npts", n_valid_points(o["pts"]))
    return Scene(cls, name, 0, h, objs, c, s, img_w, img_h, cam, **kw)


def rep4_scene(cls, name, objs, out_h=128, out_w=128, img_w=512, img_h=512, cam=None, **kw):
    """objs[b]: ONE dict(pts [8,2] image targets, NaN rows = joints without a heat-map peak, scale [3]) per image."""
    c = np.array([img_w / 2.0, img_h / 2.0], F32)
    s = float(max(img_w, img_h))
    cam = synth.default_camera(img_w, img_h) if cam is None else cam
    a, tx, ty = affine(c, s, out_w, out_h)
    B = len(objs)
    h = _blank(B, out_h, out_w)
    rows = []
    for b, o in enumerate(objs):
        pts = np.asarray(o["pts"], np.float64)
        keep = ~np.isnan(pts[:, 0])
        m = (pts - [tx, ty]) / a
        cell = np.floor(m)
        used = [tuple(v) for v in cell[keep].astype(int)]
        if len(set(used)) != len(used):
            raise ValueError("rep4_scene: two joints on one hp_offset cell")
        if keep.any() and (cell[keep].min() < 0 or cell[keep, 0].max() >= out_w or cell[keep, 1].max() >= out_h):
            raise ValueError("rep4_scene: a joint peak outside the map")
        ctr = np.clip(np.floor(np.nanmean(m, 0)) if keep.any() else [out_w // 2, out_h // 2], 0,
                      [out_w - 1, out_h - 1]).astype(int)
        cx, cy = int(ctr[0]), int(ctr[1])
        h["hm"][b, 0, cy, cx] = _score(0)
        h["wh"][b, :, cy, cx] = 10.0
        h["scale"][b, :, cy, cx] = np.asarray(o["scale"], F32)
        for j in range(J):
            tgt = m[j] if keep[j] else np.array([cx, cy], np.float64)
            h["hps"][b, 2 * j, cy, cx] = F32(tgt[0] - cx)
            h["hps"][b, 2 * j + 1, cy, cx] = F32(tgt[1] - cy)
            if keep[j]:
                jx, jy = int(cell[j, 0]), int(cell[j, 1])
                h["hm_hp"][b, j, jy, jx] = F32(0.9)
                h["hp_offset"][b, :, jy, jx] = (m[j] - cell[j]).astype(F32)
        o = dict(o, pts=np.where(keep[:, None], pts, SENT), npts=int(keep.sum()))
        rows.append([o])
    return Scene(cls, name, 4, h, rows, c, s, img_w, img_h, cam, **kw)


def rep1_scene(cls, name, B, n_obj, seed, disagree_px, drop_joints=(), **kw):
    """16 points per object from synth.planted_batch (logit heads, apply_sigmoid = 1).  Intended: 8 displacement means
    + the heat-map means of the joints that were planted."""
    hb, truths = synth.planted_batch(B, n_obj=n_obj, seed=seed, disagree_px=disagree_px, drop_joints=drop_joints)
    objs = []
    for t in truths:
        row = []
        for kp, sc in zip(t["kps_map"], t["scale"]):
            pts = np.repeat(kp * 4.0, 2, axis=0)
            for j in drop_joints:
                pts[2 * j + 1] = SENT
            # 2 px and more of disagreement can flip the pose and fail the heat-map mean's gate (a -10000 point)
            calm = disagree_px <= 1.0
            row.append({"pts": pts, "scale": F32(sc), "npts": 16 - len(drop_joints) if calm else None,
                        "want": set(HAS_POSE) if calm else None,
                        "tag": "rep1 disagree %.1f drop %d" % (disagree_px, len(drop_joints)), "loose": True})
        objs.append(row)
    return Scene(cls, name, 1, hb, objs, [256., 256.], 512.0, 512, 512, truths[0]["cam"], apply_sigmoid=1, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# poses
# ---------------------------------------------------------------------------------------------------------------------
def rot(axis, ang):
    ax = np.asarray(axis, np.float64)
    return pnp_ref.rodrigues(ax / np.linalg.norm(ax) * ang)


def rand_rot(rng, lo=0.2, hi=2.6):
    return rot(rng.normal(size=3), rng.uniform(lo, hi))


def project(scale, R, t, cam):
    """The 8 projected vertices of the cuboid the PnP builds from `scale` (pnp_ref.cuboid_vertices, fp32 arithmetic)."""
    return pnp_ref.project(pnp_ref.cuboid_vertices(np.asarray(scale, F32)), R, t, cam)


def kps_pnp(uv, w, h):
    """The nine normalised points the visibility gates read (centroid first)."""
    pp = np.vstack([uv.mean(0, keepdims=True), uv]) / [w, h]
    return pp


def n_outside(uv, w, h):
    pp = kps_pnp(uv, w, h)
    return int(((pp[:, 0] < 0) | (pp[:, 0] > 1) | (pp[:, 1] < 0) | (pp[:, 1] > 1)).sum())


def border_margin(uv, w, h):
    """Pixel distance of the nearest projected coordinate (centroid included) to a frame border."""
    p = np.vstack([uv.mean(0, keepdims=True), uv])
    return float(np.min(np.abs(np.concatenate([p[:, 0], p[:, 0] - w, p[:, 1], p[:, 1] - h]))))


def _obj(pts, scale, want=None, tag="", **extra):
    d = {"pts": np.asarray(pts, np.float64), "scale": F32(scale), "want": want, "tag": tag}
    d.update(extra)
    return d


def _noisy(rng, uv, noise):
    return uv + (rng.normal(0, noise, uv.shape) if noise > 0 else 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# the catalogue
# ---------------------------------------------------------------------------------------------------------------------
def scenes_point_count(seed=11):
    """Exactly 3 .. 8 valid points (rep_mode 4, one object per image) and 16 (rep_mode 1): 3 -> FEW_POINTS, 4 - 5 ->
    EPnP, 6 and more -> DLT + LM.  Consistent and noisy points."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    objs = []
    for n in (3, 4, 5, 6, 7, 8):
        for rep in range(6):
            noise = (0.0, 0.0, 0.5, 1.0, 2.0, 0.0)[rep]
            while True:
                scale = F32(rng.uniform(0.4, 1.6, 3))
                R, tz = rand_rot(rng), rng.uniform(3.0, 6.0)
                t = np.array([rng.uniform(-.2, .2) * tz, rng.uniform(-.2, .2) * tz, tz])
                uv = _noisy(rng, project(scale, R, t, cam), noise)
                if uv.min() < 12 or uv.max() > 500:
                    continue
                keep = np.setdiff1d(np.arange(8), drop_for(rng, scale, n))
                pts = np.full((8, 2), np.nan)
                pts[keep] = uv[keep]
                cells = [tuple(v) for v in np.floor(pts[keep] / 4).astype(int)]
                if len(set(cells)) == n:
                    break
            want = {FEW_POINTS} if n < 4 else set(HAS_POSE)
            objs.append(_obj(pts, scale, want, "n=%d noise %.1f" % (n, noise), noise=noise))
    out = [rep4_scene("point_count", "rep4_3to8", objs)]
    out.append(rep1_scene("point_count", "rep1_16", 3, 4, seed + 1, 1.0))
    out.append(rep1_scene("point_count", "rep1_16_drop", 2, 3, seed + 2, 2.0, drop_joints=(1, 6)))
    return out


MIXED_COUNTS = ((4, 6), (5, 8), (4, 7), (5, 6))


def drop_for(rng, scale, n):
    """8 - n vertex indices to drop, such that 4 kept object points are not coplanar (EPnP needs a volume)."""
    while True:
        keep = np.sort(rng.choice(8, n, replace=False))
        X = pnp_ref.cuboid_vertices(scale)[keep]
        sv = np.linalg.svd(X - X.mean(0), compute_uv=False)
        if n != 4 or sv[-1] >= 1e-2 * sv[0]:
            return np.setdiff1d(np.arange(8), keep)


def mixed_objs(B, K, seed, noise=0.5):
    """B images of K detections whose valid point counts alternate between EPnP (4 - 5) and DLT + LM (6 - 8) along
    every warp's loop (warp w solves detections w, w + 8, ...).  Dropped points sit at x = -6000."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    objs = []
    for b in range(B):
        row = []
        for i in range(K):
            epnp, dlt = MIXED_COUNTS[(i + b) % len(MIXED_COUNTS)]
            n = epnp if ((i // 8) + b) % 2 == 0 else dlt
            scale = F32(rng.uniform(0.4, 1.6, 3))
            R, tz = rand_rot(rng), rng.uniform(3.0, 8.0)
            t = np.array([rng.uniform(-.25, .25) * tz, rng.uniform(-.25, .25) * tz, tz])
            uv = _noisy(rng, project(scale, R, t, cam), noise)
            uv[drop_for(rng, scale, n), 0] = -6000.0
            row.append(_obj(uv, scale, set(HAS_POSE) | {BEHIND}, "mixed n=%d" % n, noise=noise))
        objs.append(row)
    return objs


def scenes_mixed():
    """K = 100 and 128 detections per image at batch 4; `solo` scenes put every detection alone in an image, on the
    same cell of a map of the same size (identical fp32 keypoints, identical fp64 points)."""
    out = []
    for K, seed in ((100, 21), (128, 22)):
        objs = mixed_objs(4, K, seed)
        out.append(rep0_scene("mixed", "mixed_K%d" % K, objs, out_h=64, out_w=64, K=K))
    return out


def solo_scene(sc):
    """Detection i of image b of a rep-0 scene, alone in image b * K + i, at the same cell.  Returns (scene, index)."""
    cells = _cells(sc.out_h, sc.out_w, max(len(r) for r in sc.objs))
    n = sum(len(r) for r in sc.objs)
    h = _blank(n, sc.out_h, sc.out_w)
    index, objs = [], []
    for b, row in enumerate(sc.objs):
        for i, o in enumerate(row):
            k = len(index)
            cx, cy = cells[i]
            for name, v in sc.heads.items():
                h[name][k, :, cy, cx] = v[b, :, cy, cx]
            h["hm"][k, 0, cy, cx] = sc.heads["hm"][b, 0, cy, cx]
            index.append((b, i))
            objs.append([o])
    return Scene(sc.cls, sc.name + "_solo", 0, h, objs, sc.c, sc.s, sc.img_w, sc.img_h, sc.cam,
                 visible_thresh=sc.visible_thresh, opencv_return=sc.opencv_return, K=sc.K), index


def scenes_depth(seed=31):
    """tz from behind the camera through ~0.3 (vertices near or behind z = 0, points leaving the frame) to 100 (a few
    pixels wide); noise-free and 0.5 px."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    row = []
    for tz in (-3.0, -0.8, 0.3, 0.45, 0.6, 0.9, 1.5, 4.0, 15.0, 40.0, 100.0):
        for noise in (0.0, 0.5):
            for _ in range(2):
                while True:
                    scale = F32(rng.uniform(0.5, 1.5, 3))
                    R = rand_rot(rng)
                    t = np.array([rng.uniform(-.1, .1) * abs(tz), rng.uniform(-.1, .1) * abs(tz), tz])
                    z = (pnp_ref.cuboid_vertices(scale) @ R.T + t)[:, 2]
                    if np.abs(z).min() > 0.02:
                        break
                uv = _noisy(rng, project(scale, R, t, cam), noise)
                want = {BEHIND} if tz < 0 and noise == 0 else None
                row.append(_obj(uv, scale, want, "tz %.2f noise %.1f" % (tz, noise), noise=noise))
    return [rep0_scene("depth", "depth", [row])]


def scenes_shape(seed=41):
    """Near-planar (one axis 1e-3), elongated and thin cuboids, and mirrored ones (a negative scale component)."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    shapes = ((1.0, 1.0, 1e-3), (1e-3, 1.0, 1.0), (1.0, 1e-3, 1.0), (6.0, 1.0, 0.3), (0.05, 1.0, 0.05),
              (0.3, 5.0, 0.3), (-1.0, 1.0, 0.6), (1.0, -1.0, 0.6), (0.7, 1.0, -1.2))
    row = []
    for sc in shapes:
        for noise in (0.0, 0.5):
            scale = F32(sc)
            R, tz = rand_rot(rng), rng.uniform(3.0, 5.0)
            t = np.array([rng.uniform(-.2, .2) * tz, rng.uniform(-.2, .2) * tz, tz])
            uv = _noisy(rng, project(scale, R, t, cam), noise)
            row.append(_obj(uv, scale, None, "scale %s noise %.1f" % (sc, noise), noise=noise))
    return [rep0_scene("shape", "shape", [row])]


def scenes_nonfinite(seed=45):
    """scale[1] = 0, denormal, huge or infinite and an overflowing width (vertices inf / NaN or collapsed onto a line);
    points at +inf, -inf and NaN."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    R, t = rand_rot(rng), np.array([0.1, -0.2, 4.0])
    uv = project(F32((1, 1, 1)), R, t, cam)
    row = []
    for sc in ((1.0, 0.0, 1.0), (1.0, 1e-40, 1.0), (1.0, 3e38, 1.0), (1.0, np.inf, 1.0), (3e38, 1e-3, 1.0),
               (1.0, -0.0, 1.0)):
        # scale[1] = 3e38: finite vertices collapsed onto the y axis (x, z ~ 1e-39), a degenerate point set
        row.append(_obj(uv, F32(sc), None, "scale %s" % (sc,), free=sc[1] == 3e38))
    for bad in (np.inf, -np.inf, np.nan):
        pts = uv.copy()
        pts[3, 0] = bad
        row.append(_obj(pts, F32((1, 1, 1)), None, "point %s" % bad, npts=8 if bad != -np.inf else 7))
    return [rep0_scene("nonfinite", "nonfinite", [row])]


def scenes_rotation(seed=51):
    """Rotation angles near pi (w ~ 0) and rotations at the diagonal / trace tie of mat_to_quat: diag(1, -1, -1)
    (pi about x) and pi / 2 about x (R[0][0] == trace) and small perturbations, in the frame the record reports."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    objs = []
    for ocv in (0, 1):
        row = []
        ties = [np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]), np.diag([-1.0, -1.0, 1.0]), rot([1, 0, 0], np.pi / 2),
                rot([0, 1, 0], np.pi / 2)]
        Rs = []
        for Rq in ties:
            for eps in (0.0, 1e-9, 1e-6, 1e-3):
                Rp = rot(rng.normal(size=3), eps) @ Rq
                Rs.append((Rp if ocv else M_GL @ Rp, "tie eps %g" % eps))     # the returned frame holds Rp
        for eps in (0.0, 1e-8, 1e-4, 1e-2):
            Rs.append((rot(rng.normal(size=3), np.pi - eps), "pi - %g" % eps))
        for R, tag in Rs:
            scale = F32(rng.uniform(0.5, 1.5, 3))
            tz = rng.uniform(3.0, 5.0)
            t = np.array([rng.uniform(-.15, .15) * tz, rng.uniform(-.15, .15) * tz, tz])
            row.append(_obj(project(scale, R, t, cam), scale, set(HAS_POSE), tag + " ocv %d" % ocv))
        objs.append(row)
    return [rep0_scene("rotation", "rotation_gl", [objs[0]], visible_thresh=0, opencv_return=0),
            rep0_scene("rotation", "rotation_cv", [objs[1]], visible_thresh=0, opencv_return=1)]


def scenes_noise(seed=61):
    """0, 0.5, 2 and 5 px of noise on 8 points (rep_mode 0) and 16 points (rep_mode 1)."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    row = []
    for noise in (0.0, 0.5, 2.0, 5.0):
        for _ in range(6):
            scale = F32(rng.uniform(0.4, 1.6, 3))
            R, tz = rand_rot(rng), rng.uniform(2.5, 7.0)
            t = np.array([rng.uniform(-.2, .2) * tz, rng.uniform(-.2, .2) * tz, tz])
            row.append(_obj(_noisy(rng, project(scale, R, t, cam), noise), scale, None, "noise %.1f" % noise,
                            noise=noise))
    return [rep0_scene("noise", "noise_rep0", [row]), rep1_scene("noise", "noise_rep1", 2, 4, seed + 1, 5.0)]


def scenes_camera(seed=71):
    """fx != fy with an off-centre principal point, and the 600 x 800 Objectron frame (c = (300, 400), s = 800), both
    with opencv_return 0 and 1."""
    rng = np.random.default_rng(seed)
    out = []
    cams = (("aniso", 512, 512, None, None, np.array([[700.0, 0, 280.5], [0, 540.0, 231.25], [0, 0, 1]])),
            ("objectron", 600, 800, [300.0, 400.0], 800.0, synth.default_camera(600, 800)))
    for name, w, hgt, c, s, cam in cams:
        for ocv in (0, 1):
            row = []
            for noise in (0.0, 0.0, 0.5, 2.0):
                while True:
                    scale = F32(rng.uniform(0.4, 1.6, 3))
                    R, tz = rand_rot(rng), rng.uniform(3.0, 6.0)
                    t = np.array([rng.uniform(-.2, .2) * tz, rng.uniform(-.2, .2) * tz, tz])
                    uv = _noisy(rng, project(scale, R, t, cam), noise)
                    if n_outside(uv, w, hgt) == 0:
                        break
                row.append(_obj(uv, scale, set(HAS_POSE), "%s ocv %d noise %.1f" % (name, ocv, noise), noise=noise))
            out.append(rep0_scene("camera", "%s_ocv%d" % (name, ocv), [row], img_w=w, img_h=hgt, c=c, s=s, cam=cam,
                                  opencv_return=ocv))
    return out


def _gate_pose(rng, cam, w, h, nv_want, margin=0.05):
    while True:
        scale = F32(rng.uniform(0.4, 1.6, 3))
        R, tz = rand_rot(rng), rng.uniform(0.9, 4.0)
        t = np.array([rng.uniform(-.45, .45) * tz, rng.uniform(-.45, .45) * tz, tz])
        if (pnp_ref.cuboid_vertices(scale) @ R.T + t)[:, 2].min() < 0.3:
            continue
        uv = project(scale, R, t, cam)
        pp = kps_pnp(uv, w, h)
        if not (0 < pp[0, 0] < 1 and 0 < pp[0, 1] < 1):
            continue
        if n_outside(uv, w, h) == nv_want and border_margin(uv, w, h) > margin:
            return uv, scale


def _centre_at(rng, cam, w, h, u_target):
    """A pose whose projected centroid sits at u = u_target (bisection along x), all points at least 0.05 px from
    any border."""
    while True:
        scale = F32(rng.uniform(0.4, 1.0, 3))
        R, tz = rand_rot(rng), rng.uniform(4.0, 6.0)
        ty = rng.uniform(-.1, .1) * tz
        lo, hi = -3.0 * tz, 3.0 * tz
        for _ in range(200):
            mid = 0.5 * (lo + hi)
            if project(scale, R, np.array([mid, ty, tz]), cam).mean(0)[0] < u_target:
                lo = mid
            else:
                hi = mid
        uv = project(scale, R, np.array([0.5 * (lo + hi), ty, tz]), cam)
        if abs(uv.mean(0)[0] - u_target) < 1e-6 and border_margin(uv, w, h) > 0.005:
            return uv, scale


def scenes_gates(seed=81):
    """The visibility gates of cuboid_pnp_shell.py: visible_thresh 0 / 3 / 6 with thr - 1 and thr of the nine points
    outside the frame, the centroid 0.01 px inside and outside each border, and points at x or y = -4999 / -5001
    (the `< -5000` cut-off of pnp_collect).  Every projected coordinate keeps >= 0.005 px from the borders."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    w = h = 512
    out = []
    for thr in (0, 3, 6):
        row = []
        for nv in sorted({max(thr - 1, 0), thr, 1}):
            for _ in range(3):
                uv, scale = _gate_pose(rng, cam, w, h, nv)
                want = {INVISIBLE} if thr > 0 and nv >= thr else {OK}
                row.append(_obj(uv, scale, want, "thr %d nv %d" % (thr, nv)))
        out.append(rep0_scene("gates", "visible_%d" % thr, [row], visible_thresh=thr))
    row = []
    for u_target, want in ((0.01, OK), (-0.01, INVISIBLE), (w - 0.01, OK), (w + 0.01, INVISIBLE)):
        uv, scale = _centre_at(rng, cam, w, h, u_target)
        row.append(_obj(uv, scale, {want}, "centre u %.2f" % u_target))
    out.append(rep0_scene("gates", "centre", [row], visible_thresh=0))
    row = []
    R, t = rot([0.3, 1, 0.2], 0.7), np.array([0.2, -0.1, 4.0])
    scale = F32((0.8, 1.0, 1.2))
    uv = project(scale, R, t, cam)
    for j, axis, v in ((0, 0, -4999.0), (1, 0, -5001.0), (2, 1, -4999.0), (3, 1, -5001.0)):
        for k in (1, 3):      # one or three points at the cut-off value
            pts = uv.copy()
            pts[j:j + k, axis] = v
            keep = 8 if v > -5000 else 8 - k
            row.append(_obj(pts, scale, None, "cut %s %g x%d" % ("xy"[axis], v, k), npts=keep))
    out.append(rep0_scene("gates", "cutoff", [row], visible_thresh=0))
    return out


def scenes_degenerate(seed=91):
    """All 8 points equal, and points on one line."""
    rng = np.random.default_rng(seed)
    row = []
    for p in ((256.0, 256.0), (100.25, 400.5)):
        row.append(_obj(np.tile(p, (8, 1)), F32((1, 1, 1)), None, "equal %s" % (p,), free=True))
    for _ in range(3):
        p0, d = rng.uniform(150, 350, 2), rng.normal(size=2)
        row.append(_obj(p0 + np.outer(rng.uniform(-60, 60, 8), d / np.linalg.norm(d)), F32((1, 1, 1)), None, "collinear",
                        free=True))
    row.append(_obj(np.stack([np.linspace(100, 400, 8), np.full(8, 300.0)], 1), F32((1, 1, 1)), None, "horizontal",
                    free=True))
    return [rep0_scene("degenerate", "degenerate", [row])]


# ---------------------------------------------------------------------------------------------------------------------
# the tracker's second PnP
# ---------------------------------------------------------------------------------------------------------------------
TRACK_KEEP_STD, TRACK_DROP_STD = 0.5, 20.0      # px: filter confidence ~0.93 (kept) and 0 (< 0.15: -10000) at [3, 9]


def track_record(uv, keep, scale, score, L):
    """A first-frame pose record whose filtered keypoints are exactly `uv` (fp32) where `keep`, and confidence < 0.15
    elsewhere.  With hps_uncertainty the fusion of a -10000 heat-map mean is the displacement mean itself, with the
    displacement std as its std; the filter starts from that (tracker.py:55-84), so the read-out is the fp32 point and
    the confidence follows from the std alone.  P_STATUS = OK: step 0 only tracks solved detections."""
    r = np.zeros(L.CP_POSE_RECORD, F32)
    r[L.P_SCORE] = score
    ct = np.nanmean(np.where(np.abs(uv) < 1e5, uv, np.nan), 0)
    r[L.P_BBOX:L.P_BBOX + 4] = np.concatenate([ct - 20, ct + 20])
    r[L.P_CT:L.P_CT + 2] = ct
    r[L.P_KPS:L.P_KPS + 16] = uv.reshape(-1)
    r[L.P_KPS_DISP_MEAN:L.P_KPS_DISP_MEAN + 16] = uv.reshape(-1)
    r[L.P_KPS_HM_MEAN:L.P_KPS_HM_MEAN + 16] = SENT
    r[L.P_KPS_HM_STD:L.P_KPS_HM_STD + 16] = SENT
    r[L.P_KPS_DISP_STD:L.P_KPS_DISP_STD + 16] = np.repeat(np.where(keep, TRACK_KEEP_STD, TRACK_DROP_STD), 2)
    r[L.P_OBJ_SCALE:L.P_OBJ_SCALE + 3] = scale
    r[L.P_OBJ_SCALE_UNC:L.P_OBJ_SCALE_UNC + 3] = 0.1
    r[L.P_STATUS] = OK
    r[L.P_NPTS] = 8
    return r


def track_objs(seed=101, per_stream=24, streams=3):
    """Detections for the tracker's second PnP: 3 - 8 surviving keypoints (4 - 7 are the common case there), noise-free
    and noisy, near and far.  Every detection is the first of its track (fresh streams), so the filter read-out is the
    point itself."""
    rng = np.random.default_rng(seed)
    cam = synth.default_camera()
    out = []
    for s in range(streams):
        row = []
        for i in range(per_stream):
            n = (3, 4, 5, 6, 7, 8)[(i + s) % 6]
            noise = (0.0, 0.0, 0.5, 2.0)[(i // 6 + s) % 4]
            tz = (2.5, 4.0, 6.0, 15.0)[(i // 3 + s) % 4]
            scale = F32(rng.uniform(0.4, 1.6, 3))
            R = rand_rot(rng)
            t = np.array([rng.uniform(-.25, .25) * tz, rng.uniform(-.25, .25) * tz, tz])
            uv = _noisy(rng, project(scale, R, t, cam), noise).astype(F32)
            keep = np.ones(8, bool)
            keep[drop_for(rng, scale, n)] = False
            row.append({"pts": uv, "keep": keep, "scale": scale, "npts": n, "noise": noise,
                        "tag": "track n=%d noise %.1f tz %.1f" % (n, noise, tz)})
        out.append(row)
    return out, cam


CLASSES = ("point_count", "mixed", "depth", "shape", "nonfinite", "rotation", "noise", "camera", "gates", "degenerate")
BUILDERS = {"point_count": scenes_point_count, "mixed": scenes_mixed, "depth": scenes_depth, "shape": scenes_shape,
            "nonfinite": scenes_nonfinite, "rotation": scenes_rotation, "noise": scenes_noise, "camera": scenes_camera,
            "gates": scenes_gates, "degenerate": scenes_degenerate}


def catalogue(classes=CLASSES):
    return [sc for c in classes for sc in BUILDERS[c]()]


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's decode of a scene
# ---------------------------------------------------------------------------------------------------------------------
def oracle_decode(sc, b):
    """decode -> post_process -> merge_outputs of image b by the oracle: the list of result dicts, in record order."""
    heads_b = {k: v[b] for k, v in sc.heads.items()}
    prm = sc.oracle_params()
    dets = decode_ref.decode(decode_ref.process_heads(heads_b, sc.apply_sigmoid), prm)
    pp = decode_ref.post_process(dets, sc.c, sc.s, sc.out_h, sc.out_w)
    for i, d in enumerate(pp):
        d["_k"] = i
    return decode_ref.merge_outputs(pp, prm)

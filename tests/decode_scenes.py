"""Adversarial decode inputs: head dicts whose discrete decisions (3x3 equality NMS, top-K, class merge, nearest-peak
argmin, the decode.py gates, soft-NMS) sit on ties and boundaries.

Every generator is deterministic from its arguments and returns {name: [B,C,H,W] fp32}.  The maps are meant for
`apply_sigmoid = 0` (hm / hm_hp are decoded as given), so the kernel and the oracle see the same bits, except where a
function says otherwise.  Positions are integer cells and `reg` / `hp_offset` are zero, so every centre, joint peak,
box edge and distance is an exact fp32 value: the decisions are decided by the rule, not by rounding.
"""
import numpy as np

from oracle import decode_ref

F32 = np.float32
J = 8
# the kinds of map `selection_heads` cycles through, image by image and channel by channel
KINDS = ("quant8", "quant64", "const", "plateau", "neg", "rawmix")


def _zeros(B, C, H, W):
    return np.zeros((B, C, H, W), F32)


def tie_map(kind, H, W, rng):
    """One [H,W] map of the given kind.
    quant8 / quant64: probabilities on the grid k/8 or k/64 (every value a tie class; the top class spans ~1/9 or
        ~1/65 of the map, so the K-th value is a tie of hundreds to thousands of cells);
    const: one value everywhere (every cell survives the NMS, top-K = the first K indices);
    plateau: a low quantised floor, constant rectangles of 0.5 and peaks of 0.75 on every corner and border midpoint
        (the -inf padding of the max-pool);
    neg: a raw all-negative map with exact -0.0 cells that are local maxima, one of them at index 0: every non-maximum
        becomes 0 and outranks every peak, and the -0.0 maxima tie with those zeros;
    rawmix: raw values on the grid k/16 in [-2, 2] (negative and positive peaks) with -0.0 and +0.0 cells."""
    if kind == "quant8":
        return (rng.integers(0, 9, size=(H, W)) / 8.0).astype(F32)
    if kind == "quant64":
        return (rng.integers(0, 65, size=(H, W)) / 64.0).astype(F32)
    if kind == "const":
        return np.full((H, W), 0.25, F32)
    if kind == "plateau":
        m = (rng.integers(0, 17, size=(H, W)) / 64.0).astype(F32)
        for _ in range(max(1, H * W // 400)):
            y0, x0 = rng.integers(0, H), rng.integers(0, W)
            m[y0:y0 + int(rng.integers(2, 9)), x0:x0 + int(rng.integers(2, 9))] = F32(0.5)
        for y, x in ((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (0, W // 2), (H - 1, W // 2), (H // 2, 0),
                     (H // 2, W - 1)):
            m[y, x] = F32(0.75)
        return m
    if kind == "neg":
        m = -(rng.integers(1, 33, size=(H, W)) / 32.0).astype(F32)
        m[0, 0] = F32(-0.0)
        for _ in range(max(1, H * W // 50)):
            m[rng.integers(0, H), rng.integers(0, W)] = F32(-0.0)
        return m
    if kind == "rawmix":
        m = (rng.integers(-32, 33, size=(H, W)) / 16.0).astype(F32)
        for _ in range(max(1, H * W // 50)):
            m[rng.integers(0, H), rng.integers(0, W)] = F32(-0.0) if rng.integers(0, 2) else F32(0.0)
        return m
    raise ValueError(kind)


def selection_heads(B, C, H, W, seed, kinds=KINDS):
    """Tie-heavy hm [B,C,H,W] and hm_hp [B,8,H,W]: image b, class c takes kinds[(b + c) % n] and joint j
    kinds[(b + j + 1) % n].  Classes of the same kind hold equal values across classes.  hps holds integer offsets in
    -3..3 and reg / hp_offset are zero, so the nearest-peak distances are exact and tie often."""
    rng = np.random.default_rng(seed)
    n = len(kinds)
    hm = np.stack([np.stack([tie_map(kinds[(b + c) % n], H, W, rng) for c in range(C)]) for b in range(B)])
    hp = np.stack([np.stack([tie_map(kinds[(b + j + 1) % n], H, W, rng) for j in range(J)]) for b in range(B)])
    return {"hm": hm, "hm_hp": hp, "wh": np.full((B, 2, H, W), 8.0, F32),
            "hps": rng.integers(-3, 4, size=(B, 2 * J, H, W)).astype(F32),
            "reg": _zeros(B, 2, H, W), "hp_offset": _zeros(B, 2, H, W)}


def oracle_selection(heads_b, K, apply_sigmoid=0):
    """(score, ind, cls) of the K candidates the oracle selects for one image."""
    p = decode_ref.process_heads({"hm": heads_b["hm"]}, apply_sigmoid)
    sc, ind, cls, _, _ = decode_ref.topk_classes(decode_ref.nms3x3(p["hm"]), K)
    return sc, ind, cls


# ---------------------------------------------------------------------------------------------------------------------
# Gate boundaries.  A centre at integer cell (cx, cy) with wh = (10, 10) and reg = 0 has the box [cx-5, cx+5] x
# [cy-5, cy+5] and size 10, so 0.3 * size = 3 and 0.5 * size = 5 exactly in fp32.  Each (centre, joint) gets one case:
# the regressed keypoint offset (hps) and the joint peaks (dx, dy, score) relative to the centre.
# ---------------------------------------------------------------------------------------------------------------------
TH = F32(0.1)
GATE_CASES = (
    # name,            regressed,  peaks
    ("equidistant_x",  (0, 1),    ((-2, 1, 0.5), (2, 1, 0.5))),           # equal score: lower index first in top-K order
    ("equidistant_d",  (1, 0),    ((0, -2, 0.4), (3, 1, 0.6))),           # sqrt(5) both; the higher score comes first
    ("on_l",           (-4, 0),   ((-5, 0, 0.5),)),                      # sx == l
    ("on_r",           (4, -1),   ((5, -1, 0.5),)),                      # sx == r
    ("on_t",           (1, -4),   ((1, -5, 0.5),)),                      # sy == t
    ("on_b",           (-1, 4),   ((-1, 5, 0.5),)),                      # sy == bt
    ("at_0.3_size",    (0, 0),    ((3, 0, 0.5),)),                       # distance 3 == 0.3 * size: not bad
    ("at_0.5_size",    (0, 0),    ((3, 4, 0.5),)),                       # distance 5 == 0.5 * size: bad, and ok2 fails
    ("score_0.1",      (1, 1),    ((1, 0, float(TH)),)),                 # exactly 0.1f: masked (s > th fails)
    ("score_above_0.1", (-1, -1), ((-1, 0, float(np.nextafter(TH, F32(1)))),)),
    ("outside",        (0, 0),    ((-6, 0, 0.5),)),                      # sx < l
)


def gate_heads(H=64, W=64, spacing=20, first=10):
    """One image: centres on a grid `spacing` apart with scores 0.9, 0.89, ...; centre i, joint j takes
    GATE_CASES[(i + j) % n].  Returns (heads {name: [1,C,H,W]}, [(centre index, cx, cy, joint, case name)])."""
    hm, hp = _zeros(1, 1, H, W), _zeros(1, J, H, W)
    wh, hps = _zeros(1, 2, H, W), _zeros(1, 2 * J, H, W)
    layout = []
    i = 0
    for cy in range(first, H - 5, spacing):
        for cx in range(first, W - 5, spacing):
            hm[0, 0, cy, cx] = F32(0.9 - 0.01 * i)
            wh[0, :, cy, cx] = 10.0
            for j in range(J):
                name, (rx, ry), peaks = GATE_CASES[(i + j) % len(GATE_CASES)]
                hps[0, 2 * j, cy, cx] = rx
                hps[0, 2 * j + 1, cy, cx] = ry
                for dx, dy, s in peaks:
                    hp[0, j, cy + dy, cx + dx] = F32(s)
                layout.append((i, cx, cy, j, name))
            i += 1
    heads = {"hm": hm, "hm_hp": hp, "wh": wh, "hps": hps, "reg": _zeros(1, 2, H, W),
             "hp_offset": _zeros(1, 2, H, W)}
    return heads, layout


def raw_moment_heads(seed, H=64, W=64, spacing=20, first=10):
    """One image for apply_sigmoid = 2 (opt.mse_loss): hm holds logits, hm_hp raw values.  Centres as in gate_heads
    (logits 2.0, 1.9, ...; 10 x 10 boxes); joint j of every centre has one 0.8 peak at a small integer offset, which
    is also its regressed keypoint (distance 0: every gate holds, the 11 x 11 moment window is read).  Each window
    gets its own raw floor of -0.002 ... -0.1 and, mostly, a second positive cell, so that some windows are fit
    normally with negative cells and others have a non-positive total, a non-positive centroid row or column sum,
    or a centroid outside the window -- the start points fitgaussian rejects.  Returns (heads, [(i, j, px, py)])."""
    rng = np.random.default_rng(seed)
    hm = np.full((1, 1, H, W), -10.0, F32)
    hp = np.full((1, J, H, W), -0.01, F32)
    wh, hps = _zeros(1, 2, H, W), _zeros(1, 2 * J, H, W)
    peaks = []
    i = 0
    for cy in range(first, H - 5, spacing):
        for cx in range(first, W - 5, spacing):
            hm[0, 0, cy, cx] = F32(2.0 - 0.1 * i)
            wh[0, :, cy, cx] = 10.0
            for j in range(J):
                ox, oy = int(rng.integers(-2, 3)), int(rng.integers(-2, 3))
                px, py = cx + ox, cy + oy
                hps[0, 2 * j:2 * j + 2, cy, cx] = (ox, oy)
                win = hp[0, j, py - 5:py + 6, px - 5:px + 6]
                win[...] = -F32(rng.choice([0.002, 0.02, 0.05, 0.1]))
                if rng.random() < 0.8:
                    dy, dx = rng.integers(-5, 6, size=2)
                    if max(abs(dy), abs(dx)) >= 2:
                        win[5 + dy, 5 + dx] = F32(rng.uniform(0.3, 0.7))
                win[5, 5] = F32(0.8)
                peaks.append((i, j, px, py))
            i += 1
    heads = {"hm": hm, "hm_hp": hp, "wh": wh, "hps": hps, "reg": _zeros(1, 2, H, W), "hp_offset": _zeros(1, 2, H, W)}
    return heads, peaks


def moment_window(hp_map, px, py, ran=5):
    """The 11 x 11 window decode.py:226-233 reads around the joint peak (px, py) of one [H,W] map (zero padded)."""
    H, W = hp_map.shape
    big = np.zeros((H + 2 * ran, W + 2 * ran))
    big[ran:H + ran, ran:W + ran] = hp_map
    return big[py:py + 2 * ran + 1, px:px + 2 * ran + 1]


def soft_nms_heads(H=64, W=64):
    """One image of centres for the soft-NMS: equal scores everywhere it matters.
    - a two-cell plateau of 0.8 whose reg makes both boxes identical (the second decays by exp(-2) and is dropped);
    - two 0.7 centres six cells apart with 12 x 12 boxes (IoU 0.37: the later one decays to 0.53, below the 0.6s,
      and survives);
    - three 0.6 centres far apart (no overlap: the survivors keep index order);
    - a 0.5 / 0.5 pair whose boxes share one pixel column (iw == 1 in the +1 convention)."""
    hm, wh, reg = _zeros(1, 1, H, W), _zeros(1, 2, H, W), _zeros(1, 2, H, W)

    def put(x, y, s, w, h, rx=0.0, ry=0.0):
        hm[0, 0, y, x] = F32(s)
        wh[0, :, y, x] = (w, h)
        reg[0, :, y, x] = (rx, ry)
    put(10, 10, 0.8, 8, 8, 0.5, 0.0)
    put(11, 10, 0.8, 8, 8, -0.5, 0.0)
    put(30, 10, 0.7, 12, 12)
    put(36, 10, 0.7, 12, 12)
    put(54, 10, 0.6, 6, 6)
    put(10, 40, 0.6, 6, 6)
    put(50, 40, 0.6, 6, 6)
    put(24, 56, 0.5, 4, 4)
    put(28, 56, 0.5, 4, 4)
    return {"hm": hm, "hm_hp": _zeros(1, J, H, W), "wh": wh, "hps": _zeros(1, 2 * J, H, W), "reg": reg,
            "hp_offset": _zeros(1, 2, H, W)}


def oracle_survivors(heads_b, prm, c, s, apply_sigmoid=0):
    """decode -> post_process -> merge_outputs for one image, without the PnP: [(candidate k, score)] in order."""
    dets = decode_ref.decode(decode_ref.process_heads(heads_b, apply_sigmoid), prm)
    H, W = heads_b["hm"].shape[1:]
    pp = decode_ref.post_process(dets, c, s, H, W)
    for i, d in enumerate(pp):
        d["_k"] = i
    return [(d["_k"], d["score"]) for d in decode_ref.merge_outputs(pp, prm)], dets


def sigmoid_sweep_heads(B=64, H=64, W=64, K=128, lo=-20.0, hi=20.0):
    """B one-channel logit maps, each with K isolated single-cell peaks on even cells and a -60 floor; the B * K peak
    logits sweep [lo, hi].  The K candidates of every image are exactly its peaks (sigmoid(-60) is below any of them),
    so the decoded centre scores are the kernel's sigmoid of known logits."""
    logits = np.linspace(lo, hi, B * K).astype(F32)
    hm = np.full((B, 1, H, W), -60.0, F32)
    cells = [(y, x) for y in range(0, H, 2) for x in range(0, W, 2)]
    step = len(cells) // K
    for b in range(B):
        for k in range(K):
            y, x = cells[k * step]
            hm[b, 0, y, x] = logits[b * K + k]
    z = lambda c: _zeros(B, c, H, W)
    return {"hm": hm, "hm_hp": np.full((B, J, H, W), -60.0, F32), "wh": np.full((B, 2, H, W), 4.0, F32),
            "hps": z(2 * J), "reg": z(2), "hp_offset": z(2)}


def ulp_distance(a, b):
    """Elementwise distance in units in the last place of two fp32 arrays of the same sign (int bit difference)."""
    ai = np.asarray(a, F32).view(np.int32).astype(np.int64)
    bi = np.asarray(b, F32).view(np.int32).astype(np.int64)
    return np.abs(ai - bi)

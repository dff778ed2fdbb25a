"""Crafted deformable-convolution sampling fields and a mirror of the kernels' discrete sampling decisions.

Gaussian offsets almost never land where a DCN kernel makes a discrete choice: on an integer (lh = 0, a corner of weight
exactly 0), exactly on the bounds -1 and H of the strict inside test, just inside them, on a half-integer next to the
border (one corner outside the image), or on the staged-slab boundary of dcn_tma.cu (halo 8 around an 8 x 16 patch:
an integer row offset above +6 or below -7 moves a corner out of the slab and the sample onto the global-memory path,
whose record packs the image row and column in 7 bits each).  `crafted_offsets` aims every (position, tap) at such a
target, row and column chosen independently; every target is a short dyadic number, so the fp32 sum base + offset the
kernels compute lands exactly on it.

  crafted_offsets / crafted_masks   the fields (masks as values for the stand-alone op, as logits for the plan)
  classify                          per-class counts of a field, by the decisions of coef_row (dcn_tma.cu)
  sample_ref                        a compact fp64 restatement of the op; the "trunc" and "clamp" variants are the two
                                    mistakes the fields must expose (truncation instead of floor in (-1, 0), border
                                    corners replicated with their bilinear weight instead of zeroed)
"""
import numpy as np
import torch
import torch.nn.functional as F

PATCH_H, PATCH_W, HALO = 8, 16, 8                 # dcn_tma.cu DT_PH, DT_PW, DT_HALO
SLAB_H, SLAB_W = PATCH_H + 2 * HALO, PATCH_W + 2 * HALO
SLAB_STEPS = (6.0, 6.5, 7.0, 7.5, 8.0, 9.0)       # offsets around the in-slab / global threshold, both signs
N_CLASSES = 8
CLASS_KEYS = ("samples", "outside", "dead_top", "dead_bottom", "dead_left", "dead_right", "lh0", "lw0", "slab", "global",
              "global127")

# (B, C, H, W, Co) of the stand-alone launches (tests/test_gpu_dcn_edges.py).  dcn_tma: one patch (the whole halo
# outside the image), coordinates up to 127 in both 7-bit record fields, H = 128 with one patch column, a partial N
# tile (27 of 32 columns), 16 slabs on two tiles.  The gather kernel: H > 128, W > 128 with odd H, C and Co padded.
TMA_SHAPES = [(1, 16, 8, 16, 16), (1, 32, 128, 128, 64), (2, 64, 16, 128, 32), (1, 48, 128, 16, 128),
              (3, 32, 24, 48, 27), (1, 256, 16, 16, 64)]
GATHER_SHAPES = [(1, 32, 136, 24, 64), (2, 16, 9, 150, 16), (1, 6, 10, 7, 5)]
# the DCN maps of the dla_34 plans stepped on the GPU (256 x 256 and 512 x 512 inputs)
PLAN_MAPS = [(8, 8), (16, 16), (32, 32), (64, 64), (128, 128)]


def _targets(rng, base, extent):
    """Target coordinates along one axis (extent = H or W) for samples whose integer base coordinate is `base`."""
    n = base.size
    cls = rng.integers(0, N_CLASSES, n)
    side = rng.integers(0, 2, n)
    k = rng.integers(1, 13, n).astype(np.float64)
    t = np.select(
        [cls == 0, cls == 1, cls == 2, cls == 3, cls == 4, cls == 5, cls == 6],
        [rng.integers(-2, extent + 2, n).astype(np.float64),                        # integers in [-2, extent + 1]
         np.where(side == 0, -1.0, float(extent)),                                  # exactly on the bounds
         np.where(side == 0, -1.0 + 2.0 ** -k, extent - 2.0 ** -k),                 # just inside them
         np.where(rng.integers(0, 3, n) == 0, np.where(side == 0, -0.5, extent - 0.5),
                  rng.integers(-2, extent + 1, n) + 0.5),                           # half-integers, -0.5 and extent - 0.5
         base + rng.choice(SLAB_STEPS, n) * np.where(side == 0, -1.0, 1.0),         # the slab thresholds
         base.astype(np.float64),                                                   # zero offset
         base + np.round(rng.uniform(-2.5, 2.5, n) * 2 ** 14) / 2 ** 14],           # continuous, near the base
        base + np.round(rng.uniform(-40.0, 40.0, n) * 2 ** 10) / 2 ** 10)           # far: tens of pixels out
    return t


def crafted_offsets(B, H, W, seed):
    """[B, 18, H, W] fp32 offsets (channel 2k: row, 2k + 1: column of tap k) whose fp32 positions are the targets."""
    rng = np.random.default_rng(seed)
    off = np.empty((B, 18, H, W), np.float64)
    ys = np.arange(H).reshape(1, H, 1)
    xs = np.arange(W).reshape(1, 1, W)
    for k in range(9):
        by = np.broadcast_to(ys - 1 + k // 3, (B, H, W)).ravel()
        bx = np.broadcast_to(xs - 1 + k % 3, (B, H, W)).ravel()
        off[:, 2 * k] = (_targets(rng, by, H) - by).reshape(B, H, W)
        off[:, 2 * k + 1] = (_targets(rng, bx, W) - bx).reshape(B, H, W)
    out = off.astype(np.float32)
    assert np.array_equal(out.astype(np.float64), off)
    return torch.from_numpy(out)


def crafted_masks(B, H, W, seed, logits=False):
    """[B, 9, H, W] fp32 masks: 0, 1, 0.5 and uniform values, or (logits=True, for the plan, which takes the sigmoid in
    the kernel) the logits -30, 0, +30 and normal values."""
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, 4, (B, 9, H, W))
    if logits:
        m = np.choose(cls, [-30.0, 0.0, 30.0, rng.normal(0.0, 3.0, cls.shape)])
    else:
        m = np.choose(cls, [0.0, 1.0, 0.5, rng.uniform(0.0, 1.0, cls.shape)])
    return torch.from_numpy(m.astype(np.float32))


def dcn_tma_shape(H, W):
    """Whether dcn_tma.cu takes a map of H x W (dcn_tma_supported; the channel conditions aside)."""
    return H <= 128 and W <= 128 and H % PATCH_H == 0 and W % PATCH_W == 0


def classify(off, H, W):
    """Counts of the sampling classes of `off` ([B, 18, H, W] fp32) on an H x W map, by the decisions every DCN kernel
    makes (coef_row, dcn_tma.cu): the strict (-1, H) x (-1, W) inside test, floor for the low corner, per-corner bounds;
    for a dcn_tma map also whether the clamped corners lie in the tile's staged slab (else the global path) and global
    samples with a corner on row or column 127 (the largest value of the 7-bit record fields)."""
    off = off.detach().cpu().numpy().astype(np.float32) if torch.is_tensor(off) else np.asarray(off, np.float32)
    B = off.shape[0]
    oy = np.arange(H).reshape(1, H, 1)
    ox = np.arange(W).reshape(1, 1, W)
    ys = np.broadcast_to(oy // PATCH_H * PATCH_H - HALO, (B, H, W))
    xs = np.broadcast_to(ox // PATCH_W * PATCH_W - HALO, (B, H, W))
    n = dict.fromkeys(CLASS_KEYS, 0)
    for k in range(9):
        h = np.float32(oy - 1 + k // 3) + off[:, 2 * k]           # fp32 sums, as the kernels form them
        w = np.float32(ox - 1 + k % 3) + off[:, 2 * k + 1]
        live = (h > -1) & (w > -1) & (h < H) & (w < W)
        hlo, wlo = np.floor(h), np.floor(w)
        t_ok, b_ok, l_ok, r_ok = hlo >= 0, hlo + 1 <= H - 1, wlo >= 0, wlo + 1 <= W - 1
        n["samples"] += h.size
        n["outside"] += int((~live).sum())
        for key, ok in (("dead_top", t_ok), ("dead_bottom", b_ok), ("dead_left", l_ok), ("dead_right", r_ok)):
            n[key] += int((live & ~ok).sum())
        n["lh0"] += int((live & (h == hlo)).sum())
        n["lw0"] += int((live & (w == wlo)).sum())
        if dcn_tma_shape(H, W):
            hl, hb = np.where(t_ok, hlo, 0), np.where(b_ok, hlo + 1, H - 1)
            wl, wr = np.where(l_ok, wlo, 0), np.where(r_ok, wlo + 1, W - 1)
            in_slab = (hl >= ys) & (hb < ys + SLAB_H) & (wl >= xs) & (wr < xs + SLAB_W)
            glob = live & ~in_slab
            n["slab"] += int((live & in_slab).sum())
            n["global"] += int(glob.sum())
            n["global127"] += int((glob & ((hl == 127) | (hb == 127) | (wl == 127) | (wr == 127))).sum())
    return n


def required_classes(H, W):
    """The classes a crafted field must populate on an H x W map: the slab classes on dcn_tma maps only, the global path
    where some tile's slab does not hold the whole image (H > 16 or W > 16: the clamped corners of a sample are always
    inside the image), row / column 127 on maps that have one."""
    need = ["outside", "dead_top", "dead_bottom", "dead_left", "dead_right", "lh0", "lw0"]
    if dcn_tma_shape(H, W):
        need.append("slab")
        if H > PATCH_H + HALO or W > PATCH_W:
            need.append("global")
            if max(H, W) == 128:
                need.append("global127")
    return need


def sample_ref(x, off, mask, w, b, variant="reference"):
    """Modulated deformable 3x3 conv (stride 1, pad 1) in the dtype of x, sampling at exactly the positions
    base + off.  The image is padded by one pixel, which holds every corner of a sample inside (-1, H) x (-1, W):
    zeros for the reference (a corner outside the image weighs 0); variant "clamp" pads by replication (border corners
    keep their bilinear weight), variant "trunc" takes the low corner by truncation toward zero instead of floor."""
    assert variant in ("reference", "trunc", "clamp")
    B, C, H, W = x.shape
    Co = w.shape[0]
    xp = F.pad(x, (1, 1, 1, 1), mode="replicate" if variant == "clamp" else "constant").reshape(B, C, -1)
    ys = torch.arange(H, dtype=x.dtype, device=x.device).view(1, H, 1)
    xs = torch.arange(W, dtype=x.dtype, device=x.device).view(1, 1, W)
    low = torch.trunc if variant == "trunc" else torch.floor
    cols = []
    for k in range(9):
        h = ys - 1 + k // 3 + off[:, 2 * k]
        v = xs - 1 + k % 3 + off[:, 2 * k + 1]
        inside = (h > -1) & (v > -1) & (h < H) & (v < W)
        h0, v0 = low(h), low(v)
        lh, lw = h - h0, v - v0
        h0 = h0.clamp(-1, H - 1).long() + 1          # padded coordinates of the low corner (clamped where unused)
        v0 = v0.clamp(-1, W - 1).long() + 1
        acc = 0
        for dy, dx, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
            idx = ((h0 + dy) * (W + 2) + v0 + dx).view(B, 1, H * W).expand(B, C, H * W)
            acc = acc + wt.unsqueeze(1) * torch.gather(xp, 2, idx).view(B, C, H, W)
        cols.append(acc * (mask[:, k] * inside).unsqueeze(1))
    col = torch.stack(cols, 2)                          # [B, C, 9, H, W]
    return torch.einsum("ock,bckhw->bohw", w.reshape(Co, C, 9), col) + b.view(1, Co, 1, 1)

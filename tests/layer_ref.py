"""fp64 reference and rounding-error magnitude of one op of the plan's schedule (tests/test_gpu_plan_layers.py).

For an op described by `cp_plan_op_desc` and the tensors it read, `op_ref` returns, per output, the op evaluated in
float64 (`ref`) and the same op evaluated on absolute values (`S`).  Every floating-point operation of a kernel rounds
its result with a relative error of at most the unit roundoff of its arithmetic, so |got - ref| <= c * u * S holds
element by element for a correct kernel, with c set by the summation structure, not by the data.  The per-op score

    r = max over elements of |got - ref| / (S + eps),   eps = EPS_REL * max(S)

is therefore comparable across ops and shapes: it does not let an error in a small output hide behind a large one
(as an error relative to max|ref| would), and a single launch has no deformable amplification, so each precision
gets one ceiling (tests/util.py, LAYER_CEIL).

The functions work on any device and take plain tensors; `ActReader` turns cp_act_desc records into tensors.
"""
import torch
import torch.nn.functional as F

from oracle.net_ref import dcn_v2_forward_ref

EPS_REL = 1e-12


class ActReader(object):
    """NCHW float64 views of cp_act_desc records for the frames `frames` of a batch.
    arena: flat tensor (the plan's arena or an fp64 copy), ext: the four external NCHW inputs (or None)."""

    def __init__(self, arena, ext, frames, max_batch):
        self.arena, self.ext, self.frames, self.max_batch = arena, ext, list(frames), max_batch

    def view(self, a):
        """[max_batch, C, H, W] view of the arena (no copy, arena dtype)."""
        n = self.max_batch * a["H"] * a["W"] * a["stride"]
        t = self.arena[a["off"]:a["off"] + n].view(self.max_batch, a["H"], a["W"], a["stride"])
        return t[..., :a["C"]].permute(0, 3, 1, 2)

    def get(self, a):
        if a["ext"] >= 0:
            return self.ext[a["ext"]][self.frames].double()
        return self.view(a)[self.frames].double()

    def put(self, a, value):
        """Write `value` [len(frames), C, H, W] into the arena slots of `a` (chained evaluation)."""
        self.view(a)[self.frames] = value.to(self.arena.dtype)


def conv_weight(w, w_ld, kh, Cin, Cout):
    """Packed [Kpad][w_ld] matrix (row k = (ky*kh + kx)*Cin + ci) -> OIHW float64."""
    m = w.reshape(-1, w_ld)[:kh * kh * Cin, :Cout].double()
    return m.reshape(kh, kh, Cin, Cout).permute(3, 2, 0, 1).contiguous()


def conv_ref(x, W, b, stride, pad, relu, res=None, res_after_relu=False):
    """(ref, S) of out = [relu](conv(x, W) + b [+ res]) or relu(conv(x, W) + b) + res."""
    ref = F.conv2d(x, W, b, stride, pad)
    S = F.conv2d(x.abs(), W.abs(), b.abs(), stride, pad)
    if res is not None:
        S = S + res.abs()
        if not res_after_relu:
            ref = ref + res
    if relu:
        ref = ref.clamp_min(0)
    if res is not None and res_after_relu:
        ref = ref + res
    return ref, S


def fp32_positions(off):
    """Offsets whose sampling positions y - 1 + i + dy, x - 1 + j + dx are the fp32 values every DCN kernel computes
    (igemm_fp32.cu, igemm_umma.cu, dcn_tma.cu, like the reference's own float im2col): one fp32 rounding of the sum.
    The position is part of the op's definition; with offsets of tens of pixels its rounding moves a sample by up to
    2^-24 * |position| pixels, which at a steep corner difference is far more than the sampling arithmetic's rounding,
    so the fp64 reference samples at exactly these positions."""
    B, _, H, W = off.shape
    ys = torch.arange(H, dtype=off.dtype, device=off.device).view(1, H, 1)
    xs = torch.arange(W, dtype=off.dtype, device=off.device).view(1, 1, W)
    out = off.clone()
    for k in range(9):
        by, bx = ys - 1 + k // 3, xs - 1 + k % 3
        out[:, 2 * k] = (by + off[:, 2 * k]).float().double() - by
        out[:, 2 * k + 1] = (bx + off[:, 2 * k + 1]).float().double() - bx
    return out


def dcn_ref(x, om, W, b, relu, fp32_pos=True):
    """(ref, S) of the plan's deformable conv: offsets = om[:, :18], mask = sigmoid(om[:, 18:27]) taken in the kernel,
    samples at the fp32 positions (fp32_positions; fp32_pos=False: at the exact fp64 positions, as the fp64 oracle
    network does)."""
    off = fp32_positions(om[:, :18]) if fp32_pos else om[:, :18]
    mask = torch.sigmoid(om[:, 18:27])
    ref = dcn_v2_forward_ref(x, off, mask, W, b)
    S = dcn_v2_forward_ref(x.abs(), off, mask, W.abs(), b.abs())
    if relu:
        ref = ref.clamp_min(0)
    return ref, S


def fused_head_ref(hidden, S_hidden, W1, b1):
    """(ref, S) of a per-head 1x1 conv that reads relu(conv3x3) = `hidden` inside its parent's epilogue: the error the
    hidden value carries (<= r * S_hidden) and the 1x1's own rounding both scale with |W1| (S_hidden + |hidden|)."""
    ref = F.conv2d(hidden, W1, b1)
    S = F.conv2d(S_hidden + hidden.abs(), W1.abs(), b1.abs())
    return ref, S


def maxpool_ref(x):
    ref = F.max_pool2d(x, 2, 2)
    return ref, ref.abs()


def upadd_ref(x, w_kkc, f, skip):
    """Depthwise ConvTranspose2d(C, C, 2f, stride f, pad f/2) with weights packed [ky][kx][C], plus the skip."""
    C = x.shape[1]
    k = 2 * f
    w = w_kkc.reshape(k, k, C).permute(2, 0, 1).unsqueeze(1).double()
    ref = F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=C)
    S = F.conv_transpose2d(x.abs(), w.abs(), None, stride=f, padding=f // 2, groups=C)
    if skip is not None:
        ref = ref + skip
        S = S + skip.abs()
    return ref, S


def gn_relu_ref(x, gamma, beta, groups, eps=1e-5):
    """GroupNorm (fp64 statistics) + ReLU; S = (|x| + |mean|) rstd |gamma| + |beta| (the fp32 normalisation)."""
    Fn, C, H, W = x.shape
    g = x.reshape(Fn, groups, -1)
    mean = g.mean(-1, keepdim=True)
    var = g.var(-1, unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    gamma, beta = gamma.double().view(1, C, 1, 1), beta.double().view(1, C, 1, 1)
    xn = ((g - mean) * rstd).reshape(Fn, C, H, W)
    ref = (xn * gamma + beta).clamp_min(0)
    mean_c = mean.expand(Fn, groups, C // groups).reshape(Fn, C, 1, 1)
    rstd_c = rstd.expand(Fn, groups, C // groups).reshape(Fn, C, 1, 1)
    S = (x.abs() + mean_c.abs()) * rstd_c * gamma.abs() + beta.abs()
    return ref, S


def gru_ref(gx, gh, hprev):
    """convGRU gate (convGRU.py:32-39); gh / hprev None at the first step (h = 0).  S is the first-order magnitude of
    the fp32 evaluation: each gate g = act(a) contributes |g| + |act'(a)| (|a-inputs|)."""
    C = gx.shape[1] // 3
    xr, xz, xn = gx[:, :C], gx[:, C:2 * C], gx[:, 2 * C:]
    if gh is None:
        hr = hz = hn = h = torch.zeros_like(xr)
    else:
        hr, hz, hn, h = gh[:, :C], gh[:, C:2 * C], gh[:, 2 * C:], hprev
    r = torch.sigmoid(xr + hr)
    z = torch.sigmoid(xz + hz)
    n = torch.tanh(xn + r * hn)
    ref = (1 - z) * n + z * h
    Sr = r + r * (1 - r) * (xr.abs() + hr.abs())
    Sz = z + z * (1 - z) * (xz.abs() + hz.abs())
    Sa = xn.abs() + r * hn.abs() + Sr * hn.abs()
    Sn = n.abs() + (1 - n * n) * Sa
    S = (1 - z) * Sn + Sz * (n.abs() + h.abs()) + z * h.abs() + ref.abs()
    return ref, S


def op_ref(d, rd, fetch, descs=None, fp32_pos=True):
    """fp64 (ref, S) of every output of op `d` (an Engine.op_descs() record) from the tensors it reads through `rd`
    (ActReader).  fetch(ptr, n) -> tensor of n floats at device pointer ptr.  Returns a list of (target, ref, S) with
    target ("act", act_desc) or ("head", index).  A fused-heads op yields one entry per head (its hidden tile is
    never stored); `descs` (all op records) supplies the children.  fp32_pos: see dcn_ref."""
    fam = d["family"]
    kind = d["kind"]
    if d["fused_away"]:
        return []
    if kind in (0, 1, 2):
        W = conv_weight(fetch(d["w"], d["Kpad"] * d["w_ld"]), d["w_ld"], d["kh"], d["Cin"], d["Cout"])
        b = fetch(d["bias"], d["Cout"]).double()
        if kind == 2:
            ref, S = dcn_ref(rd.get(d["src"][0]), rd.get(d["om"]), W, b, bool(d["relu"]), fp32_pos)
        else:
            x = torch.cat([rd.get(a) for a in d["src"][:d["nsrc"]]], 1)
            res = rd.get(d["res"]) if d["has_res"] else None
            ref, S = conv_ref(x, W, b, d["stride"], d["pad"], bool(d["relu"]), res, bool(d["res_after_relu"]))
        if d["fuse_heads"]:
            out = []
            hc = d["Cout"] // len(d["children"])
            for gi, ci in enumerate(d["children"]):
                c = descs[ci]
                W1 = conv_weight(fetch(c["w"], c["Kpad"] * c["w_ld"]), c["w_ld"], 1, c["Cin"], c["Cout"])
                b1 = fetch(c["bias"], c["Cout"]).double()
                sl = slice(gi * hc, (gi + 1) * hc)
                hr, hs = fused_head_ref(ref[:, sl], S[:, sl], W1, b1)
                out.append((("head", c["out_head"]), hr, hs))
            return out
        if d["out_head"] >= 0:
            return [(("head", d["out_head"]), ref, S)]
        return [(("act", d["out"]), ref, S)]
    if kind == 10:
        ref, S = maxpool_ref(rd.get(d["src"][0]))
    elif kind == 20:
        C = d["src"][0]["C"]
        w = fetch(d["up_w"], 4 * d["f"] * d["f"] * C)
        ref, S = upadd_ref(rd.get(d["src"][0]), w, d["f"], rd.get(d["skip"]) if d["has_skip"] else None)
    elif kind == 30:
        C = d["out"]["C"]
        ref, S = gn_relu_ref(rd.get(d["out"]), fetch(d["gamma"], C), fetch(d["beta"], C), d["groups"])
    elif kind == 40:
        first = bool(d["first_step"])
        ref, S = gru_ref(rd.get(d["gx"]), None if first else rd.get(d["gh"]), None if first else rd.get(d["gprev"]))
    else:
        raise ValueError("unknown op kind %d (family %d)" % (kind, fam))
    return [(("act", d["out"]), ref, S)]


def score(got, ref, S):
    """r = max |got - ref| / (S + EPS_REL max S) over every element (got / ref / S of the same shape)."""
    got = got.double()
    eps = EPS_REL * float(S.max()) if S.numel() else 0.0
    if not torch.isfinite(got).all():
        return float("inf")
    return float(((got - ref).abs() / (S + eps + 1e-300)).max())

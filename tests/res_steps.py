"""Per-op fp64 references of the ResNet schedule and the stepping loop that scores them (tests/test_gpu_res.py).

The ResNet plan has two op kinds the DLA schedule does not: the 4x4/2/1 transposed conv (kind 3, four packed phase
weight blocks) and the 3x3/2 max-pool with an optional residual (kind 11).  `op_ref` evaluates those here and hands
every other kind to tests/layer_ref.py, so a ResNet op is scored with the same metric r = max |got - ref| / S and the
same LAYER_CEIL as the DLA ops of tests/test_gpu_plan_layers.py.
"""
import torch
import torch.nn.functional as F

from centerpose_b200 import _lib
from tests import layer_ref
from tests.plan_steps import _ceiling, _engine, _fetch, _heads, _inputs


def maxpool3_ref(x, res=None, fp32_add=True):
    """MaxPool2d(3, 2, 1) [+ res]: the max is exact; the sum is the one fp32 addition the kernel makes (fp32_add) or the
    exact sum (chained fp64 evaluation)."""
    ref = F.max_pool2d(x, 3, 2, 1)
    if res is not None:
        ref = (res.float() + ref.float()).double() if fp32_add else res + ref
    return ref, ref.abs()


def deconv_weight(w, w_ld, Kpad, Cin, Cout):
    """The four packed phase blocks [4][Kpad][w_ld] of a kind-3 op -> ConvTranspose2d weight [Cin][Cout][4][4] float64
    (phase py * 2 + px, row (2a + b) * Cin + ci holds tap ky = 1 + 2a (py 0) or 2a (py 1), kx likewise)."""
    m = w.reshape(4, Kpad, w_ld).double()
    W = torch.zeros(Cin, Cout, 4, 4, dtype=torch.float64, device=w.device)
    for ph in range(4):
        py, px = ph >> 1, ph & 1
        for a in range(2):
            for b in range(2):
                ky, kx = (2 * a if py else 1 + 2 * a), (2 * b if px else 1 + 2 * b)
                W[:, :, ky, kx] = m[ph, (2 * a + b) * Cin:(2 * a + b + 1) * Cin, :Cout]
    return W


def deconv_ref(x, W, b, relu):
    """(ref, S) of [relu](ConvTranspose2d(x, W, k 4, stride 2, pad 1) + b)."""
    ref = F.conv_transpose2d(x, W, b, stride=2, padding=1)
    S = F.conv_transpose2d(x.abs(), W.abs(), b.abs(), stride=2, padding=1)
    if relu:
        ref = ref.clamp_min(0)
    return ref, S


def op_ref(d, rd, fetch, descs=None, fp32_pos=True):
    """layer_ref.op_ref, with the kinds 3 and 11 of the ResNet schedule.  fp32_pos=False (chained fp64 evaluation) also
    takes the max-pool's residual sum exactly."""
    if d["kind"] == 3:
        W = deconv_weight(fetch(d["w"], 4 * d["Kpad"] * d["w_ld"]), d["w_ld"], d["Kpad"], d["Cin"], d["Cout"])
        ref, S = deconv_ref(rd.get(d["src"][0]), W, fetch(d["bias"], d["Cout"]).double(), bool(d["relu"]))
        return [(("act", d["out"]), ref, S)]
    if d["kind"] == 11:
        ref, S = maxpool3_ref(rd.get(d["src"][0]), rd.get(d["res"]) if d["has_res"] else None, fp32_pos)
        return [(("act", d["out"]), ref, S)]
    return layer_ref.op_ref(d, rd, fetch, descs, fp32_pos)


def step_and_score(arch, trk, H, W, batch, max_batch, prec):
    """Run the schedule op by op (cp_plan_run_ops), each op teacher-forced from the arena the plan produced, and score it
    against op_ref: one record per launched op (config, prec, name, kind, family, x3, stride, Cin, has_res, BN, r and
    its LAYER_CEIL key).  Max-pools must be bit-exact."""
    eng, _, _ = _engine(arch, trk, H, W, max_batch, prec)
    descs = eng.op_descs()
    x, ext = _inputs(eng, batch)
    heads = _heads(eng, batch)
    rd = layer_ref.ActReader(eng.arena(), ext, sorted({0, batch - 1}), max_batch)
    config = "%s%s %dx%d b%d/%d %s" % (arch, "+trk" if trk else "", H, W, batch, max_batch, prec)
    recs = []
    for i, d in enumerate(descs):
        with torch.no_grad():
            want = op_ref(d, rd, _fetch, descs)
        li = eng.run_ops(x, i, i + 1, heads, *ext[1:])[0]
        torch.cuda.synchronize()
        if d["fused_away"]:
            assert li["family"] == _lib.FAM_NONE
            continue
        assert li["family"] == d["family"], (d["name"], li, d["family"])
        r = 0.0
        for (kind, tgt), ref, S in want:
            got = rd.get(tgt) if kind == "act" else heads[eng.head_names[tgt]][rd.frames].double()
            if d["family"] == _lib.FAM_MAXPOOL:
                r = max(r, 0.0 if torch.equal(got, ref) else float("inf"))
            else:
                r = max(r, layer_ref.score(got, ref, S))
        recs.append(dict(config=config, prec=prec, batch=batch, index=i, name=d["name"], kind=d["kind"],
                         family=d["family"], x3=d["x3"], stride=d["stride"], Cin=d["Cin"], has_res=d["has_res"],
                         BN=li["BN"], ksplit=li["ksplit"], r=r, ceil=_ceiling(d, prec)))
    eng.close()
    return recs


def chained_heads(eng, ext, B):
    """The fp64 op references chained through the ResNet schedule (no teacher forcing, an fp64 arena) from the external
    inputs `ext`: {head name: [B,C,H/4,W/4] float64} (plan_steps.chained_heads with op_ref above)."""
    arena64 = torch.zeros(eng.arena().numel(), dtype=torch.float64, device="cuda")
    rd = layer_ref.ActReader(arena64, ext, range(B), B)
    descs = eng.op_descs()
    heads = {}
    with torch.no_grad():
        for d in descs:
            for (kind, tgt), ref, _ in op_ref(d, rd, _fetch, descs, fp32_pos=False):
                if kind == "act":
                    rd.put(tgt, ref)
                else:
                    heads[eng.head_names[tgt]] = ref
    return heads

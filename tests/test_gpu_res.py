"""The ResNet backbones (res_18 .. res_152, msra_resnet.py) on the GPU.

  * heads against the reference's golden tensors and the fp64 oracle (oracle/net_ref_res.py), at the Stage-B bar of
    tests/test_gpu_net.py, in fp32 and tf32x3; the tf32 / bf16 drift is printed;
  * every launch of the schedule teacher-forced against its fp64 reference (tests/res_steps.py) under LAYER_CEIL, with
    the coverage of the new kernels: the transposed conv in each kernel family, the 3x3/2 max-pool and the stride-2 stem;
  * the op descriptors chained in fp64 reproduce the oracle network;
  * bit equality: packed against full arena, a 3-model plan against three one-model plans, run() against both forms of
    run_batch, run_batch(track=True) against run() per slot, and the keep_res shape 832 x 608.
Run with -s for the tables.
"""
import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.engine import Engine
from tests.plan_steps import FAM, _engine, _exact_bn, _inputs, over_ceiling, print_records
from tests.res_steps import chained_heads, step_and_score
from tests.util import TOL_HEAD_REL, TOL_HEAD_REL_512, golden, net_case_inputs, no_splitk

pytestmark = pytest.mark.gpu

GOLDEN = ["net_res18_b2_96x128", "net_res50_b1_64x64", "net_res18track_b1_64x96", "net_res101_b1_512"]


def _model(arch, trk, wseed, precision, offset_std=0.3):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.precision = precision
    sd = synth.seeded_state_dict(m, seed=wseed, offset_std=offset_std)
    m.load_state_dict(sd)
    return m.cuda().eval(), opt, sd


def golden_head(g, h, got):
    """(stored reference head, the same cells of `got`, max|reference head| over the whole map): a fixture keeps every
    sub-th row and column of its maps (oracle/make_golden_res.py)."""
    sub = int(g["sub"])
    return g["head_" + h], got[..., ::sub, ::sub], float(g["absmax_" + h])


def _truth(x, extra, sd, heads, arch):
    """fp64 evaluation of the oracle graph (on the GPU: res_101 at 512 x 512 is 130 GFLOP)."""
    from oracle import net_ref_res
    sd64 = {k: (v.double().cuda() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    kw = {k: torch.from_numpy(v).double().cuda() for k, v in extra.items()}
    out = net_ref_res.forward(torch.from_numpy(x).double().cuda(), sd64, heads, arch, **kw)
    return {h: v.cpu().numpy() for h, v in out.items()}


@pytest.mark.parametrize("name", GOLDEN)
def test_heads_match_reference_golden_and_fp64(name, cplib):
    g = golden(name)
    arch, trk = str(g["arch"]), bool(int(g["tracking"]))
    rel = TOL_HEAD_REL_512 if int(g["H"]) >= 512 else TOL_HEAD_REL
    x, extra = net_case_inputs(g)
    kw = {k: torch.from_numpy(v).cuda() for k, v in extra.items()}
    truth = None
    for prec in ("fp32", "tf32x3", "tf32", "bf16"):
        m, opt, sd = _model(arch, trk, int(g["wseed"]), prec, float(g["offset_std"]))
        assert int(g["head_conv"]) == m.head_conv == 64
        if truth is None:
            truth = _truth(x, extra, sd, opt.heads, arch)
        out = m(torch.from_numpy(x).cuda(), **kw)[-1]
        assert list(out) == list(opt.heads)
        for h in opt.heads:
            full = out[h].float().cpu().numpy()
            assert full.shape == (int(g["batch"]), opt.heads[h], int(g["H"]) // 4, int(g["W"]) // 4), h
            assert np.isfinite(full).all(), h
            w, got, mag = golden_head(g, h, full)
            _, t, _ = golden_head(g, h, truth[h])
            mag = max(1e-6, mag)
            e = float(np.abs(got - w).max()) / mag
            e_gpu = float(np.abs(got.astype(np.float64) - t).max()) / mag
            e_ref = float(np.abs(w.astype(np.float64) - t).max()) / mag
            print("%s %-7s head %-18s gpu-vs-ref %.2e  gpu-vs-fp64 %.2e  ref-fp32-vs-fp64 %.2e" % (
                name, prec, h, e, e_gpu, e_ref))
            if prec in ("fp32", "tf32x3"):       # fp32-equivalent: the Stage-B bar and the fp64-truth criterion
                assert e <= rel, (prec, h, e)
                assert e_gpu <= 4.0 * e_ref + 3e-5, (prec, h, e_gpu, e_ref)
        del m
        torch.cuda.empty_cache()


# (arch, tracking_task, H, W, batch, max_batch, precisions)
CONFIGS = [
    ("res_18", False, 512, 512, 1, 3, ("fp32", "tf32x3", "tf32", "bf16")),
    ("res_18", False, 512, 512, 3, 3, ("fp32", "tf32x3", "tf32", "bf16")),
    ("res_50", False, 512, 512, 2, 2, ("fp32", "tf32x3")),
    ("res_18", True, 256, 256, 2, 2, ("fp32", "tf32x3")),
]


@pytest.fixture(scope="module")
def res_layer_records(cplib):
    recs = []
    for arch, trk, H, W, b, mb, precs in CONFIGS:
        for prec in precs:
            recs += step_and_score(arch, trk, H, W, b, mb, prec)
    print_records(recs)
    return recs


def test_every_res_op_under_its_ceiling(res_layer_records):
    bad = over_ceiling(res_layer_records)
    assert not bad, "\n".join(bad)


def test_res_launch_coverage(res_layer_records):
    """The transposed conv ran on CUDA cores (fp32), on the wgmma gather kernel in tf32x3 (precisions tf32x3 and tf32,
    whose gather kernel splits in three) and in bf16; the 3x3/2 max-pool ran with and without its residual; the stem ran
    at stride 2 on its direct kernel."""
    have = set()
    for q in res_layer_records:
        if q["kind"] == 3:
            have.add(("deconv", q["prec"], FAM[q["family"]], q["x3"]))
        if q["kind"] == 11:
            have.add(("maxpool3", q["has_res"]))
        if q["family"] == L.FAM_STEM and q["stride"] == 2:
            have.add(("stem s2", q["Cin"]))
    need = {("deconv", "fp32", FAM[L.FAM_IGEMM_FP32], 0), ("deconv", "tf32x3", FAM[L.FAM_IGEMM_UMMA], 1),
            ("deconv", "tf32", FAM[L.FAM_IGEMM_UMMA], 1), ("deconv", "bf16", FAM[L.FAM_IGEMM_UMMA], 0),
            ("maxpool3", 0), ("maxpool3", 1), ("stem s2", 3), ("stem s2", 1), ("stem s2", 8)}
    print("coverage: %s" % sorted(map(str, have)))
    assert not (need - have), sorted(map(str, need - have))


@pytest.mark.parametrize("name", ["net_res18_b2_96x128", "net_res50_b1_64x64", "net_res18track_b1_64x96"])
def test_chained_op_references_are_the_network(name, cplib):
    """The descriptors of the ResNet schedule (transposed-conv phase blocks, max-pool residuals, downsample placement)
    chained in fp64 reproduce the fp64 oracle network."""
    from oracle import net_ref_res
    g = golden(name)
    arch, trk, B, H, W = str(g["arch"]), bool(int(g["tracking"])), int(g["batch"]), int(g["H"]), int(g["W"])
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = _exact_bn(synth.seeded_state_dict(m, seed=int(g["wseed"]), offset_std=float(g["offset_std"])))
    eng, _, _ = _engine(arch, trk, H, W, B, "fp32", sd=sd)
    x, extra = net_case_inputs(g)
    ext = [torch.from_numpy(x).cuda().double()] + [
        torch.from_numpy(extra[k]).cuda().double() if k in extra else None for k in ("pre_img", "pre_hm", "pre_hm_hp")]
    heads = chained_heads(eng, ext, B)
    with torch.no_grad():
        sd64 = {k: v.double().cuda() if v.dtype.is_floating_point else v for k, v in sd.items()}
        want = net_ref_res.forward(ext[0], sd64, opt.heads, arch, pre_img=ext[1], pre_hm=ext[2], pre_hm_hp=ext[3])
    eng.close()
    assert sorted(heads) == sorted(want)
    for h in want:
        e = float((heads[h] - want[h]).abs().max()) / max(1e-30, float(want[h].abs().max()))
        print("%s head %-18s chained-vs-oracle %.2e" % (name, h, e))
        assert e <= 1e-10, (h, e)


# ---- bit equality ------------------------------------------------------------------------------------------------------
def _engines(arch, trk, H, W, B, prec, models=1, reuse=(False, True)):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    out = []
    for r in reuse:
        e = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, tracking=trk, precision=prec, models=models,
                   reuse_activations=r)
        for i in range(models):
            e.load_state_dict(synth.seeded_state_dict(m, seed=11 + i, offset_std=0.3), model=i)
        out.append(e)
    return out, opt, m


def _forward_infer(eng, opt, B, seed, poison=False):
    x, ext = _inputs(eng, B, seed=seed)
    if poison:
        eng.arena().fill_(float("nan"))
    heads = eng.forward(x, *ext[1:])
    meta = cpb.make_meta(B, [eng.width / 2, eng.height / 2], float(max(eng.height, eng.width)), eng.width, eng.height,
                         synth.default_camera(eng.width, eng.height), device="cuda")
    prm = cpb.decode_params(opt)
    if eng.models > 1:
        prm = [prm] * eng.models
    if poison:
        eng.arena().fill_(float("nan"))
    _, poses, n_valid = eng.infer(x, meta, prm, *ext[1:])
    torch.cuda.synchronize()
    return heads, poses, n_valid


RES_REUSE = [
    ("res_18 512", "res_18", False, 512, 512, 2, ("fp32", "tf32x3", "tf32", "bf16")),
    ("res_50 256", "res_50", False, 256, 256, 2, ("tf32x3",)),
    ("res_18 tracking 256", "res_18", True, 256, 256, 2, ("fp32", "tf32x3")),
    ("res_18 keep_res 832x608", "res_18", False, 608, 832, 1, ("fp32", "tf32x3")),
]


@pytest.mark.parametrize("case", RES_REUSE, ids=[c[0] for c in RES_REUSE])
def test_packed_arena_bit_equal(case, cplib):
    label, arch, trk, H, W, MB, precs = case
    for prec in precs:
        (full, reuse), opt, _ = _engines(arch, trk, H, W, MB, prec)
        assert reuse.memory["activation"] < full.memory["activation"]
        for B in sorted({1, MB}):
            a = _forward_infer(full, opt, B, 317)
            b = _forward_infer(reuse, opt, B, 317, poison=True)
            for h in a[0]:
                assert torch.equal(a[0][h], b[0][h]), (label, prec, B, h)
                assert torch.isfinite(a[0][h]).all(), (label, prec, B, h)
            assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), (label, prec, B)
        full.close()
        reuse.close()


@pytest.mark.parametrize("prec", ["fp32", "tf32x3"])
def test_three_model_plan_equals_single_plans(prec, cplib):
    """A 3-model res_18 plan (one launch per layer for all models) against three one-model plans, bit for bit (K partition
    held fixed: the split-K factor follows the launch's size, see tests/util.py no_splitk)."""
    with no_splitk():
        (multi,), opt, m = _engines("res_18", False, 256, 256, 2, prec, models=3, reuse=(True,))
        x, _ = _inputs(multi, 2, seed=9)
        got = multi.forward(x)
        for i in range(3):
            e = Engine("res_18", m.heads, m.head_conv, 2, 256, 256, 0, precision=prec, reuse_activations=True)
            e.load_state_dict(synth.seeded_state_dict(m, seed=11 + i, offset_std=0.3))
            want = e.forward(x)
            for h in want:
                assert torch.equal(got[h][i], want[h]), (prec, i, h)
            e.close()
        multi.close()


def _detector(arch, trk, seed=21):
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=seed, offset_std=0.3, head_gain=6.0 if trk else 1.0))
    m = m.cuda().eval()
    if not trk:
        x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(1, 512, 512, seed=5))).cuda()
        with torch.no_grad():
            synth.calibrate_head_bias(m, m(x)[-1], target=4)
    return cpb.ObjectPoseDetector(opt, model=m), opt


def _same_records(results, poses, n):
    assert len(results) == int(n)
    for i, d in enumerate(results):
        assert d["score"] == poses[i, L.P_SCORE]
        assert np.array_equal(np.asarray(d["kps"], np.float32), poses[i, L.P_KPS:L.P_KPS + 16])
        assert np.array_equal(np.asarray(d["bbox"], np.float32), poses[i, L.P_BBOX:L.P_BBOX + 4])


def test_run_equals_both_forms_of_run_batch(cplib):
    """res_18: run() of each frame == run_batch of the uint8 array and of a list of mixed-size frames."""
    det, opt = _detector("res_18", False)
    cam = synth.default_camera(512, 512)
    arr = synth.synthetic_frames(3, 512, 512, seed=9)
    lst = [synth.synthetic_frames(1, 480, 640, seed=82)[0], synth.synthetic_frames(1, 600, 800, seed=83)[0]]
    cams = [synth.default_camera(640, 480), synth.default_camera(800, 600)]
    total = 0
    with no_splitk():
        poses, n_valid = det.run_batch(arr, cam)
        for b in range(3):
            ret = det.run(arr[b], meta_inp={"camera_matrix": cam})
            _same_records(ret["results"], poses[b], n_valid[b])
            total += int(n_valid[b])
        poses, n_valid = det.run_batch(lst, np.stack(cams))
        for b in range(2):
            ret = det.run(lst[b], meta_inp={"camera_matrix": cams[b]})
            _same_records(ret["results"], poses[b], n_valid[b])
            total += int(n_valid[b])
    print("res_18 run vs run_batch: %d detections compared" % total)


def test_run_batch_tracking_equals_run_per_slot(cplib):
    """res_18 tracking: two video slots through run_batch(track=True) == each video alone through run()."""
    det, opt = _detector("res_18", True, seed=31)
    cam = synth.default_camera(512, 512)
    vids = [synth.synthetic_frames(3, 512, 512, seed=100 + v) for v in range(2)]
    with no_splitk():
        per_stream = []
        for v in range(2):
            det.reset_tracking()
            rows = []
            for f in range(3):
                ret = det.run(vids[v][f], meta_inp={"camera_matrix": cam})
                rows.append([(d["tracking_id"], d["score"]) for d in ret["results"]])
            per_stream.append(rows)
        det.reset_tracking()
        print("res_18 run_batch(track=True) vs run: %d tracks compared" % sum(len(r) for rows in per_stream for r in rows))
        for f in range(3):
            tracks, nt = det.run_batch(np.stack([vids[0][f], vids[1][f]]), cam, track=True)
            for v in range(2):
                want = per_stream[v][f]
                assert int(nt[v]) == len(want), (f, v)
                for i, (tid, score) in enumerate(want):
                    assert int(tracks[v, i, L.T_ID]) == tid
                    assert float(tracks[v, i, L.P_SCORE]) == np.float32(score)


def test_demo_flow_res_18(cplib, tmp_path):
    """The demo flow of src/demo.py (as tests/test_dropin_demo.py runs it for dla_34) with --arch res_18: a detector
    from a seeded checkpoint path, run() on the committed frames, the --debug 4 JSON files."""
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    opt = cpb.default_opt("res_18", debug=4)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=9, offset_std=0.3, head_gain=6.0))
    ck = str(tmp_path / "chair_res18_seeded.pth")
    cpb.save_model(ck, 1, m)
    opt.load_model = ck
    opt.demo = os.path.join(root, "tests", "data")
    opt.demo_save = str(tmp_path / "save")
    cam = np.array([[663.0287679036459, 0, 300.2775065104167], [0, 663.0287679036459, 395.00066121419275], [0, 0, 1]])
    det = cpb.detector_factory["object_pose"](opt)
    assert isinstance(det.model, cpb.PoseResNetB200)
    det.pause = False
    for f in sorted(f for f in os.listdir(opt.demo) if f.endswith(".png")):
        ret = det.run(os.path.join(opt.demo, f), meta_inp={"camera_matrix": cam})
        assert ret["output"]["hm"].shape[-2:] == (128, 128)
        j = json.load(open(os.path.join(opt.demo_save, "data", os.path.splitext(f)[0] + ".json")))
        assert set(j) == {"camera_data", "objects"} and len(j["objects"]) == len(ret["boxes"])

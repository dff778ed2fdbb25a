"""Multi-model plans on the GPU: each model's slice of a plan of M = 3 checkpoints (seeded state dicts with different
seeds, so a wrong model index changes every layer) against that checkpoint's own plan.

  * bit equality of the head logits with a fixed K partition (CP_NO_SPLITK=1), at the geometries and precisions that
    reach every kernel family (tests/test_gpu_plan_geometry.py), with a coverage list of the families launched;
  * with split-K on, every op of every model against fp64 (tests/plan_steps.py, tests/layer_ref.py) under LAYER_CEIL;
  * cp_infer_multi per model against decode_pnp of that model's heads; mismatched decode parameters are refused;
  * MultiCategoryDetector.run_batch against each category's ObjectPoseDetector.run_batch;
  * one launch per op for all models.
"""
import ctypes

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib, synth
from centerpose_b200.engine import Engine
from tests import layer_ref
from tests.plan_steps import FAM, _ceiling, _fetch, _inputs
from tests.util import LAYER_CEIL, no_splitk

pytestmark = pytest.mark.gpu

M = 3
SEEDS = (11, 12, 13)


def _engines(arch, H, W, B, prec, env=None, calibrate=False):
    """(multi-model engine, [single-model engines], state dicts, model)."""
    opt = cpb.default_opt(arch)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sds = []
    for s in SEEDS:
        sd = synth.seeded_state_dict(m, seed=s, offset_std=0.3)
        if calibrate:
            m.load_state_dict(sd)
            m = m.cuda()
            x, _ = _inputs(m.engine(B, H, W), B)
            synth.calibrate_head_bias(m, m(x)[-1], target=4)
            sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
        sds.append(sd)
    kw = dict(tracking_task_gru=False, precision=prec)
    with layer_ref_env(env):
        multi = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, models=M, **kw)
        singles = [Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, **kw) for _ in range(M)]
    for i, sd in enumerate(sds):
        multi.load_state_dict(sd, model=i)
        singles[i].load_state_dict(sd)
    return multi, singles, sds, opt


def layer_ref_env(env):
    from tests.plan_steps import _env
    return _env(env)


# (label, arch, H, W, batch, precisions, environment at plan creation)
GEOMETRIES = [
    ("512 b1", "dla_34", 512, 512, 1, ("tf32x3",), None),
    ("512 b2", "dla_34", 512, 512, 2, ("fp32", "tf32x3", "tf32", "bf16"), None),
    ("keep_res 832x608", "dla_34", 832, 608, 2, ("fp32", "tf32x3", "tf32", "bf16"), None),
    ("keep_res 736x1312", "dla_34", 736, 1312, 1, ("tf32x3",), None),
    ("no dcn_tma", "dla_34", 512, 512, 2, ("tf32x3",), {"CP_NO_DCN_TMA": "1"}),
    ("dlav1 128x160", "dlav1_34", 128, 160, 2, ("fp32", "tf32x3"), None),
]
CASES = [(g[0], g[1], g[2], g[3], g[4], p, g[6]) for g in GEOMETRIES for p in g[5]]


def _family_key(d, info):
    fam = FAM[info["family"]]
    if info["family"] == _lib.FAM_IGEMM_UMMA:
        return fam + (" deformable" if d["kind"] == 2 else " strided" if d["stride"] > 1 else "")
    if info["family"] == _lib.FAM_CONV_TMA:
        return fam + (" fused" if d["fuse_heads"] else " %dx%d" % (d["kh"], d["kh"]))
    return fam


def _slice_case(label, arch, H, W, B, prec, env):
    """One geometry / precision: every model's heads (cp_forward and cp_plan_run_ops) against its own plan, bit for bit,
    with the K partition fixed.  Returns the set of kernel families (_family_key) the multi-model plan launched."""
    with no_splitk():
        multi, singles, _, _ = _engines(arch, H, W, B, prec, env)
        x, _ = _inputs(multi, B)
        n_ops = len(multi.op_descs())
        heads = {n: torch.full((M, B, c, H // 4, W // 4), float("nan"), device="cuda") for n, c in multi.heads.items()}
        infos = multi.run_ops(x, 0, n_ops, heads)
        got = multi.forward(x)
        for i, eng in enumerate(singles):
            want = eng.forward(x)
            assert multi.L.cp_plan_forward_launches(multi.plan) == eng.L.cp_plan_forward_launches(eng.plan)
            for n in want:
                assert torch.equal(got[n][i], want[n]), (label, prec, "model", i, n)
                assert torch.equal(heads[n][i], want[n]), (label, prec, "model", i, n, "run_ops")
    return {_family_key(d, info) for d, info in zip(multi.op_descs(), infos) if info["family"] != _lib.FAM_NONE}


@pytest.fixture(scope="module")
def slice_case():
    """_slice_case, each case run once per module whichever test asks for it first."""
    done = {}

    def run(case):
        key = repr(case)
        if key not in done:
            done[key] = _slice_case(*case)
        return done[key]
    return run


@pytest.mark.parametrize("case", CASES, ids=["%s %s" % (c[0], c[5]) for c in CASES])
def test_model_slice_bit_equal(slice_case, case):
    slice_case(case)


def test_every_family_reached(slice_case):
    """Every kernel family ran on a multi-model plan over the cases above."""
    reached = set()
    for case in CASES:
        reached |= slice_case(case)
    want = {"stem", "conv3_c16", "igemm_fp32", "igemm_umma strided", "igemm_umma deformable", "conv_tma 3x3",
            "conv_tma 1x1", "conv_tma fused", "dcn_tma", "upadd", "gn_relu", "gru"}
    missing = sorted(w for w in want if not any(n.startswith(w) for n in reached))
    assert not missing, (missing, sorted(reached))


def test_model_index_and_loading_checked():
    """Out-of-range model indices return CP_ERR_INVALID; a plan runs only once every model is loaded."""
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    sd = synth.seeded_state_dict(m, seed=1)
    eng = Engine(m._arch(), m.heads, m.head_conv, 1, 64, 96, 0, models=M, precision="tf32x3")
    assert eng.L.cp_plan_num_models(eng.plan) == M
    d = _lib.CpOpDesc()
    for bad in (-1, M):
        assert eng.L.cp_plan_op_desc_model(eng.plan, bad, 0, ctypes.byref(d)) == -1          # CP_ERR_INVALID
        with pytest.raises(RuntimeError, match="model index out of range"):
            eng.load_state_dict(sd, model=bad)
    x, _ = _inputs(eng, 1)
    for i in range(M - 1):
        eng.load_state_dict(sd, model=i)
        with pytest.raises(RuntimeError, match="cp_plan_load_weights_model for every model|call cp_plan_load_weights"):
            eng.forward(x)
        heads = {n: torch.empty((M, 1, c, 16, 24), device="cuda") for n, c in eng.heads.items()}
        hp = (ctypes.c_void_p * len(eng.head_names))(*[heads[n].data_ptr() for n in eng.head_names])
        assert eng.L.cp_forward(eng.plan, 1, ctypes.c_void_p(x.data_ptr()), None, None, None, hp, None) == -3
    eng.load_state_dict(sd, model=M - 1)
    out = eng.forward(x)
    assert all(torch.isfinite(v).all() for v in out.values())


def test_splitk_ops_under_ceiling():
    """Split-K on, 512 x 512, batch 1: every op of every model against fp64; at least one conv_tma and one dcn_tma
    launch splits K."""
    multi, _, _, _ = _engines("dla_34", 512, 512, 1, "tf32x3")
    x, ext = _inputs(multi, 1)
    heads = {n: torch.full((M, 1, c, 128, 128), float("nan"), device="cuda") for n, c in multi.heads.items()}
    descs = [multi.op_descs(model=i) for i in range(M)]
    split = set()
    bad = []
    for k in range(len(descs[0])):
        wants = []
        with torch.no_grad():
            for i in range(M):
                rd = layer_ref.ActReader(multi.arena(), ext, [0], 1)
                wants.append((rd, layer_ref.op_ref(descs[i][k], rd, _fetch, descs[i])))
        info = multi.run_ops(x, k, k + 1, heads)[0]
        torch.cuda.synchronize()
        d = descs[0][k]
        if d["fused_away"]:
            continue
        if info["ksplit"] > 1:
            split.add(info["family"])
        for i, (rd, want) in enumerate(wants):
            r = 0.0
            for (kind, tgt), ref, S in want:
                got = rd.get(tgt) if kind == "act" else heads[multi.head_names[tgt]][i].double()
                r = max(r, (0.0 if torch.equal(got, ref) else float("inf")) if d["family"] == _lib.FAM_MAXPOOL
                        else layer_ref.score(got, ref, S))
            if not r <= LAYER_CEIL[_ceiling(d, "tf32x3")]:
                bad.append((i, k, d["name"], r))
    assert not bad, bad
    assert _lib.FAM_CONV_TMA in split and _lib.FAM_DCN_TMA in split, split


def test_infer_multi_matches_decode_per_model():
    cats = ("chair", "cup", "laptop")      # visible_thresh 6 / 3 / 0
    with no_splitk():
        multi, _, _, opt = _engines("dla_34", 512, 512, 2, "tf32x3", calibrate=True)
        x, _ = _inputs(multi, 2)
        cam = synth.default_camera(512, 512)
        meta = cpb.make_meta(2, np.array([256., 256.], np.float32), 512.0, 512, 512, cam, device="cuda")
        prms = [cpb.decode_params(opt, c=c) for c in cats]
        heads = {n: torch.empty((M, 2, c, 128, 128), device="cuda") for n, c in multi.heads.items()}
        _, poses, n_valid = multi.infer(x, meta, prms, heads_out=heads)
        torch.cuda.synchronize()
        for i, c in enumerate(cats):
            _, want_p, want_n = cpb.decode_pnp({n: heads[n][i] for n in heads}, meta, cpb.decode_params(opt, c=c))
            assert (want_n > 0).all(), (c, want_n)
            assert torch.equal(n_valid[i], want_n), c
            for b in range(2):
                k = int(want_n[b])
                assert torch.equal(poses[i, b, :k], want_p[b, :k]), (c, b)
    bad = [cpb.decode_params(opt, c=c) for c in cats]
    bad[1].K = 50
    with pytest.raises(RuntimeError, match="visible_thresh and balance only"):
        multi.infer(x, meta, bad)


def test_detector_matches_per_category(tmp_path):
    cats = ("chair", "cup", "laptop")
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt).cuda()
    frames = synth.synthetic_frames(2, 512, 512, seed=5)        # the array form's network input is x itself
    x = torch.from_numpy(synth.normalize_frames(frames)).cuda()
    paths = {}
    for c, s in zip(cats, SEEDS):
        m.load_state_dict(synth.seeded_state_dict(m, seed=s, offset_std=0.3))
        synth.calibrate_head_bias(m, m(x)[-1], target=4)
        paths[c] = str(tmp_path / (c + ".pth"))
        cpb.save_model(paths[c], 1, m)
    cam = synth.default_camera(512, 512)
    ragged = [frames[0], synth.synthetic_frames(1, 600, 800, seed=6)[0]]
    with no_splitk():
        det = cpb.MultiCategoryDetector(opt, paths)
        assert det.categories == list(cats)
        got_a = det.run_batch(frames, cam)
        got_l = det.run_batch(ragged, cam)
        out = (torch.empty((M, 2, opt.K, _lib.CP_POSE_RECORD), device="cuda"),
               torch.empty((M, 2), dtype=torch.int32, device="cuda"))
        ret = det.run_batch(frames, cam, to_host=False, out=out)
        assert ret[0] is out[0] and ret[1] is out[1]
        for i, c in enumerate(cats):
            o = cpb.default_opt("dla_34", c=c, load_model=paths[c])
            one = cpb.ObjectPoseDetector(o)
            for got, fr in ((got_a, frames), (got_l, ragged)):
                wp, wn = one.run_batch(fr, cam)
                assert wn.sum() > 0 and np.array_equal(got[1][i], wn), (c, got[1][i], wn)
                for b in range(2):
                    assert np.array_equal(got[0][i, b, :wn[b]], wp[b, :wn[b]]), (c, b)
            assert np.array_equal(out[1][i].cpu().numpy(), got_a[1][i])
        with pytest.raises(NotImplementedError):
            det.process(torch.from_numpy(synth.normalize_frames(frames)).cuda())
        # one category: the same [M, B, ...] outputs, M = 1
        one_cat = cpb.MultiCategoryDetector(opt, {"cup": paths["cup"]})
        p1, n1 = one_cat.run_batch(frames, cam)
        assert p1.shape == (1, 2, opt.K, _lib.CP_POSE_RECORD) and n1.shape == (1, 2)
        assert np.array_equal(n1[0], got_a[1][1])
        for b in range(2):
            assert np.array_equal(p1[0, b, :n1[0, b]], got_a[0][1, b, :n1[0, b]]), b
        out1 = (torch.empty((1, 2, opt.K, _lib.CP_POSE_RECORD), device="cuda"),
                torch.empty((1, 2), dtype=torch.int32, device="cuda"))
        ret1 = one_cat.run_batch(frames, cam, to_host=False, out=out1)
        assert ret1[0] is out1[0] and ret1[1] is out1[1] and np.array_equal(out1[1].cpu().numpy(), n1)

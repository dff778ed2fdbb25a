"""Plans with a liveness-packed activation arena (CP_PLAN_REUSE_ACTIVATIONS) on the GPU: bit for bit what the full arena
computes.

  * heads (cp_forward) and poses / n_valid (cp_infer, cp_infer_multi, cp_infer_multi_track) of a reuse plan against a
    full plan with the same weights, in every precision and on every architecture, with PDL forced on and off, with the
    deformable convs on the gather kernel, and through an InferGraph replay;
  * stale data: the reuse arena is filled with NaN before every call, and frames B after frames A on one plan equal
    frames B on a fresh plan, so nothing relies on zeroed or leftover memory;
  * the product paths (run_batch, MultiCategoryTracker.run_batch) against the same paths on full-arena engines;
  * a reuse plan stepped op by op against the fp64 per-op references (tests/layer_ref.py);
  * the plan's arena and cp_plan_bytes equal the host dry run (cp_plan_memory).
Split-K stays at its default: its partition depends on shapes only, so both plans add the same partial sums.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

import centerpose_b200 as cpb
from centerpose_b200 import _lib as L
from centerpose_b200 import synth
from centerpose_b200.engine import Engine, InferGraph, plan_memory
from tests import layer_ref
from tests.plan_steps import _ceiling, _env, _fetch, _heads, _inputs
from tests.test_gpu_multi_category_track import _checkpoints, _steps
from tests.util import LAYER_CEIL

pytestmark = pytest.mark.gpu


def _pair(arch, trk, H, W, B, prec, models=1, env=None):
    """(full engine, reuse engine) with the same seeded weights (one seed per model)."""
    opt = cpb.default_opt(arch, tracking_task=trk)
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    kw = dict(tracking=trk, tracking_task_gru=m.use_convGRU and m.tracking_task, precision=prec, models=models)
    with _env(env):
        full = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, **kw)
        reuse = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, reuse_activations=True, **kw)
    for i in range(models):
        sd = synth.seeded_state_dict(m, seed=11 + i, offset_std=0.3)
        full.load_state_dict(sd, model=i)
        reuse.load_state_dict(sd, model=i)
    return full, reuse, opt


def _poison(eng):
    eng.arena().fill_(float("nan"))


def _ext(eng, B, seed):
    x, ext = _inputs(eng, B, seed=seed)
    if eng.tracking and eng.models > 1:
        g = torch.Generator(device="cuda").manual_seed(seed + 7)
        ext[2] = torch.rand((eng.models, B, 1, eng.height, eng.width), device="cuda", generator=g)
        ext[3] = torch.rand((eng.models, B, 8, eng.height, eng.width), device="cuda", generator=g)
    return x, ext


def _call(eng, opt, B, seed, poison):
    """heads (cp_forward) and (poses, n_valid) (cp_infer*) of frames `seed`."""
    x, ext = _ext(eng, B, seed)
    if poison:
        _poison(eng)
    heads = eng.forward(x, *ext[1:])
    meta = cpb.make_meta(B, [eng.width / 2, eng.height / 2], float(max(eng.height, eng.width)), eng.width, eng.height,
                         synth.default_camera(eng.width, eng.height), device="cuda")
    prm = cpb.decode_params(opt)
    if eng.models > 1:
        prm = [prm] * eng.models
    if poison:
        _poison(eng)
    _, poses, n_valid = eng.infer(x, meta, prm, *ext[1:])
    torch.cuda.synchronize()
    return heads, poses, n_valid


def _assert_same(a, b, label):
    ha, pa, na = a
    hb, pb, nb = b
    for h in ha:
        assert torch.equal(ha[h], hb[h]), (label, h)
    assert torch.equal(na, nb), (label, "n_valid")
    assert torch.equal(pa, pb), (label, "poses")


# (label, arch, tracking, H, W, max_batch, precisions, models, env at plan creation)
CASES = [
    ("dla34 512", "dla_34", False, 512, 512, 2, ("fp32", "tf32x3", "tf32", "bf16"), 1, None),
    ("dla34 keep_res", "dla_34", False, 608, 832, 1, ("tf32x3",), 1, None),
    ("dlav1 128x160", "dlav1_34", False, 128, 160, 2, ("fp32", "tf32x3"), 1, None),
    ("dla34 tracking", "dla_34", True, 512, 512, 2, ("tf32x3",), 1, None),
    ("dlav1 tracking", "dlav1_34", True, 128, 160, 2, ("tf32x3",), 1, None),
    ("dla34 M3", "dla_34", False, 256, 256, 2, ("tf32x3",), 3, None),
    ("dla34 tracking M3", "dla_34", True, 256, 256, 2, ("tf32x3",), 3, None),
    ("dla34 no dcn_tma", "dla_34", False, 512, 512, 2, ("tf32x3",), 1, {"CP_NO_DCN_TMA": "1"}),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_reuse_plan_bit_equal(case):
    label, arch, trk, H, W, MB, precs, M, env = case
    for prec in precs:
        full, reuse, opt = _pair(arch, trk, H, W, MB, prec, M, env)
        assert reuse.memory["activation"] < full.memory["activation"]
        for B in sorted({1, MB}):
            want = _call(full, opt, B, 317, False)
            _assert_same(want, _call(reuse, opt, B, 317, True), (label, prec, B))
        full.close()
        reuse.close()


@pytest.mark.parametrize("pdl", ["CP_PDL", "CP_NO_PDL"])
def test_reuse_plan_bit_equal_pdl(pdl):
    full, reuse, opt = _pair("dla_34", False, 512, 512, 2, "tf32x3")
    old = {k: os.environ.pop(k, None) for k in ("CP_PDL", "CP_NO_PDL")}
    try:
        with _env({pdl: "1"}):
            for B in (1, 2):
                _assert_same(_call(full, opt, B, 318, False), _call(reuse, opt, B, 318, True), (pdl, B))
    finally:
        os.environ.update({k: v for k, v in old.items() if v is not None})
    full.close()
    reuse.close()


def test_stale_frames_do_not_leak():
    """Frames B after frames A on one reuse plan equal frames B on a fresh reuse plan and on a full plan."""
    full, reuse, opt = _pair("dla_34", True, 256, 256, 2, "tf32x3")
    _, fresh, _ = _pair("dla_34", True, 256, 256, 2, "tf32x3")
    _call(reuse, opt, 2, 400, False)
    b_after_a = _call(reuse, opt, 2, 401, False)
    _assert_same(_call(fresh, opt, 2, 401, False), b_after_a, "fresh")
    _assert_same(_call(full, opt, 2, 401, False), b_after_a, "full")
    for e in (full, reuse, fresh):
        e.close()


def test_infer_graph_replay():
    full, reuse, opt = _pair("dla_34", False, 512, 512, 1, "tf32x3")
    prm = cpb.decode_params(opt)
    _poison(reuse)
    graph = InferGraph(reuse, 1, prm)
    for seed in (501, 502):
        x, _ = _inputs(full, 1, seed=seed)
        meta = graph.meta.clone()
        _, wp, wn = full.infer(x, meta, prm)
        _poison(reuse)
        gp, gn = graph(x, meta)
        torch.cuda.synchronize()
        assert torch.equal(gn, wn) and torch.equal(gp, wp), seed
    full.close()
    reuse.close()


def test_memory_matches_dry_run():
    """The plan allocates what cp_plan_memory computes on the host, with and without reuse."""
    full, reuse, _ = _pair("dla_34", True, 512, 512, 2, "tf32x3", models=2)
    opt = cpb.default_opt("dla_34", tracking_task=True)
    for eng in (full, reuse):
        dry = plan_memory("dla_34", opt.heads, opt.head_conv, 2, 512, 512, tracking=True, precision="tf32x3", models=2,
                          reuse_activations=eng.reuse_activations)
        assert eng.memory == dry
        assert eng.arena().numel() * 4 == dry["activation"]
        assert eng.plan_bytes == dry["activation"] + dry["weights"]
    assert reuse.memory["activation"] * 4 < full.memory["activation"]
    full.close()
    reuse.close()


def test_reuse_plan_steps_under_ceiling():
    """A reuse plan stepped op by op from op 0: every op's inputs are still live when it runs, and every op scores
    under its LAYER_CEIL against the fp64 reference taken from them."""
    _, eng, _ = _pair("dla_34", True, 512, 512, 2, "tf32x3")
    descs = eng.op_descs()
    x, ext = _inputs(eng, 2)
    heads = _heads(eng, 2)
    _poison(eng)
    rd = layer_ref.ActReader(eng.arena(), ext, [0, 1], 2)
    bad = []
    for i, d in enumerate(descs):
        with torch.no_grad():
            want = layer_ref.op_ref(d, rd, _fetch, descs)
        li = eng.run_ops(x, i, i + 1, heads, *ext[1:])[0]
        torch.cuda.synchronize()
        assert li["family"] == (L.FAM_NONE if d["fused_away"] else d["family"]), d["name"]
        for (kind, tgt), ref, S in want:
            got = rd.get(tgt) if kind == "act" else heads[eng.head_names[tgt]][[0, 1]].double()
            r = (0.0 if torch.equal(got, ref) else float("inf")) if d["family"] == L.FAM_MAXPOOL else layer_ref.score(got, ref, S)
            if not r <= LAYER_CEIL[_ceiling(d, "tf32x3")]:
                bad.append("op %d %s: r %.3e" % (i, d["name"], r))
    eng.close()
    assert not bad, "\n".join(bad)


# ---- the product paths -------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _full_arena_engines():
    """Every Engine made inside the block has the full arena (what the product paths used before reuse)."""
    init = Engine.__init__

    def full(self, *a, **k):
        k["reuse_activations"] = False
        init(self, *a, **k)

    Engine.__init__ = full
    try:
        yield
    finally:
        Engine.__init__ = init


def _plain_detector():
    opt = cpb.default_opt("dla_34")
    m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
    m.load_state_dict(synth.seeded_state_dict(m, seed=3, offset_std=0.3))
    m = m.cuda().eval()
    x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(1, 512, 512, seed=5))).cuda()
    synth.calibrate_head_bias(m, m(x)[-1], target=4)
    return cpb.ObjectPoseDetector(opt, model=m)


def _run_products(tmp_path):
    tmp_path.mkdir()
    cam = synth.default_camera(512, 512)
    out = []
    det = _plain_detector()
    arr = synth.synthetic_frames(2, 512, 512, seed=81)
    lst = [synth.synthetic_frames(1, 480, 640, seed=82)[0], synth.synthetic_frames(1, 600, 800, seed=83)[0]]
    cams = np.stack([synth.default_camera(640, 480), synth.default_camera(800, 600)])
    out.append(det.run_batch(arr, cam))
    out.append(det.run_batch(lst, cams))
    engines = list(det.model._engines.values())
    opt, paths = _checkpoints(tmp_path, False)
    one = cpb.ObjectPoseDetector(cpb.default_opt("dla_34", tracking_task=True, c="cup", load_model=paths["cup"]))
    multi = cpb.MultiCategoryTracker(opt, paths)
    for frames, cams_k, new_video, _ in _steps(cam):
        kw = {} if new_video is None else {"new_video": new_video}
        out.append(one.run_batch(frames, cams_k, track=True, **kw))
        out.append(multi.run_batch(frames, cams_k, **kw))
    engines += list(one.model._engines.values()) + [multi._eng]
    return out, engines


def test_product_paths_match_full_arena(tmp_path):
    got, engines = _run_products(tmp_path / "reuse")
    assert engines and all(e.reuse_activations for e in engines)
    with _full_arena_engines():
        want, full_engines = _run_products(tmp_path / "full")
    assert not any(e.reuse_activations for e in full_engines)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        for a, b in zip(g, w):
            assert np.array_equal(np.asarray(a), np.asarray(b)), k

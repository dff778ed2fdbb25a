"""Every DCN op's output and every head of cp_forward from two builds of the library, compared bit for bit (SHA-256 of
each tensor), on the plans that run dcn_tma: batch 32 at 512 x 512 in tf32x3 and tf32, the tracking plan at batch 8,
a 2-model plan, 384 x 640 in tf32x3 and tf32, and batch-invariant plans at batches 2 and 4.  The plans keep every
activation (no arena reuse), so each DCN op's output is still in the arena after the forward.

    python scripts/dcn_ab.py LIB_A LIB_B OUT_DIR     # digests with each library (CP_LIB_PATH), then compares
    python scripts/dcn_ab.py --dump OUT.json         # the digests of the library CP_LIB_PATH names
"""
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, tracking plan, models, batch, H, W, precision, batch-invariant)
PLANS = [("b32_512_x3", False, 1, 32, 512, 512, "tf32x3", False),
         ("b32_512_tf32", False, 1, 32, 512, 512, "tf32", False),
         ("track_b8_512_x3", True, 1, 8, 512, 512, "tf32x3", False),
         ("two_models_b4_256_x3", False, 2, 4, 256, 256, "tf32x3", False),
         ("b3_384x640_x3", False, 1, 3, 384, 640, "tf32x3", False),
         ("b3_384x640_tf32", False, 1, 3, 384, 640, "tf32", False),
         ("invariant_b2_512_x3", False, 1, 2, 512, 512, "tf32x3", True),
         ("invariant_b4_512_x3", False, 1, 4, 512, 512, "tf32x3", True)]


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def dump(path):
    import torch
    import centerpose_b200 as cpb
    from centerpose_b200 import _lib
    from centerpose_b200 import synth
    from centerpose_b200.engine import Engine
    out = {}
    for name, trk, models, B, H, W, prec, inv in PLANS:
        opt = cpb.default_opt("dla_34", tracking_task=trk)
        m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
        eng = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, tracking=m.tracking_inputs,
                     tracking_task_gru=m.use_convGRU and m.tracking_task, precision=prec, models=models,
                     batch_invariant=inv)
        for i in range(models):
            eng.load_state_dict(synth.seeded_state_dict(m, seed=31 + i, offset_std=0.3), model=i)
        x = torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, H, W, seed=5))).cuda()
        ext = {}
        if trk:
            g = torch.Generator(device="cuda").manual_seed(6)
            ext = dict(pre_img=torch.from_numpy(synth.normalize_frames(synth.synthetic_frames(B, H, W, seed=7))).cuda(),
                       pre_hm=torch.rand((B, 1, H, W), device="cuda", generator=g),
                       pre_hm_hp=torch.rand((B, 8, H, W), device="cuda", generator=g))
        heads = eng.forward(x, **ext)
        torch.cuda.synchronize()
        for n, t in heads.items():
            out["%s/head %s" % (name, n)] = _digest(t)
        arena = eng.arena()
        n_dcn = 0
        for model in range(models):
            for d in eng.op_descs(model):
                if d["family"] != _lib.FAM_DCN_TMA or d["out_head"] >= 0:
                    continue
                a = d["out"]
                n = min(B * a["H"] * a["W"] * a["stride"], arena.numel() - a["off"])
                out["%s/model %d %s" % (name, model, d["name"])] = _digest(arena[a["off"]:a["off"] + n])
                n_dcn += 1
        assert n_dcn, "%s: no dcn_tma op" % name
        eng.close()
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


def compare(a, b):
    A, B = json.load(open(a)), json.load(open(b))
    assert sorted(A) == sorted(B), (sorted(set(A) ^ set(B)))
    bad = [k for k in A if A[k] != B[k]]
    for k in sorted(A):
        print("%-60s %s" % (k, "equal" if k not in bad else "DIFFER"))
    print("%d of %d tensors bit-identical" % (len(A) - len(bad), len(A)))
    return not bad


if __name__ == "__main__":
    if sys.argv[1] == "--dump":
        dump(sys.argv[2])
        sys.exit(0)
    lib_a, lib_b, out_dir = sys.argv[1:4]
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for tag, lib in (("a", lib_a), ("b", lib_b)):
        p = os.path.join(out_dir, "digests_%s.json" % tag)
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", p],
                              env=dict(os.environ, CP_LIB_PATH=os.path.abspath(lib)))
        paths.append(p)
    sys.exit(0 if compare(*paths) else 1)

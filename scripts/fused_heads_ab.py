"""Head tensors of cp_forward from two builds of the library, compared bit for bit, on the plans that run the tf32x3
fused-heads 3x3: batch 32 at 512 x 512, the 11-head tracking plan at batch 8, a 2-model plan and a 96 x 160 head map.

    python scripts/fused_heads_ab.py LIB_A LIB_B OUT_DIR     # dumps with each library (CP_LIB_PATH), then compares
    python scripts/fused_heads_ab.py --dump OUT.npz          # the heads of the library CP_LIB_PATH names
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

# (name, tracking plan, models, batch, H, W)
PLANS = [("b32_512", False, 1, 32, 512, 512), ("track_b8_512", True, 1, 8, 512, 512),
         ("two_models_b4_256", False, 2, 4, 256, 256), ("b3_384x640", False, 1, 3, 384, 640)]


def dump(path):
    import torch
    import centerpose_b200 as cpb
    from centerpose_b200 import synth
    from centerpose_b200.engine import Engine
    out = {}
    for name, trk, models, B, H, W in PLANS:
        opt = cpb.default_opt("dla_34", tracking_task=trk)
        m = cpb.create_model(opt.arch, opt.heads, opt.head_conv, opt)
        eng = Engine(m._arch(), m.heads, m.head_conv, B, H, W, 0, tracking=m.tracking_inputs,
                     tracking_task_gru=m.use_convGRU and m.tracking_task, precision="tf32x3",
                     **({"models": models} if models > 1 else {}))
        for i in range(models):
            sd = synth.seeded_state_dict(m, seed=31 + i, offset_std=0.3)
            if models > 1:
                eng.load_state_dict(sd, model=i)
            else:
                eng.load_state_dict(sd)
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
            out["%s/%s" % (name, n)] = t.cpu().numpy()
        eng.close()
    np.savez(path, **out)


def compare(a, b):
    A, B = np.load(a), np.load(b)
    assert sorted(A.files) == sorted(B.files), (A.files, B.files)
    bad = [k for k in A.files if not np.array_equal(A[k], B[k])]
    for k in sorted(A.files):
        print("%-40s %-6s %s" % (k, "equal" if k not in bad else "DIFFER", A[k].shape))
    print("%d of %d head tensors bit-identical" % (len(A.files) - len(bad), len(A.files)))
    return not bad


if __name__ == "__main__":
    if sys.argv[1] == "--dump":
        dump(sys.argv[2])
        sys.exit(0)
    lib_a, lib_b, out_dir = sys.argv[1:4]
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    for tag, lib in (("a", lib_a), ("b", lib_b)):
        p = os.path.join(out_dir, "heads_%s.npz" % tag)
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", p],
                              env=dict(os.environ, CP_LIB_PATH=os.path.abspath(lib)))
        paths.append(p)
    sys.exit(0 if compare(*paths) else 1)

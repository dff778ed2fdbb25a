"""TEST INFRASTRUCTURE ONLY -- generates the ResNet network fixtures
tests/golden/net_res*.npz by running the UNMODIFIED reference PoseResNet
(msra_resnet.py, through oracle/ref_shims.py, whose `load_url` shim stands in
for the ImageNet download of init_weights) on seeded weights.

    python -m oracle.make_golden_res [name ...]

The fixtures have the layout of oracle/make_golden.py's net_*.npz (inputs are
regenerated from the seeds by tests/util.net_case_inputs), plus `sub`: the head
maps `head_<name>` hold every sub-th row and column ([..., ::sub, ::sub]), and
`absmax_<name>` is max|head| over the whole map.  Only the names given
(default: all of RES_NET_CASES) are written; no other golden file is touched.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shims          # noqa: E402
from oracle.make_golden import GOLD, net_inputs      # noqa: E402
from centerpose_b200 import synth     # noqa: E402

RES_NET_CASES = [
    # name, arch, tracking, batch, H, W, weight seed, input seed, stored cell stride
    ("net_res18_b2_96x128", "res_18", False, 2, 96, 128, 21, 201, 1),
    ("net_res50_b1_64x64", "res_50", False, 1, 64, 64, 22, 202, 1),
    ("net_res18track_b1_64x96", "res_18", True, 1, 64, 96, 23, 203, 1),
    # the benched resolution at the depth opts.py:77-79 calls tested.  Its 128 x 128 maps are stored at every 3rd row
    # and column (an odd stride samples all four sub-pixel phases of the last transposed conv) with each head's max|head|
    # over the whole map, which keeps the fixture small.
    ("net_res101_b1_512", "res_101", False, 1, 512, 512, 24, 204, 3),
]


def make_res_net(only=None):
    import centerpose_b200 as cpb
    from lib.models.model import create_model as ref_create
    for name, arch, trk, B, H, W, wseed, iseed, sub in RES_NET_CASES:
        if only and name not in only:
            continue
        opt = ref_shims.make_opt(arch, tracking_task=trk)
        ours = cpb.create_model(opt.arch, opt.heads, opt.head_conv, cpb.default_opt(arch, tracking_task=trk))
        sd = synth.seeded_state_dict(ours, seed=wseed, offset_std=0.3)
        ref = ref_create(opt.arch, opt.heads, opt.head_conv, opt).eval()
        missing = ref.load_state_dict(sd, strict=True)
        x, extra = net_inputs(B, H, W, iseed, trk)
        with torch.no_grad():
            out = ref(torch.from_numpy(x), *[torch.from_numpy(extra[k]) if k in extra else None
                                             for k in ("pre_img", "pre_hm", "pre_hm_hp")])[-1]
        heads = {"head_" + k: v[..., ::sub, ::sub].numpy() for k, v in out.items()}
        heads.update({"absmax_" + k: float(v.abs().max()) for k, v in out.items()})
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), arch=arch, tracking=int(trk), batch=B, H=H, W=W,
                            wseed=wseed, iseed=iseed, offset_std=0.3, head_conv=int(opt.head_conv), sub=sub, **heads)
        print(name, {k: float(v.abs().max()) for k, v in out.items()}, missing)


if __name__ == "__main__":
    if not ref_shims.reference_available():
        raise SystemExit("reference tree not present: goldens can only be generated where it is")
    ref_shims.install()
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    make_res_net(set(sys.argv[1:]))

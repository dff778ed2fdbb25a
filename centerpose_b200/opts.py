"""Default configuration of the CenterPose inference path, for use WITHOUT the
reference tree (tests / bench on the GPU box).  When the reference's own
`opts().parse(...)`/`init(...)` Namespace is available it is consumed as-is;
this module only mirrors the fields the hot path reads, with the reference's
defaults (citations: /root/reference/src/lib/opts.py and src/demo.py).
"""
from types import SimpleNamespace

CATEGORIES = ("bike", "book", "bottle", "camera", "cereal_box", "chair", "cup", "mug", "laptop", "shoe")


def default_opt(arch="dla_34", tracking_task=False, rep_mode=1, c="chair", gpus="0", K=100,
                vis_thresh=0.3, show_axes=False, load_model="", input_res=512, debug=0):
    o = SimpleNamespace()
    o.task = "object_pose"                 # opts.py:19
    o.dataset = "objectron"
    o.arch = arch                          # opts.py:77
    o.head_conv = 256                      # opts.py:344-345 ('dla' in arch)
    o.down_ratio = 4                       # opts.py:85
    o.K = K                                # opts.py:120
    o.rep_mode = rep_mode                  # opts.py:211-220
    o.vis_thresh = vis_thresh              # opts.py:68
    o.c = c                                # opts.py:191
    o.show_axes = show_axes
    o.load_model = load_model
    o.debug = debug
    o.gpus = [0] if not str(gpus).startswith("-") else [-1]
    o.test_scales = [1.0]                  # opts.py:116
    o.fix_res = True                       # not keep_res (opts.py:337)
    o.fix_short = -1
    o.pad = 31
    o.input_h = o.input_w = input_res      # default_resolution 512 (opts.py:434)
    o.input_res = input_res
    o.output_h = o.output_w = input_res // 4
    o.mean = [0.408, 0.447, 0.470]         # opts.py:436-437
    o.std = [0.289, 0.274, 0.278]
    o.num_classes = 1
    o.flip_idx = [[1, 5], [3, 7], [2, 6], [4, 8]]
    o.balance_coefficient = {k: 2 for k in CATEGORIES}      # opts.py:239-241
    o.conf_border = [3, 9]
    o.R = 20
    o.max_age = 5
    # demo.py:113-149
    o.nms = True
    o.obj_scale = True
    o.use_pnp = True
    o.reg_offset = True
    o.reg_bbox = True
    o.hm_hp = True
    o.reg_hp_offset = True
    o.mse_loss = False
    o.tracking_task = bool(tracking_task)
    o.refined_Kalman = False
    o.pre_img = o.pre_hm = o.pre_hm_hp = bool(tracking_task)
    o.tracking = o.tracking_hp = bool(tracking_task)
    o.obj_scale_uncertainty = o.hps_uncertainty = bool(tracking_task)
    o.kalman = o.scale_pool = bool(tracking_task)
    o.hungarian = False                    # opts.py:295
    o.gt_pre_hm_hmhp = False               # opts.py:307-312
    o.gt_pre_hm_hmhp_first = False
    o.empty_pre_hm = False
    o.track_thresh = 0.1
    if tracking_task:
        o.vis_thresh = max(o.track_thresh, o.vis_thresh)
    o.cam_intrinsic = None
    # head table, opts.py:394-426 (insertion order matters: it is the state_dict order)
    heads = {"hm": 1, "wh": 2, "hps": 16}
    if o.hps_uncertainty:
        heads["hps_uncertainty"] = 16
    heads["reg"] = 2
    heads["hm_hp"] = 8
    heads["hp_offset"] = 2
    heads["scale"] = 3
    if o.obj_scale_uncertainty:
        heads["scale_uncertainty"] = 3
    if o.tracking:
        heads["tracking"] = 2
    if o.tracking_hp:
        heads["tracking_hp"] = 16
    o.heads = heads
    return o

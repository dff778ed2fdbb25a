"""Thin Python wrapper over the C ABI: one `Engine` = one native plan
(fixed arch / heads / resolution / max batch on one GPU) plus the output
buffers of the fused decode + PnP stage.  PyTorch only provides device
memory and the current stream here.
"""
import ctypes

import numpy as np
import torch

from . import _lib

HEAD_FIELDS = ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset", "scale", "hps_uncertainty",
               "scale_uncertainty", "tracking", "tracking_hp")
_VISIBLE = {"book": 6, "chair": 6, "cereal_box": 6, "camera": 3, "bottle": 3, "cup": 3,
            "bike": 0, "laptop": 0, "shoe": 0}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def decode_params(opt=None, **over):
    """cp_decode_params from a reference-style `opt` (or keyword overrides)."""
    g = lambda n, d: over.get(n, getattr(opt, n, d) if opt is not None else d)
    p = _lib.CpDecodeParams()
    p.num_classes = int(g("num_classes", 1))
    p.num_joints = 8
    p.K = int(g("K", 100))
    p.rep_mode = int(g("rep_mode", 1))
    p.use_moments = int(bool(g("tracking_task", False)) or bool(g("refined_Kalman", False)))
    scales = list(g("test_scales", [1.0]))
    p.nms = int(bool(g("nms", True)))
    # object_pose.py:188-193: merge_outputs reads detections[0] (the first scale) and forces the soft-NMS when several
    # scales were requested; `test_scale` is the scale of the pass being decoded (detector.run passes it per pass)
    p.num_scales = len(scales)
    p.test_scale = float(over.get("test_scale", scales[0] if scales else 1.0))
    cat = g("c", "chair")
    if cat not in _VISIBLE:
        raise ValueError("unknown category '%s' (cuboid_pnp_shell.py:59-66)" % cat)
    p.visible_thresh = _VISIBLE[cat]
    p.opencv_return = int(bool(g("show_axes", False)))
    # object_pose.py:136-138: hm always goes through sigmoid_, hm_hp only when not opt.mse_loss
    p.apply_sigmoid = int(over.get("apply_sigmoid", 2 if bool(g("mse_loss", False)) else 1))
    p.use_pnp = int(bool(g("use_pnp", True)))
    p.vis_thresh = float(g("vis_thresh", 0.3))
    bal = g("balance_coefficient", None)
    p.balance = float(bal[cat]) if isinstance(bal, dict) else float(bal if bal is not None else 2.0)
    # DESIGN.md section 5: 0 = the reference as pinned (torch==1.1.0 integer adds), 1 = the reference on torch >= 1.2
    p.modern_bool_semantics = int(bool(g("modern_bool_semantics", False)))
    if "use_moments" in over:
        p.use_moments = int(over["use_moments"])
    if "visible_thresh" in over:
        p.visible_thresh = int(over["visible_thresh"])
    return p


def make_meta(batch, c, s, img_w, img_h, cam, device=None, out=None):
    """[B,16] float64 meta rows (see centerpose_b200.h).  Scalars broadcast over the batch.  s is one scale for the
    batch, a 1-D array of exactly `batch` per-image scales, or [B,2] (w, h) pairs; a single (w, h) pair, as
    pre_process returns in the keep_res and fix_short modes, is reduced to its width by the caller
    (detector.scale_width)."""
    m = np.zeros((batch, _lib.CP_META_DOUBLES), np.float64)
    c = np.broadcast_to(np.asarray(c, np.float64).reshape(-1, 2), (batch, 2))
    m[:, 0:2] = c
    s_arr = np.asarray(s, np.float64)
    if s_arr.ndim == 0:
        m[:, 2] = float(s_arr)                 # one scalar for the whole batch
    elif s_arr.ndim == 1:
        if s_arr.shape[0] != batch:
            raise ValueError("make_meta: a 1-D s holds one scale per image; got %d values for a batch of %d (reduce a "
                             "(w, h) pair to its width first)" % (s_arr.shape[0], batch))
        m[:, 2] = s_arr                        # per-image scalar
    else:
        m[:, 2] = s_arr.reshape(batch, -1)[:, 0]     # [B,2] (w,h) pairs: the affine uses the width only
    m[:, 3] = img_w
    m[:, 4] = img_h
    m[:, 5:14] = np.broadcast_to(np.asarray(cam, np.float64).reshape(-1, 9), (batch, 9))
    t = torch.from_numpy(m)
    if device is not None:
        t = t.to(device)
    return t


def decode_pnp(heads, meta, prm, want_dets=True):
    """Run cp_decode_pnp on a dict of NCHW fp32 CUDA head tensors.
    Returns (dets [B,K,128] or None, poses [B,K,192], n_valid [B]) device tensors."""
    L = _lib.load()
    hm = heads["hm"]
    if not hm.is_cuda:
        raise RuntimeError("centerpose_b200.decode_pnp needs CUDA tensors (no CPU fallback)")
    B, _, H, W = hm.shape
    prm.batch, prm.out_h, prm.out_w = B, H, W
    hs = _lib.CpHeads()
    keep = []
    for f in HEAD_FIELDS:
        t = heads.get(f)
        if t is not None:
            t = t.contiguous().float()
            keep.append(t)
            setattr(hs, f, t.data_ptr())
    dev = hm.device
    meta = meta.to(dev, torch.float64).contiguous()
    dets = torch.empty((B, prm.K, _lib.CP_DETS_RECORD), dtype=torch.float32, device=dev) if want_dets else None
    poses = torch.empty((B, prm.K, _lib.CP_POSE_RECORD), dtype=torch.float32, device=dev)
    n_valid = torch.empty((B,), dtype=torch.int32, device=dev)
    nbytes = L.cp_decode_workspace_bytes(ctypes.byref(prm))
    if nbytes == 0:
        _lib.check(-1, "cp_decode_workspace_bytes")
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = L.cp_decode_pnp(ctypes.byref(prm), ctypes.byref(hs), _ptr(meta), _ptr(dets), _ptr(poses),
                             _ptr(n_valid), _ptr(ws), ctypes.c_size_t(nbytes), _stream())
    _lib.check(rc, "cp_decode_pnp")
    # the workspace must outlive the kernels; tie it to the outputs
    poses._cp_keep = (ws, keep, meta)
    return dets, poses, n_valid


class _CudaArray(object):
    """__cuda_array_interface__ of plan-owned fp32 device memory (torch.as_tensor wraps it without a copy)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 3}


def _device_view(ptr, n, device):
    with torch.cuda.device(device):
        return torch.as_tensor(_CudaArray(ptr, n), device=device)


ARCHS = {"dla_34": _lib.CP_ARCH_DLA34, "dlav1_34": _lib.CP_ARCH_DLAV1_34, "res_18": _lib.CP_ARCH_RES_18,
         "res_34": _lib.CP_ARCH_RES_34, "res_50": _lib.CP_ARCH_RES_50, "res_101": _lib.CP_ARCH_RES_101,
         "res_152": _lib.CP_ARCH_RES_152}      # cp_arch


def _config(arch, heads, head_conv, max_batch, height, width, device_index=0, tracking=False, tracking_task_gru=False,
            precision="fp32"):
    """(cp_config, the encoded head names it points to: keep them alive while the config is used)."""
    cfg = _lib.CpConfig()
    cfg.arch = ARCHS[arch]
    cfg.tracking = int(tracking)
    cfg.tracking_task_gru = int(tracking_task_gru)
    cfg.max_batch, cfg.height, cfg.width = int(max_batch), int(height), int(width)
    cfg.precision = _lib.PRECISIONS[precision]
    cfg.device = device_index
    cfg.head_conv = int(head_conv)
    names = [n.encode() for n in heads]
    cfg.num_heads = len(names)
    for i, (n, c) in enumerate(zip(names, heads.values())):
        cfg.head_names[i] = n
        cfg.head_channels[i] = int(c)
    return cfg, names


def _plan_flags(tracking, models, reuse_activations, batch_invariant=False):
    return ((_lib.CP_PLAN_MULTI_TRACK if tracking and models > 1 else 0) |
            (_lib.CP_PLAN_REUSE_ACTIVATIONS if reuse_activations else 0) |
            (_lib.CP_PLAN_BATCH_INVARIANT if batch_invariant else 0))


def plan_memory(arch, heads, head_conv, max_batch, height, width, tracking=False, tracking_task_gru=False,
                precision="fp32", models=1, reuse_activations=False, batch_invariant=False):
    """cp_plan_memory: the device bytes an Engine of these arguments owns, computed on the host without a GPU.
    dict(activation, weights, tiles, workspace, total)."""
    L = _lib.load()
    cfg, keep = _config(arch, dict(heads), head_conv, max_batch, height, width, 0, tracking, tracking_task_gru, precision)
    m = _lib.CpMemoryInfo()
    flags = _plan_flags(tracking, int(models), reuse_activations, batch_invariant)
    _lib.check(L.cp_plan_memory(ctypes.byref(cfg), int(models), flags, ctypes.byref(m)), "cp_plan_memory")
    out = dict(activation=int(m.activation_bytes), weights=int(m.weight_bytes), tiles=int(m.tile_bytes),
               workspace=int(m.workspace_bytes))
    out["total"] = sum(out.values())
    return out


def plan_ksegments(arch, heads, head_conv, max_batch, height, width, tracking=False, tracking_task_gru=False,
                   precision="fp32", models=1, reuse_activations=False, batch_invariant=False):
    """cp_plan_ksegments: the K segments of every op of an Engine of these arguments, on the host without a GPU.  With
    batch_invariant the fixed G of each op (1 where it never splits); without it 0 for every op."""
    L = _lib.load()
    cfg, keep = _config(arch, dict(heads), head_conv, max_batch, height, width, 0, tracking, tracking_task_gru, precision)
    flags = _plan_flags(tracking, int(models), reuse_activations, batch_invariant)
    n = ctypes.c_int32(0)
    buf = (ctypes.c_int32 * 1024)()
    _lib.check(L.cp_plan_ksegments(ctypes.byref(cfg), int(models), flags, buf, 1024, ctypes.byref(n)), "cp_plan_ksegments")
    return [int(buf[i]) for i in range(min(n.value, 1024))]


class Engine(object):
    """One native plan.  models > 1 (cp_plan_create_multi): `models` checkpoints of the same architecture run over the
    same frames, every layer one launch for all of them; load each with load_state_dict(sd, model=m).  forward / infer
    outputs then carry a leading [models] axis.  With tracking=True and models > 1 (cp_plan_create_multi_track) every
    model also takes its own previous-frame heat maps: pre_hm [models,B,1,H,W] and pre_hm_hp [models,B,8,H,W], while
    the frames and pre_img stay [B,...].

    reuse_activations=True (CP_PLAN_REUSE_ACTIVATIONS) packs the activation arena by liveness: the results are the same
    bits in a fraction of the memory, but the arena no longer holds every layer's output after a call, which the
    per-layer diagnostics (op_descs, arena, run_ops from the middle of the schedule) read.  `memory` is the byte
    breakdown of the plan (plan_memory).

    batch_invariant=True (CP_PLAN_BATCH_INVARIANT) fixes every launch's K reduction by the layer's shape: each frame's
    outputs are the same bits at any batch, in any row, with any number of models and on any SM count (README, "Batch
    invariance").  It costs no memory; the default plan is unchanged."""

    def __init__(self, arch, heads, head_conv, max_batch, height, width, device_index, tracking=False,
                 tracking_task_gru=False, precision="fp32", models=1, reuse_activations=False, batch_invariant=False):
        self.L = _lib.load()
        self.models = int(models)
        self.heads = dict(heads)
        self.head_names = list(heads.keys())
        self.max_batch, self.height, self.width = int(max_batch), int(height), int(width)
        self.device = torch.device("cuda", device_index)
        self.tracking = bool(tracking)
        self.reuse_activations = bool(reuse_activations)
        self.batch_invariant = bool(batch_invariant)
        cfg, self._names = _config(arch, self.heads, head_conv, max_batch, height, width, device_index, tracking,
                                   tracking_task_gru, precision)
        self._cfg = cfg
        plan = ctypes.c_void_p()
        flags = _plan_flags(self.tracking, self.models, self.reuse_activations, self.batch_invariant)
        with torch.cuda.device(self.device):
            _lib.check(self.L.cp_plan_create_ex(ctypes.byref(cfg), self.models, flags, ctypes.byref(plan)), "cp_plan_create")
        self.plan = plan
        self.weights_sig = None
        self.forward_launches = int(self.L.cp_plan_forward_launches(plan))
        self.plan_bytes = int(self.L.cp_plan_bytes(plan))
        self.memory = plan_memory(arch, heads, head_conv, max_batch, height, width, tracking, tracking_task_gru, precision,
                                  self.models, self.reuse_activations, self.batch_invariant)

    def close(self):
        if getattr(self, "plan", None):
            self.L.cp_plan_destroy(self.plan)
            self.plan = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state_dict(self, sd, model=0):
        names, ptrs, numel, keep = [], [], [], []
        for k, v in sd.items():
            if not torch.is_tensor(v) or not v.dtype.is_floating_point:
                continue
            t = v.detach().to(self.device, torch.float32).contiguous()
            keep.append(t)
            names.append(k.encode())
            ptrs.append(t.data_ptr())
            numel.append(t.numel())
        n = len(names)
        a_names = (ctypes.c_char_p * n)(*names)
        a_ptrs = (ctypes.c_void_p * n)(*ptrs)
        a_numel = (ctypes.c_int64 * n)(*numel)
        with torch.cuda.device(self.device):
            rc = self.L.cp_plan_load_weights_model(self.plan, int(model), a_names, a_ptrs, a_numel, n, _stream())
            _lib.check(rc, "cp_plan_load_weights")
            torch.cuda.current_stream().synchronize()   # borrowed tensors may be freed after this

    def _dev(self, t, name, shape):
        """Every tensor handed to the kernels by data_ptr() must be a contiguous fp32 tensor ON THE PLAN'S DEVICE: a
        CPU tensor or one on another GPU would become a wild device pointer (sticky illegal-address error).  Like the
        reference (`images.to(opt.device)`, base_detector.py:436-441) tensors that live elsewhere are moved."""
        if not torch.is_tensor(t):
            raise TypeError("%s must be a torch tensor" % name)
        if tuple(t.shape) != tuple(shape):
            raise ValueError("%s %s does not fit the plan: expected %s" % (name, tuple(t.shape), tuple(shape)))
        if t.device != self.device or t.dtype != torch.float32:
            t = t.to(self.device, torch.float32)
        return t.contiguous()

    def _check_inputs(self, x, pre_img, pre_hm, pre_hm_hp):
        B = x.shape[0]
        if x.dim() != 4 or tuple(x.shape[1:]) != (3, self.height, self.width) or B > self.max_batch or B < 1:
            raise ValueError("input %s does not fit the plan (%d,3,%d,%d)" % (tuple(x.shape), self.max_batch,
                                                                            self.height, self.width))
        xs = [self._dev(x, "images", (B, 3, self.height, self.width))]
        if self.tracking:
            if pre_img is None or pre_hm is None or pre_hm_hp is None:
                raise ValueError("a tracking plan needs pre_img, pre_hm and pre_hm_hp")
            lead = self._lead(B)          # the heat maps are per model on a multi-model plan
            xs += [self._dev(pre_img, "pre_img", (B, 3, self.height, self.width)),
                   self._dev(pre_hm, "pre_hm", lead + (1, self.height, self.width)),
                   self._dev(pre_hm_hp, "pre_hm_hp", lead + (8, self.height, self.width))]
        else:
            xs += [None, None, None]
        return B, xs

    def _out_tensor(self, t, name, shape, dtype):
        if t.device != self.device or t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
            raise ValueError("%s must be a contiguous %s tensor of shape %s on %s" % (name, dtype, tuple(shape), self.device))
        return t

    def _lead(self, B):
        """Leading axes of every output: (B,) or, on a multi-model plan, (models, B)."""
        return (self.models, B) if self.models > 1 else (B,)

    def _head_shape(self, B, c):
        return self._lead(B) + (c, self.height // 4, self.width // 4)

    def forward(self, x, pre_img=None, pre_hm=None, pre_hm_hp=None, out=None):
        """Head logits {name: [B,C,H/4,W/4] fp32 CUDA} ([models,B,C,H/4,W/4] on a multi-model plan)."""
        B, xs = self._check_inputs(x, pre_img, pre_hm, pre_hm_hp)
        if out is None:
            out = {n: torch.empty(self._head_shape(B, c), dtype=torch.float32, device=self.device)
                   for n, c in self.heads.items()}
        else:
            for n, c in self.heads.items():
                self._out_tensor(out[n], "out[%s]" % n, self._head_shape(B, c), torch.float32)
        hp = (ctypes.c_void_p * len(self.head_names))(*[out[n].data_ptr() for n in self.head_names])
        with torch.cuda.device(self.device):
            rc = self.L.cp_forward(self.plan, B, _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), _ptr(xs[3]), hp, _stream())
        _lib.check(rc, "cp_forward")
        return out

    def profile(self, x, pre_img=None, pre_hm=None, pre_hm_hp=None):
        """One forward with CUDA events between the ops: list of dicts(name, kind, ms, flops, bytes)."""
        B, xs = self._check_inputs(x, pre_img, pre_hm, pre_hm_hp)
        out = {n: torch.empty(self._head_shape(B, c), dtype=torch.float32, device=self.device)
               for n, c in self.heads.items()}
        hp = (ctypes.c_void_p * len(self.head_names))(*[out[n].data_ptr() for n in self.head_names])
        n_ops = int(self.L.cp_plan_num_ops(self.plan))
        stats = (_lib.CpOpStat * n_ops)()
        n = ctypes.c_int32(0)
        with torch.cuda.device(self.device):
            rc = self.L.cp_plan_profile(self.plan, B, _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), _ptr(xs[3]), hp, _stream(),
                                        stats, n_ops, ctypes.byref(n))
        _lib.check(rc, "cp_plan_profile")
        return [dict(name=stats[i].name.decode(), kind=int(stats[i].kind), ms=float(stats[i].ms),
                     flops=float(stats[i].flops), bytes=float(stats[i].bytes)) for i in range(n.value)]

    # ---- diagnostics (per-layer parity tests): the schedule as data, and one op at a time ----
    @staticmethod
    def _act(a):
        return dict(off=int(a.off), ext=int(a.ext), C=int(a.C), H=int(a.H), W=int(a.W), stride=int(a.stride))

    def op_descs(self, model=0):
        """cp_plan_op_desc_model of every op: list of dicts (device pointers as ints, activations as dicts of
        cp_act_desc), as model `model` sees them at max_batch."""
        out = []
        for i in range(int(self.L.cp_plan_num_ops(self.plan))):
            d = _lib.CpOpDesc()
            _lib.check(self.L.cp_plan_op_desc_model(self.plan, int(model), i, ctypes.byref(d)), "cp_plan_op_desc")
            r = {}
            for name, _ in _lib.CpOpDesc._fields_:
                v = getattr(d, name)
                if isinstance(v, _lib.CpActDesc):
                    v = self._act(v)
                elif name == "src":
                    v = [self._act(a) for a in v][:max(1, int(d.nsrc))]
                elif name == "children":
                    v = [int(c) for c in v][:int(d.n_children)]
                elif name == "name":
                    v = v.decode()
                elif v is None:
                    v = 0
                r[name] = v
            r["index"] = i
            out.append(r)
        return out

    def arena(self):
        """The activation arena as a flat fp32 CUDA tensor (a view of plan-owned memory, valid while the plan lives)."""
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        _lib.check(self.L.cp_plan_arena(self.plan, ctypes.byref(p), ctypes.byref(n)), "cp_plan_arena")
        return _device_view(p.value, int(n.value), self.device)

    def run_ops(self, x, first, last, out, pre_img=None, pre_hm=None, pre_hm_hp=None):
        """cp_plan_run_ops: ops [first, last) at batch x.shape[0] into the head tensors `out` (dict, as forward()).
        Returns one dict(family, BN, ksplit, grid) per op."""
        B, xs = self._check_inputs(x, pre_img, pre_hm, pre_hm_hp)
        for n, c in self.heads.items():
            self._out_tensor(out[n], "out[%s]" % n, self._head_shape(B, c), torch.float32)
        hp = (ctypes.c_void_p * len(self.head_names))(*[out[n].data_ptr() for n in self.head_names])
        n = max(0, last - first)
        info = (_lib.CpOpLaunch * max(1, n))()
        with torch.cuda.device(self.device):
            rc = self.L.cp_plan_run_ops(self.plan, B, first, last, _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), _ptr(xs[3]),
                                        hp, _stream(), info)
        _lib.check(rc, "cp_plan_run_ops")
        return [dict(family=int(info[i].family), BN=int(info[i].BN), ksplit=int(info[i].ksplit),
                     grid=int(info[i].grid)) for i in range(n)]

    def op_ksegments(self, i):
        """cp_plan_op_ksegments of op i: dict(segments = the fixed G of a batch-invariant plan, 0 in a default one;
        last_segments, last_path = the split-K factor and cp_kpath (_lib.KPATH_*) of the op's latest launch)."""
        g, ls, lp = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        _lib.check(self.L.cp_plan_op_ksegments(self.plan, int(i), ctypes.byref(g), ctypes.byref(ls), ctypes.byref(lp)),
                   "cp_plan_op_ksegments")
        return dict(segments=int(g.value), last_segments=int(ls.value), last_path=int(lp.value))

    def infer(self, x, meta, prm, pre_img=None, pre_hm=None, pre_hm_hp=None, heads_out=None, want_dets=False,
              poses=None, n_valid=None, dets=None):
        """forward + decode + PnP in one native call.  Returns (dets|None, poses, n_valid).  On a multi-model plan `prm`
        is one cp_decode_params per model (cp_infer_multi) and the outputs are [models, B, ...]."""
        B, xs = self._check_inputs(x, pre_img, pre_hm, pre_hm_hp)
        lead = self._lead(B)
        if not torch.is_tensor(meta) or tuple(meta.shape) != (B, _lib.CP_META_DOUBLES):
            raise ValueError("meta must be a [%d,%d] tensor (make_meta)" % (B, _lib.CP_META_DOUBLES))
        if meta.device != self.device or meta.dtype != torch.float64 or not meta.is_contiguous():
            meta = meta.to(self.device, torch.float64).contiguous()
        if self.models > 1:
            prms = list(prm)
            if len(prms) != self.models:
                raise ValueError("a plan of %d models needs %d decode parameter sets, got %d" % (self.models, self.models,
                                                                                                len(prms)))
            K = prms[0].K
        else:
            K = prm.K
        if poses is None:
            poses = torch.empty(lead + (K, _lib.CP_POSE_RECORD), dtype=torch.float32, device=self.device)
        else:
            self._out_tensor(poses, "poses", lead + (K, _lib.CP_POSE_RECORD), torch.float32)
        if n_valid is None:
            n_valid = torch.empty(lead, dtype=torch.int32, device=self.device)
        else:
            self._out_tensor(n_valid, "n_valid", lead, torch.int32)
        if want_dets and dets is None:
            dets = torch.empty(lead + (K, _lib.CP_DETS_RECORD), dtype=torch.float32, device=self.device)
        elif dets is not None:
            self._out_tensor(dets, "dets", lead + (K, _lib.CP_DETS_RECORD), torch.float32)
        hp = None
        if heads_out is not None:
            for n, c in self.heads.items():
                self._out_tensor(heads_out[n], "heads_out[%s]" % n, self._head_shape(B, c), torch.float32)
            hp = (ctypes.c_void_p * len(self.head_names))(*[heads_out[n].data_ptr() for n in self.head_names])
        with torch.cuda.device(self.device):
            if self.models > 1 and self.tracking:
                arr = (_lib.CpDecodeParams * self.models)(*prms)
                rc = self.L.cp_infer_multi_track(self.plan, B, _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), _ptr(xs[3]), arr,
                                                 _ptr(meta), hp, _ptr(dets), _ptr(poses), _ptr(n_valid), _stream())
            elif self.models > 1:
                arr = (_lib.CpDecodeParams * self.models)(*prms)
                rc = self.L.cp_infer_multi(self.plan, B, _ptr(xs[0]), arr, _ptr(meta), hp, _ptr(dets), _ptr(poses),
                                           _ptr(n_valid), _stream())
            else:
                rc = self.L.cp_infer(self.plan, B, _ptr(xs[0]), _ptr(xs[1]), _ptr(xs[2]), _ptr(xs[3]), ctypes.byref(prm),
                                     _ptr(meta), hp, _ptr(dets), _ptr(poses), _ptr(n_valid), _stream())
        _lib.check(rc, ("cp_infer_multi_track" if self.tracking else "cp_infer_multi") if self.models > 1 else "cp_infer")
        return dets, poses, n_valid


class InferGraph(object):
    """cp_infer captured once in a CUDA graph (static buffers): a step is two small copies + one graph launch instead of
    ~80 kernel launches driven from the host -- what matters at batch 1, where the launch sequence, not the kernels,
    sets the latency.  `graph(x, meta)` -> (poses, n_valid) (views of the graph's own output buffers)."""

    def __init__(self, eng, batch, prm, tracking=False):
        self.eng, self.prm = eng, prm
        dev = eng.device
        H, W = eng.height, eng.width
        self.x = torch.zeros((batch, 3, H, W), dtype=torch.float32, device=dev)
        self.meta = torch.zeros((batch, _lib.CP_META_DOUBLES), dtype=torch.float64, device=dev)
        self.meta[:, 2] = float(max(H, W))
        self.meta[:, 3], self.meta[:, 4] = W, H
        self.meta[:, 5], self.meta[:, 9], self.meta[:, 13] = 1.0, 1.0, 1.0
        self.pre = None
        if tracking:
            self.pre = (torch.zeros_like(self.x), torch.zeros((batch, 1, H, W), dtype=torch.float32, device=dev),
                        torch.zeros((batch, 8, H, W), dtype=torch.float32, device=dev))
        self.poses = torch.zeros((batch, prm.K, _lib.CP_POSE_RECORD), dtype=torch.float32, device=dev)
        self.n_valid = torch.zeros((batch,), dtype=torch.int32, device=dev)
        pre = self.pre if self.pre is not None else (None, None, None)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):            # warm-up outside the capture: lazy allocations, launch attributes
            for _ in range(2):
                eng.infer(self.x, self.meta, prm, *pre, poses=self.poses, n_valid=self.n_valid)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            eng.infer(self.x, self.meta, prm, *pre, poses=self.poses, n_valid=self.n_valid)

    def __call__(self, x, meta, pre_img=None, pre_hm=None, pre_hm_hp=None):
        self.x.copy_(x, non_blocking=True)
        self.meta.copy_(meta, non_blocking=True)
        if self.pre is not None:
            for dst, src in zip(self.pre, (pre_img, pre_hm, pre_hm_hp)):
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.poses, self.n_valid


def preprocess(frames_u8, dst_h, dst_w, mean, std, out=None, trans_input=None, resize_hw=None):
    """cp_preprocess: uint8 [B,H,W,3] CUDA -> fp32 [B,3,dst_h,dst_w] CUDA (bit-exact cv2.warpAffine + normalise).
    trans_input: optional 2x3 forward affine (meta['trans_input']); default = the fix_res affine of the frame size.
    resize_hw: (rh, rw) to warp cv2.resize(frame, (rw, rh)) instead of the frame, as pre_process does at a test scale
    (cp_preprocess_resize_affine); trans_input then maps the resized image and must be given."""
    L = _lib.load()
    if not frames_u8.is_cuda or frames_u8.dtype != torch.uint8:
        raise RuntimeError("preprocess needs a uint8 CUDA tensor")
    if resize_hw is not None and trans_input is None:
        raise ValueError("preprocess: resize_hw needs the trans_input of the resized image")
    B, sh, sw, _ = frames_u8.shape
    if out is None:
        out = torch.empty((B, 3, dst_h, dst_w), dtype=torch.float32, device=frames_u8.device)
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(frames_u8.device):
        if trans_input is not None:
            tm = (ctypes.c_double * 6)(*[float(v) for v in np.asarray(trans_input, np.float64).reshape(-1)])
            if resize_hw is not None:
                rc = L.cp_preprocess_resize_affine(_ptr(frames_u8.contiguous()), _ptr(out), B, sh, sw, int(resize_hw[0]),
                                                   int(resize_hw[1]), dst_h, dst_w, tm, m, s, _stream())
            else:
                rc = L.cp_preprocess_affine(_ptr(frames_u8.contiguous()), _ptr(out), B, sh, sw, dst_h, dst_w, tm, m, s,
                                            _stream())
        else:
            rc = L.cp_preprocess(_ptr(frames_u8.contiguous()), _ptr(out), B, sh, sw, dst_h, dst_w, m, s, _stream())
    _lib.check(rc, "cp_preprocess")
    return out


def is_jpeg(data):
    """True for encoded bytes that start like a JPEG file (FF D8 FF)."""
    return len(data) >= 3 and bytes(data[:3]) == b"\xff\xd8\xff"


def jpeg_bytes(frame):
    """An encoded JPEG as run_batch(pixel_format="jpeg") takes it (bytes, a 1-D uint8 numpy array or CPU tensor) ->
    a contiguous uint8 numpy array, or None for anything else."""
    if isinstance(frame, (bytes, bytearray, memoryview)):
        return np.frombuffer(frame, np.uint8)
    if isinstance(frame, np.ndarray) and frame.dtype == np.uint8 and frame.ndim == 1:
        return np.ascontiguousarray(frame)
    if isinstance(frame, torch.Tensor) and frame.dtype == torch.uint8 and frame.dim() == 1 and not frame.is_cuda:
        return frame.contiguous().numpy()
    return None


def jpeg_parse(data):
    """cp_jpeg_parse of one encoded file (a uint8 numpy array) -> its CpJpegHeader; header.status is 0 for a supported
    file, else the cp_jpeg_refusal (_lib.JPEG_REFUSALS names it)."""
    L = _lib.load()
    h = _lib.CpJpegHeader()
    L.cp_jpeg_parse(data.ctypes.data_as(ctypes.c_void_p), len(data), ctypes.byref(h))
    return h


def jpeg_decode(headers, bytes_u8, byte_offsets, out_u8, out_offsets, subseq_words=0):
    """cp_jpeg_decode: the parsed JPEGs whose files start byte_offsets[b] into bytes_u8 (uint8 CUDA) decoded, bit for
    bit cv2.imdecode, into uint8 BGR [out_h, out_w, 3] at out_offsets[b] of out_u8 (uint8 CUDA).  Returns the int32 CUDA
    error word of each frame (0: decoded exactly; else _lib.JPEG_ERR_* bits)."""
    L = _lib.load()
    B = len(headers)
    hs = (_lib.CpJpegHeader * B)(*headers)
    dev = bytes_u8.device
    ws_bytes = L.cp_jpeg_workspace_bytes(hs, B)
    if ws_bytes == 0:
        _lib.check(-1, "cp_jpeg_workspace_bytes")
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    errors = torch.empty((B,), dtype=torch.int32, device=dev)
    bo = (ctypes.c_int64 * B)(*[int(v) for v in byte_offsets])
    oo = (ctypes.c_int64 * B)(*[int(v) for v in out_offsets])
    with torch.cuda.device(dev):
        rc = L.cp_jpeg_decode(hs, B, _ptr(bytes_u8), bo, _ptr(out_u8), oo, _ptr(ws), ctypes.c_size_t(ws_bytes),
                              _ptr(errors), int(subseq_words), _stream())
    _lib.check(rc, "cp_jpeg_decode")
    return errors


def jpeg_error_text(word):
    """The cp_jpeg_error bits of a frame's error word, in words."""
    return ", ".join(v for k, v in sorted(_lib.JPEG_ERRORS.items()) if int(word) & k)


def _preprocess_packed(who, packed_u8, offsets, src_hw, fmt, dst_h, dst_w, mean, std, out, trans_input):
    """The call of cp_<who> on B frames packed into one buffer: (packed_u8, its bytes, offsets, src_hw, *fmt, out, B,
    dst_h, dst_w, trans_input, mean, std, stream), fmt being the entry point's format argument, if it has one."""
    L = _lib.load()
    if not packed_u8.is_cuda or packed_u8.dtype != torch.uint8 or not packed_u8.is_contiguous():
        raise RuntimeError("%s needs a contiguous uint8 CUDA buffer" % who)
    offs = np.ascontiguousarray(offsets, np.int64).reshape(-1)
    hw = np.ascontiguousarray(src_hw, np.int32).reshape(-1, 2)
    B = offs.shape[0]
    if hw.shape[0] != B:
        raise ValueError("%s: %d offsets for %d frame sizes" % (who, B, hw.shape[0]))
    if out is None:
        out = torch.empty((B, 3, dst_h, dst_w), dtype=torch.float32, device=packed_u8.device)
    tm = None
    if trans_input is not None:
        tr = np.ascontiguousarray(trans_input, np.float64).reshape(-1)
        if tr.shape[0] != 6 * B:
            raise ValueError("%s: trans_input must hold %d 2x3 matrices" % (who, B))
        tm = tr.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    s = (ctypes.c_float * 3)(*[float(v) for v in std])
    with torch.cuda.device(packed_u8.device):
        rc = getattr(L, "cp_" + who)(_ptr(packed_u8), packed_u8.numel(), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                     hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), *fmt, _ptr(out), B, dst_h, dst_w,
                                     tm, m, s, _stream())
    _lib.check(rc, "cp_" + who)
    return out


def preprocess_ragged(packed_u8, offsets, src_hw, dst_h, dst_w, mean, std, out=None, trans_input=None):
    """cp_preprocess_ragged: B frames of different sizes in one launch.  packed_u8: flat uint8 CUDA buffer holding frame b
    (uint8 [src_hw[b][0], src_hw[b][1], 3]) at byte offsets[b] -> fp32 [B,3,dst_h,dst_w] CUDA, frame b bit for bit what
    `preprocess` gives for it alone.  trans_input: optional [B,2,3] forward affines; default = each frame's fix_res affine."""
    return _preprocess_packed("preprocess_ragged", packed_u8, offsets, src_hw, (), dst_h, dst_w, mean, std, out,
                              trans_input)


_YUV420 = {"nv12": _lib.CP_PIX_NV12, "i420": _lib.CP_PIX_I420}
# the buffer of one H x W image in each pixel_format: [3H/2,W] for YUV 4:2:0, [H,W] for the sensor formats, else
# [H,W,C]
_LAYOUT = dict({"bgr": "[H,W,3]", "nv12": "[3H/2,W]", "i420": "[3H/2,W]", "rgb24": "[H,W,3]", "rgba": "[H,W,4]",
                "bgra": "[H,W,4]", "yuyv422": "[H,W,2]", "uyvy422": "[H,W,2]"},
               **{f: "[H,W]" for f in _lib.SENSOR_FORMATS})
_CHANNELS = {"bgr": 3, "rgb24": 3, "rgba": 4, "bgra": 4, "yuyv422": 2, "uyvy422": 2}
_ALL_FORMATS = _lib.PIXEL_FORMATS + _lib.SENSOR_FORMATS


# encoded JPEG frames: not a cp_pixel_format (the pre-process never sees one); run_batch(list) decodes them to BGR first
JPEG = "jpeg"


# an MJPEG camera: encoded baseline JPEG frames of one decoded size, which the live-video graphs decode (graph.py)
MJPEG = "mjpeg"


def _refuse_jpeg(pixel_format):
    if isinstance(pixel_format, str) and pixel_format == JPEG:
        raise ValueError("pixel_format \"jpeg\" takes encoded JPEG frames, which have no fixed shape to stage or capture: "
                         "pass them as a list to run_batch(list, pixel_format=\"jpeg\")")
    if isinstance(pixel_format, str) and pixel_format == MJPEG:
        raise ValueError("pixel_format \"mjpeg\" is an MJPEG camera of one frame size, decoded inside the live-video "
                         "graphs (DetectGraph, TrackGraph and their multi-category forms); encoded frames of any size go "
                         "as a list to run_batch(list, pixel_format=\"jpeg\")")


def _min_side(pixel_format):
    """The least height and width of a frame in a sensor format: a Bayer mosaic's demosaic needs 3 x 3 pixels."""
    return 3 if pixel_format.startswith("bayer_") else 1


def check_pixel_format(pixel_format):
    """pixel_format (cp_pixel_format): "bgr" (uint8 [H,W,3], cv2.imread's), "nv12" or "i420" (uint8 [3H/2,W], H and W
    even), a camera format named as ffmpeg's pix_fmt: "rgb24" ([H,W,3]), "rgba" / "bgra" ([H,W,4], alpha ignored),
    "yuyv422" / "uyvy422" ([H,W,2] packed YUV 4:2:2, W even), or a sensor format, one [H,W] plane: "gray" (mono) or a
    Bayer mosaic "bayer_rggb8" / "bayer_bggr8" / "bayer_gbrg8" / "bayer_grbg8" (H and W at least 3), demosaiced as
    cv2's bilinear COLOR_Bayer??2BGR.  One name; a list (one per camera) goes through slot_formats where frames come as
    a list."""
    if isinstance(pixel_format, (list, tuple)):
        raise ValueError("pixel_format must be one name here, got a list %r; one name per camera goes with a list of "
                         "frames (run_batch(list), a graph built with one frame_hw per slot)" % (list(pixel_format),))
    _refuse_jpeg(pixel_format)
    if pixel_format not in _ALL_FORMATS:
        raise ValueError("pixel_format must be one of %s, got %r" % (", ".join(_ALL_FORMATS), pixel_format))
    return pixel_format


def slot_formats(pixel_format, n, who="run_batch"):
    """The pixel formats of n frames or slots: one name for all of them, or a list of n names (one per camera)."""
    if not isinstance(pixel_format, (list, tuple)):
        return [check_pixel_format(pixel_format)] * n
    if len(pixel_format) != n:
        raise ValueError("%s: pixel_format is one name or one per frame, got %d names for %d frames"
                         % (who, len(pixel_format), n))
    for f in pixel_format:
        _refuse_jpeg(f)
        if isinstance(f, (list, tuple)) or f not in _ALL_FORMATS:
            raise ValueError("pixel_format must be one of %s, got %r in %r"
                             % (", ".join(_ALL_FORMATS), f, list(pixel_format)))
    return list(pixel_format)


def frame_layout(pixel_format):
    """"[H,W,3]", "[3H/2,W]", ...: the buffer of one image in pixel_format, for messages."""
    return _LAYOUT[check_pixel_format(pixel_format)]


def frame_shape(h, w, pixel_format):
    """The buffer shape of one h x w image in pixel_format: [h,w,3] for "bgr" / "rgb24", [h,w,4] for "rgba" / "bgra",
    [h,w,2] for "yuyv422" / "uyvy422" (w even), [3h/2,w] for "nv12" / "i420" (h and w even), [h,w] for "gray" and the
    Bayer mosaics (h and w at least 3); else ValueError."""
    if check_pixel_format(pixel_format) in _lib.SENSOR_FORMATS:
        m = _min_side(pixel_format)
        if h < m or w < m:
            raise ValueError("%s frames need at least %d x %d pixels; got %d x %d" % (pixel_format, m, m, h, w))
        return (int(h), int(w))
    c = _CHANNELS.get(pixel_format)
    if c is not None:
        if c == 2 and (w % 2 or h < 1 or w < 2):
            raise ValueError("%s frames need an even, positive width; got %d x %d" % (pixel_format, h, w))
        return (int(h), int(w), c)
    if h % 2 or w % 2 or h < 2 or w < 2:
        raise ValueError("%s frames need an even, positive image size; got %d x %d" % (pixel_format, h, w))
    return (int(h) * 3 // 2, int(w))


def image_size(shape, pixel_format, what="frame"):
    """(H, W) of the image a buffer of `shape` holds in pixel_format; ValueError (naming the expected shape) when the
    shape is not one of that format."""
    shape = tuple(int(v) for v in shape)
    if check_pixel_format(pixel_format) in _lib.SENSOR_FORMATS:
        m = _min_side(pixel_format)
        if len(shape) != 2 or shape[0] < m or shape[1] < m:
            raise ValueError("%s has shape %s, expected a %s frame [H,W]%s" % (what, shape, pixel_format,
                                                                              " with H and W at least 3" if m > 1 else ""))
        return shape
    c = _CHANNELS.get(pixel_format)
    if c is not None:
        if len(shape) != 3 or shape[2] != c or shape[0] < 1 or shape[1] < 1 or (c == 2 and shape[1] % 2):
            raise ValueError("%s has shape %s, expected %s[H,W,%d]%s" % (what, shape, "" if c == 3 else "a %s frame "
                                                                        % pixel_format, c, " with W even" if c == 2 else ""))
        return shape[0], shape[1]
    if len(shape) == 2 and shape[0] % 3 == 0:
        h, w = shape[0] * 2 // 3, shape[1]
        if h >= 2 and w >= 2 and h % 2 == 0 and w % 2 == 0:
            return h, w
    raise ValueError("%s has shape %s, expected a %s frame [3H/2,W] with H and W even" % (what, shape, pixel_format))


def preprocess_formats(packed_u8, offsets, src_hw, pixel_format, dst_h, dst_w, mean, std, out=None, trans_input=None):
    """cp_preprocess_formats: preprocess_ragged for frames in any pixel_format, one name for every frame or a list of B
    names (one per frame).  packed_u8: flat uint8 CUDA buffer holding frame b (its pixel format's buffer of image size
    src_hw[b]) at byte offsets[b] -> fp32 [B,3,dst_h,dst_w] CUDA, frame b bit for bit what preprocess_ragged gives for
    cv2.cvtColor(frame) to BGR.  trans_input: optional [B,2,3] forward affines; default = each frame's fix_res affine."""
    _lib.load()
    codes = np.array([_lib.PIXEL_FORMAT_CODES[f] for f in slot_formats(pixel_format, np.size(offsets),
                                                                       "preprocess_formats")], np.int32)
    return _preprocess_packed("preprocess_formats", packed_u8, offsets, src_hw,
                              (codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),), dst_h, dst_w, mean, std, out,
                              trans_input)


def map_pointers(maps, n, dst_h, dst_w, device, who):
    """The host array of n device pointers of cp_preprocess_remap / cp_preprocess_frame_table_maps: maps is a list of n
    float32 [dst_h, dst_w, 2] contiguous CUDA tensors on `device` (lens.undistort_map's layout), None for a frame that
    keeps its affine.  The caller keeps the tensors alive while a launch can read them."""
    maps = list(maps)
    if len(maps) != n:
        raise ValueError("%s: %d maps for %d frames" % (who, len(maps), n))
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    for b, m in enumerate(maps):
        if m is not None and (not torch.is_tensor(m) or m.dtype != torch.float32 or tuple(m.shape) != (dst_h, dst_w, 2)
                              or m.device != device or not m.is_contiguous()):
            raise ValueError("%s: map %d must be a contiguous float32 [%d,%d,2] tensor on %s, got %s"
                             % (who, b, dst_h, dst_w, device, (m.dtype, tuple(m.shape), str(m.device))
                                if torch.is_tensor(m) else type(m).__name__))
    return (ctypes.c_void_p * n)(*[None if m is None else m.data_ptr() for m in maps])


def preprocess_remap(packed_u8, offsets, src_hw, pixel_format, maps, dst_h, dst_w, mean, std, out=None,
                     trans_input=None):
    """cp_preprocess_remap: preprocess_formats with a coordinate map per frame (lens distortion).  maps: one float32
    [dst_h, dst_w, 2] CUDA tensor per frame, or None for a frame that keeps its affine (trans_input[b], or its fix_res
    affine).  A mapped frame's output is bit for bit cv2.remap(cv2.cvtColor(frame) to BGR, map x, map y, INTER_LINEAR,
    BORDER_CONSTANT, 0), normalised."""
    _lib.load()
    B = int(np.size(offsets))
    codes = np.array([_lib.PIXEL_FORMAT_CODES[f] for f in slot_formats(pixel_format, B, "preprocess_remap")], np.int32)
    ptrs = map_pointers(maps, B, dst_h, dst_w, packed_u8.device, "preprocess_remap")
    return _preprocess_packed("preprocess_remap", packed_u8, offsets, src_hw,
                              (codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ptrs), dst_h, dst_w, mean, std,
                              out, trans_input)


def preprocess_yuv420(packed_u8, offsets, src_hw, pixel_format, dst_h, dst_w, mean, std, out=None, trans_input=None):
    """cp_preprocess_yuv420: preprocess_ragged for YUV 4:2:0 frames.  packed_u8: flat uint8 CUDA buffer holding frame b
    (uint8 [3H/2,W] in pixel_format "nv12" or "i420", (H, W) = src_hw[b], both even) at byte offsets[b] -> fp32
    [B,3,dst_h,dst_w] CUDA, frame b bit for bit what preprocess_ragged gives for cv2.cvtColor(frame, COLOR_YUV2BGR_*).
    trans_input: optional [B,2,3] forward affines; default = each frame's fix_res affine (that of `preprocess`)."""
    _lib.load()
    if pixel_format not in _YUV420:
        raise ValueError("preprocess_yuv420: pixel_format must be 'nv12' or 'i420', got %r" % (pixel_format,))
    return _preprocess_packed("preprocess_yuv420", packed_u8, offsets, src_hw, (_YUV420[pixel_format],), dst_h, dst_w,
                              mean, std, out, trans_input)


def conv2d_nhwc(x, weight, bias=None, residual=None, stride=1, pad=0, relu=False, precision="fp32"):
    """cp_conv2d: x [B,H,W,Cin] NHWC fp32 CUDA, weight OIHW -> [B,Ho,Wo,Cout] NHWC."""
    L = _lib.load()
    if not x.is_cuda:
        raise RuntimeError("centerpose_b200 conv2d_nhwc needs CUDA tensors (no CPU fallback)")
    B, H, W, Cin = x.shape
    Cout, _, k, _ = weight.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    out = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    ts = [t.contiguous().float() if t is not None else None for t in (x, weight, bias, residual)]
    with torch.cuda.device(x.device):
        rc = L.cp_conv2d(_ptr(ts[0]), _ptr(ts[1]), _ptr(ts[2]), _ptr(ts[3]), _ptr(out), B, H, W, Cin, Cout, k, stride,
                         pad, int(relu), _lib.PRECISIONS[precision], _stream())
    _lib.check(rc, "cp_conv2d")
    return out


def dcn_v2_forward(inp, weight, bias, offset, mask, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, dh=1, dw=1, dg=1,
                   precision="fp32"):
    """`_ext.dcn_v2_forward` signature (DCNv2/src/vision.cpp:4-9) on top of cp_dcn_v2_forward."""
    if (kh, kw, sh, sw, ph, pw, dh, dw, dg) != (3, 3, 1, 1, 1, 1, 1, 1, 1):
        raise RuntimeError("centerpose_b200 dcn_v2_forward: only 3x3 / stride 1 / pad 1 / dilation 1 / "
                           "deformable_group 1 is implemented (the configuration CenterPose uses)")
    if not inp.is_cuda:
        raise RuntimeError("centerpose_b200 dcn_v2_forward needs CUDA tensors (no CPU fallback)")
    L = _lib.load()
    B, C, H, W = inp.shape
    Co = weight.shape[0]
    out = torch.empty((B, Co, H, W), dtype=torch.float32, device=inp.device)
    ts = [t.contiguous().float() for t in (inp, weight, bias, offset, mask)]
    with torch.cuda.device(inp.device):
        rc = L.cp_dcn_v2_forward_ex(_ptr(ts[0]), _ptr(ts[1]), _ptr(ts[2]), _ptr(ts[3]), _ptr(ts[4]), _ptr(out),
                                    B, C, H, W, Co, _lib.PRECISIONS[precision], _stream())
    _lib.check(rc, "cp_dcn_v2_forward")
    out._cp_keep = ts
    return out


def dcn_v2_backward(inp, weight, bias, offset, mask, grad_output, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, dh=1, dw=1, dg=1,
                    precision="fp32"):
    """`_ext.dcn_v2_backward` signature (DCNv2/src/vision.cpp:11-17, dcn_v2.py:63-76) on top of cp_dcn_v2_backward.
    Returns (grad_input, grad_offset, grad_mask, grad_weight, grad_bias) as fresh tensors, like the reference."""
    if (kh, kw, sh, sw, ph, pw, dh, dw, dg) != (3, 3, 1, 1, 1, 1, 1, 1, 1):
        raise RuntimeError("centerpose_b200 dcn_v2_backward: only 3x3 / stride 1 / pad 1 / dilation 1 / "
                           "deformable_group 1 is implemented (the configuration CenterPose uses)")
    if not inp.is_cuda:
        raise RuntimeError("centerpose_b200 dcn_v2_backward needs CUDA tensors (no CPU fallback)")
    L = _lib.load()
    B, C, H, W = inp.shape
    Co = weight.shape[0]
    ts = [t.contiguous().float() for t in (inp, weight, offset, mask, grad_output)]
    for t, shape in zip(ts, ((B, C, H, W), (Co, C, 3, 3), (B, 18, H, W), (B, 9, H, W), (B, Co, H, W))):
        if tuple(t.shape) != shape or t.device != inp.device:
            raise ValueError("dcn_v2_backward: expected a %s tensor on %s, got %s on %s" % (shape, inp.device, tuple(t.shape), t.device))
    grads = [torch.empty_like(ts[0]), torch.empty_like(ts[2]), torch.empty_like(ts[3]), torch.empty_like(ts[1]),
             torch.empty((Co,), dtype=torch.float32, device=inp.device)]
    with torch.cuda.device(inp.device):
        rc = L.cp_dcn_v2_backward(*[_ptr(t) for t in ts], *[_ptr(g) for g in grads], B, C, H, W, Co,
                                  _lib.PRECISIONS[precision], _stream())
    _lib.check(rc, "cp_dcn_v2_backward")
    return tuple(grads)

/*
 * centerpose_b200.h -- C ABI of libcenterpose_b200.so (sm_90a).
 *
 * The drop-in boundary for the CenterPose inference hot path
 * (SURVEY.md section 8b).  Plain pointers and sizes only; every function
 * returns 0 on success or a negative cp_status, and cp_last_error() returns a
 * thread-local message.  The library never allocates in steady state: the
 * caller (PyTorch on the Python side) owns every input / output buffer, a
 * plan owns its packed weights and activation arena.  All device work is
 * enqueued on the cudaStream_t passed as `stream` (pass
 * torch.cuda.current_stream().cuda_stream); no call synchronises the device
 * unless documented.
 *
 * Reference interfaces each entry point replaces (paths relative to
 * /root/reference/src/lib):
 *
 *   cp_plan_create / cp_plan_load_weights / cp_plan_destroy
 *       models/model.py:26-31 create_model(), :34-87 load_model()
 *       models/networks/pose_dla_dcn.py:457-521 DLASeg.__init__, :573-590 factories
 *   cp_forward
 *       models/networks/pose_dla_dcn.py:523-570 DLASeg.forward
 *       (DLA :310-322, DLAUp :437-443, IDAUp :411-417, DeformConv :377-389,
 *        convGRU.py:72-94, GN.py:4-9)
 *   cp_dcn_v2_forward
 *       models/networks/DCNv2/src/vision.cpp:4-9  _ext.dcn_v2_forward
 *       models/networks/DCNv2/src/dcn_v2.h:9-45, src/cuda/dcn_v2_cuda.cu:42-172,
 *       src/cuda/dcn_v2_im2col_cuda.cu:125-195
 *   cp_decode_pnp
 *       detectors/object_pose.py:131-165 process() [sigmoid + object_pose_decode]
 *       models/decode.py:72-375, utils/post_process.py:12-68,
 *       detectors/object_pose.py:184-197 merge_outputs + :27-124 soft_nms_nvidia,
 *       detectors/base_detector.py:548-654 point assembly + pnp_shell,
 *       utils/pnp/cuboid_pnp_shell.py:11-93, utils/pnp/cuboid_pnp_solver.py:91-239
 *   cp_infer
 *       detectors/base_detector.py:473-654 (process -> post_process -> merge -> PnP)
 *   cp_preprocess / cp_preprocess_affine / cp_preprocess_ragged / cp_preprocess_yuv420 / cp_preprocess_formats /
 *   cp_preprocess_resize_affine
 *       detectors/base_detector.py:91-148 pre_process (resize + affine warp + normalise)
 *   cp_jpeg_parse / cp_jpeg_decode
 *       detectors/base_detector.py:412 cv2.imread of run()'s image path (libjpeg-turbo's baseline decoder)
 */
#ifndef CENTERPOSE_B200_H_
#define CENTERPOSE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CP_ABI_VERSION 1

/* ---- status codes --------------------------------------------------------- */
enum cp_status {
  CP_OK = 0,
  CP_ERR_INVALID = -1,      /* bad argument / unsupported configuration        */
  CP_ERR_CUDA = -2,         /* a CUDA runtime call failed (message has details) */
  CP_ERR_NOT_LOADED = -3,   /* plan used before cp_plan_load_weights           */
  CP_ERR_MISSING_KEY = -4,  /* a state_dict key the plan needs was not supplied */
  CP_ERR_SHAPE = -5         /* tensor element count does not match the plan     */
};

/* ---- architecture / precision -------------------------------------------- */
enum cp_arch {
  CP_ARCH_DLA34 = 0,        /* 'dla_34'   : DLA-34 + DCNv2            (model.py:19) */
  CP_ARCH_DLAV1_34 = 1,     /* 'dlav1_34' : + convGRU + GroupNorm heads (model.py:20) */
  /* 'res_N' (model.py:17, networks/msra_resnet.py; opts.py:77-79 lists res_101 as tested): 7x7/2 stem + 3x3/2 max-pool
   * (:116-120), layer1..4 of BasicBlocks (18, 34) or Bottlenecks (50, 101, 152) per resnet_spec (:300-304), three
   * ConvTranspose2d 4x4/2/1 + BN + ReLU to 256 channels (:208-233), heads 3x3 -> ReLU -> 1x1 (:157-174).  Tracking
   * configs add the pre_img / pre_hm / pre_hm_hp stems, each summed after its own max-pool (:126-147, 242-247).
   * tracking_task_gru is CP_ERR_INVALID (no convGRU); head_conv as for DLA (the reference's default for res is 64,
   * opts.py:344-345). */
  CP_ARCH_RES_18 = 2,
  CP_ARCH_RES_34 = 3,
  CP_ARCH_RES_50 = 4,
  CP_ARCH_RES_101 = 5,
  CP_ARCH_RES_152 = 6
};

enum cp_precision {
  CP_PREC_FP32 = 0,         /* fp32 operands and accumulation on CUDA cores (parity mode)      */
  CP_PREC_TF32X3 = 1,       /* wgmma tf32, 3-term split + promoted accumulation: fp32-equivalent
                             * tensor-core mode, meets the same parity bar as CP_PREC_FP32; the Python host's
                             * default                                                                      */
  CP_PREC_BF16 = 2,         /* wgmma bf16 operands, fp32 accumulation (fast mode)  */
  CP_PREC_TF32 = 3          /* wgmma tf32 single pass -- the math PyTorch's cuDNN convolutions use by
                             * default (allow_tf32); stride-2 convs run the 3-term split gather kernel     */
};

#define CP_MAX_HEADS 16
#define CP_POSE_RECORD 192  /* floats per detection slot in `poses`  */
#define CP_DETS_RECORD 128  /* floats per candidate slot in `dets`   */
#define CP_META_DOUBLES 16  /* doubles per image in `meta`           */
#define CP_MAX_K 128
#define CP_MAX_CLASSES 80   /* hm channels the decode stage merges (decode.py:52-68 _topk) */
#define CP_MAX_MODELS 16    /* checkpoints one multi-model plan holds (cp_plan_create_multi) */

typedef struct cp_plan cp_plan;

typedef struct cp_config {
  int32_t arch;                 /* cp_arch                                                */
  int32_t tracking;             /* 1: pre_img / pre_hm / pre_hm_hp stems (pose_dla_dcn.py:253-271) */
  int32_t tracking_task_gru;    /* dlav1 only: 4 GRU steps + tracking routing (:473-477,545-555)   */
  int32_t max_batch;
  int32_t height, width;        /* network input, multiples of 32                         */
  int32_t precision;            /* cp_precision                                           */
  int32_t device;               /* CUDA ordinal                                           */
  int32_t head_conv;            /* 256                                                    */
  int32_t num_heads;
  const char* head_names[CP_MAX_HEADS];    /* in opt.heads order (opts.py:394-426)        */
  int32_t head_channels[CP_MAX_HEADS];
} cp_config;

/* Create a plan: builds the static layer schedule and allocates the
 * activation arena + packed-weight storage on cfg->device.  Synchronous. */
int cp_plan_create(const cp_config* cfg, cp_plan** out);
int cp_plan_destroy(cp_plan* plan);

/* ---- multi-model plans: several checkpoints of one architecture (one per object category) over the same frames ----
 * cp_plan_create_multi builds one schedule for `num_models` models (1..CP_MAX_MODELS; cp_plan_create is this call with
 * 1).  Every op is ONE launch for all models: model m's weights are the m-th copy of the weight storage, and image b of
 * model m is image m * batch + b of each launch, where batch is the number of frames of the call.  So the activations
 * of a call at `batch` frames are [num_models * batch, ...] and model m's are a contiguous slice of them.
 *   - images (and pre_img ...) and meta rows are [batch, ...]: every model reads the same frames, nothing is copied.
 *   - head_out[i] of cp_forward / cp_plan_profile / cp_plan_run_ops is [num_models, batch, C, H/4, W/4].
 *   - tracking configs take num_models == 1 only here; several tracking models go through cp_plan_create_multi_track.
 * cp_plan_load_weights_model fills model `model` (cp_plan_load_weights fills model 0); running before every model is
 * loaded returns CP_ERR_NOT_LOADED. */
int cp_plan_create_multi(const cp_config* cfg, int32_t num_models, cp_plan** out);
/* A multi-model plan of `num_models` TRACKING models (cfg->tracking must be 1, else CP_ERR_INVALID; 1..CP_MAX_MODELS
 * models, both archs).  Every category tracks its own objects, so its previous-frame heat maps are its own:
 *   - images and pre_img are [batch, 3, H, W], shared by every model, as in cp_plan_create_multi;
 *   - pre_hm is [num_models, batch, 1, H, W] and pre_hm_hp [num_models, batch, 8, H, W]: model m reads slice m.
 * This layout holds for cp_forward, cp_plan_profile, cp_plan_run_ops and cp_infer_multi_track; outputs are
 * [num_models, batch, ...] as in cp_plan_create_multi, and the schedule has the launches of a one-model tracking plan. */
int cp_plan_create_multi_track(const cp_config* cfg, int32_t num_models, cp_plan** out);

/* ---- plan flags: cp_plan_create_ex / cp_plan_memory ----------------------------------------------------------------
 * CP_PLAN_REUSE_ACTIVATIONS: activations whose lifetimes do not overlap share arena memory.  An allocation is live from
 *   the op that first writes it to the op that last reads it; the head buffers cp_infer decodes stay live to the end of
 *   the call.  The plan computes bit for bit what a plan without the flag computes, in a fraction of the arena (README).
 *   Consequences for the diagnostics: the cp_act_desc offsets of different ops may coincide, an allocation no op touches
 *   (the merged heads' hidden tile when the 1x1s are fused into its epilogue) reports off = -1, and cp_plan_run_ops is
 *   valid for op ranges whose inputs are still live, for example when stepping from op 0 in order.
 * CP_PLAN_MULTI_TRACK: the per-model pre_hm / pre_hm_hp layout of cp_plan_create_multi_track (needs cfg->tracking = 1;
 *   a tracking config of several models needs it).
 * CP_PLAN_BATCH_INVARIANT: every output element is the same bits whatever the batch of the call, the frame's row in it,
 *   the number of models in the plan and the device's SM count.  By default the tf32x3 conv_tma launches (not fused) and
 *   the dcn_tma launches split their K loop over a number of CTAs chosen from the launch's tiles and the SM count, so a
 *   frame's sums depend on its batch.  With the flag every such launch cuts K into G segments fixed by the layer's shape
 *   (G: the largest divisor of the launch's channel slabs with G x the (m, n) tiles of one image of one model <= 132; 1
 *   wherever the default never splits), sums each segment as a split CTA of it does and adds the segments in order,
 *   ((0 + seg 0) + seg 1) + ..., before the epilogue.  The segments run on separate CTAs when their partial sums fit the
 *   plan's split-K workspace and back to back in one CTA per tile otherwise; the choice never changes a bit
 *   (cp_plan_op_ksegments reports it).  G is what the default picks at batch 1 on a 132-SM H100, so there the flag gives
 *   the bits of a batch-1 call of a default plan.  It adds no memory; fp32 and bf16 plans accept it and are unchanged. */
#define CP_PLAN_REUSE_ACTIVATIONS 1u
#define CP_PLAN_MULTI_TRACK 2u
#define CP_PLAN_BATCH_INVARIANT 32u
/* cp_plan_create_multi (flags 0) or cp_plan_create_multi_track (CP_PLAN_MULTI_TRACK) with flags; unknown flag bits return
 * CP_ERR_INVALID.  The three creators above are this call with those flags. */
int cp_plan_create_ex(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_plan** out);
/* Device memory a plan of these arguments owns, in bytes, computed on the host without a device (to size a deployment
 * before creating the plan).  cp_plan_bytes of the created plan is activation_bytes + weight_bytes.  The decode workspace
 * cp_infer sizes on its first call is not included (cp_decode_workspace_bytes). */
typedef struct cp_memory_info {
  int64_t activation_bytes;  /* the activation arena                                                               */
  int64_t weight_bytes;      /* packed fp32 weights of every model                                                 */
  int64_t tile_bytes;        /* pre-swizzled tensor-core weight tiles of every model                               */
  int64_t workspace_bytes;   /* GroupNorm statistics and split-K partial sums                                      */
} cp_memory_info;
int cp_plan_memory(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_memory_info* out);
/* The arena allocations of such a plan (host only, like cp_plan_memory): allocation i takes `floats` floats at `off`
 * floats into the arena and is live over ops [first, last] of the schedule (last = cp_plan_num_ops: to the end of the
 * call; first = -1 when no op touches it); floats = 0 and off = -1 when it gets no memory.  Fills the first max_allocs
 * records at most; *n_allocs receives the number of allocations. */
typedef struct cp_act_alloc {
  int64_t floats;
  int64_t off;
  int32_t first, last;
} cp_act_alloc;
int cp_plan_allocations(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_act_alloc* out, int32_t max_allocs,
                        int32_t* n_allocs);

int cp_plan_load_weights_model(cp_plan* plan, int32_t model, const char* const* names, const void* const* dev_ptrs,
                               const int64_t* numel, int32_t n, void* stream);
int32_t cp_plan_num_models(const cp_plan* plan);

/* Ingest a reference state_dict (Appendix A of SURVEY.md).  names[i] is the
 * reference key (an optional leading "module." is ignored, model.py:43-47),
 * dev_ptrs[i] a DEVICE pointer to contiguous fp32 data in the reference's
 * layout (OIHW conv weights, [C] vectors), numel[i] its element count.  The
 * pointers are only borrowed for the duration of the call: BatchNorm is
 * folded, weights are repacked (K-major, padded) into plan-owned storage.
 * Unknown keys (e.g. base.fc.*, num_batches_tracked) are ignored; a key the
 * plan needs but does not get returns CP_ERR_MISSING_KEY.  Enqueued on
 * `stream`; the borrowed tensors must stay alive until that work completes. */
int cp_plan_load_weights(cp_plan* plan, const char* const* names, const void* const* dev_ptrs,
                         const int64_t* numel, int32_t n, void* stream);

/* Network forward.  images: device fp32 NCHW [batch,3,H,W]; pre_img [batch,3,H,W],
 * pre_hm [batch,1,H,W], pre_hm_hp [batch,8,H,W] or NULL (tracking plans only).
 * head_out[i]: device fp32 NCHW [batch, head_channels[i], H/4, W/4] receiving the
 * LOGITS of head i (the reference applies sigmoid later, object_pose.py:136-138). */
int cp_forward(cp_plan* plan, int32_t batch, const float* images, const float* pre_img,
               const float* pre_hm, const float* pre_hm_hp, float* const* head_out, void* stream);

/* Per-op timing of one forward (the reference only has wall-clock stamps around whole stages,
 * base_detector.py:466-498): CUDA events are recorded on `stream` between the ops of the
 * schedule; the call synchronises on the last event.  `flops` / `bytes` are the ALGORITHMIC
 * work of the op (2*MAC; fp32 tensors touched once), used for the roofline in bench.py.
 * kind = op_type*10 + igemm_mode  (0: NCHW stem conv, 1: NHWC conv, 2: deformable conv,
 * 3: dense ConvTranspose2d 4x4 stride 2 pad 1 (ResNet up-sampling), 10: 2x2 max-pool, 11: 3x3 stride-2 pad-1
 * max-pool [+ residual] (ResNet stems), 20: up-sample+add, 30: GroupNorm+ReLU, 40: GRU gate). */
typedef struct cp_op_stat {
  char name[96];
  int32_t kind;
  float ms;
  double flops;
  double bytes;
} cp_op_stat;
int cp_plan_num_ops(const cp_plan* plan);
int cp_plan_profile(cp_plan* plan, int32_t batch, const float* images, const float* pre_img,
                    const float* pre_hm, const float* pre_hm_hp, float* const* head_out, void* stream,
                    cp_op_stat* stats, int32_t max_stats, int32_t* n_stats);

/* ---- diagnostics: inspect and step the schedule (per-layer parity tests) ----------------------------------------
 * cp_plan_op_desc describes op i of the schedule as the plan stores it; cp_plan_arena gives the activation arena every
 * cp_act_desc points into; cp_plan_run_ops runs ops [first, last) exactly as cp_forward does (PDL off) and reports for
 * each one what its launcher decided.  Together they let a test snapshot an op's inputs, run the op alone and compare
 * its output with an independent evaluation.  Not needed for inference. */
enum cp_op_family {
  CP_FAM_NONE = 0,          /* not launched (fused into its parent's epilogue)              */
  CP_FAM_IGEMM_FP32 = 1,    /* generic fp32 CUDA-core implicit GEMM (igemm_fp32.cu)          */
  CP_FAM_STEM = 2,          /* 7x7 NCHW stem (stem_conv.cu)                                   */
  CP_FAM_CONV3_C16 = 3,     /* direct 3x3 16 -> 16 (stem_conv.cu)                             */
  CP_FAM_IGEMM_UMMA = 4,    /* wgmma gather implicit GEMM (igemm_umma.cu)                     */
  CP_FAM_CONV_TMA = 5,      /* TMA-fed wgmma convolution (conv_tma.cu)                        */
  CP_FAM_DCN_TMA = 6,       /* TMA-staged wgmma deformable convolution (dcn_tma.cu)           */
  CP_FAM_MAXPOOL = 7, CP_FAM_UPADD = 8, CP_FAM_GN_RELU = 9, CP_FAM_GRU = 10
};
typedef struct cp_act_desc {
  int64_t off;              /* floats into the arena: element (n, y, x, c) is at off + ((n*H + y)*W + x)*stride + c,
                             * n < max_batch; -1 when the slot is unused                                            */
  int32_t ext;              /* >= 0: external NCHW input instead (0 images, 1 pre_img, 2 pre_hm, 3 pre_hm_hp)       */
  int32_t C, H, W, stride;
} cp_act_desc;
typedef struct cp_op_desc {
  char name[96];
  int32_t kind;             /* as cp_op_stat.kind                                                                   */
  int32_t family;           /* cp_op_family chosen at plan time (fp32 CUDA-core ops: the kernel at max_batch)      */
  int32_t x3;               /* tensor-core families: 1 = three-term tf32 split, 0 = single pass / bf16              */
  int32_t nsrc;             /* conv: sources, concatenated along channels in this order                             */
  cp_act_desc src[4];       /* conv / maxpool / up-sample input (src[0])                                            */
  cp_act_desc out;          /* output (GroupNorm: the channel slice it normalises in place)                         */
  int32_t out_head;         /* >= 0: the conv writes head out_head as NCHW instead of `out`                        */
  int32_t kh, stride, pad, Cin, Cout, CoutPad, Kpad;
  const float* w;           /* device fp32 [Kpad][w_ld], row k = (ky*kh + kx)*Cin + ci, BN folded.  kind 3: four phase
                             * blocks [4][Kpad][w_ld], Kpad = 4 Cin; phase py*2+px, row (2a+b)*Cin + ci holds
                             * weight[ci][co][ky][kx] with ky = 1+2a (py 0) or 2a (py 1) and kx likewise; it feeds output
                             * (2y+py, 2x+px) from input (y+dy, x+dx), dy = -a (py 0) or 1-a (py 1)                   */
  int32_t w_ld;
  const float* bias;        /* device fp32 [Cout]                                                                  */
  int32_t relu, has_res, res_after_relu;   /* out = relu(acc + bias [+ res]) or relu(acc + bias) + res           */
  cp_act_desc res;
  cp_act_desc om;           /* deformable conv: raw offset / mask logits (dy, dx of tap k at 2k, 2k+1; mask 18+k) */
  const float* up_w;        /* up-sample: device fp32 [2f][2f][C] depthwise ConvTranspose weights                 */
  int32_t f, has_skip;
  cp_act_desc skip;
  const float* gamma;       /* GroupNorm+ReLU                                                                      */
  const float* beta;
  int32_t groups;
  cp_act_desc gx, gh, gprev; /* GRU gates: x-side and h-side pre-activations [r | z | n], previous state            */
  int32_t first_step;
  int32_t fuse_heads;       /* 1: the per-head 1x1 convs `children` run in this op's epilogue                       */
  int32_t fused_away;       /* 1: this 1x1 runs inside op `parent`                                                 */
  int32_t parent;
  int32_t n_children;
  int32_t children[CP_MAX_HEADS];
} cp_op_desc;
typedef struct cp_op_launch {
  int32_t family;           /* cp_op_family of the kernel that ran (CP_FAM_NONE: fused away)                        */
  int32_t BN;               /* N tile (tensor-core families; 0 otherwise)                                          */
  int32_t ksplit;           /* split-K factor (1 = off)                                                            */
  int32_t grid;             /* CTAs of the main kernel (tensor-core families; 0 otherwise)                         */
} cp_op_launch;
/* How a launch summed its K segments (cp_plan_op_ksegments). */
enum cp_kpath {
  CP_KPATH_NONE = 0,        /* not a conv_tma / dcn_tma launch, or not launched yet                                   */
  CP_KPATH_ONE = 1,         /* one segment: each (m, n) tile on one CTA over the whole K                               */
  CP_KPATH_SPLIT = 2,       /* split-K: one CTA per (tile, segment), partial sums added by the finish kernel           */
  CP_KPATH_FOLD = 3         /* CP_PLAN_BATCH_INVARIANT: one CTA per tile runs the segments back to back                */
};
/* Op i's K segments: *segments receives the G of a CP_PLAN_BATCH_INVARIANT plan (1 where it never splits) and 0 for
 * every op of a default plan, whose launches choose; *last_segments and *last_path (either may be NULL) what the op's
 * latest launch (cp_forward, cp_infer*, cp_plan_run_ops ...) did: its split-K factor and a cp_kpath. */
int cp_plan_op_ksegments(const cp_plan* plan, int32_t i, int32_t* segments, int32_t* last_segments, int32_t* last_path);
/* The segments of every op of a plan of these arguments, as cp_plan_op_ksegments' *segments, computed on the host
 * without a device (like cp_plan_memory).  Fills the first max_ops entries at most; *n_ops receives cp_plan_num_ops. */
int cp_plan_ksegments(const cp_config* cfg, int32_t num_models, uint32_t flags, int32_t* segments, int32_t max_ops,
                      int32_t* n_ops);
int cp_plan_op_desc(const cp_plan* plan, int32_t i, cp_op_desc* out);
/* op i as model `model` of a multi-model plan sees it: its weight, bias, up-sample and GroupNorm pointers, and
 * activation offsets moved to its images for a call at the plan's max_batch (model m's images start at image
 * m * max_batch; at a smaller batch they start at m * batch).  cp_plan_op_desc is this call with model 0. */
int cp_plan_op_desc_model(const cp_plan* plan, int32_t model, int32_t i, cp_op_desc* out);
int cp_plan_arena(const cp_plan* plan, float** act, int64_t* floats);
/* `info` (may be NULL) receives last - first records. */
int cp_plan_run_ops(cp_plan* plan, int32_t batch, int32_t first, int32_t last, const float* images, const float* pre_img,
                    const float* pre_hm, const float* pre_hm_hp, float* const* head_out, void* stream,
                    cp_op_launch* info);

/* Arena / weight bytes owned by the plan (for logging): activation_bytes + weight_bytes of cp_plan_memory. */
int64_t cp_plan_bytes(const cp_plan* plan);
/* Number of kernel launches one cp_forward enqueues (for bench gpu_launches). */
int32_t cp_plan_forward_launches(const cp_plan* plan);

/* ---- decode + grouping + post-process + soft-NMS + PnP --------------------- */
typedef struct cp_heads {
  /* device fp32 NCHW [batch, C, out_h, out_w]; NULL when the head is absent */
  const float* hm;                /* [B,num_classes,..] logits (or probabilities if !apply_sigmoid) */
  const float* wh;                /* [B,2,..]   */
  const float* hps;               /* [B,2J,..]  */
  const float* reg;               /* [B,2,..]   or NULL */
  const float* hm_hp;             /* [B,J,..]   */
  const float* hp_offset;         /* [B,2,..]   or NULL */
  const float* scale;             /* [B,3,..]   or NULL */
  const float* hps_uncertainty;   /* [B,2J,..]  or NULL */
  const float* scale_uncertainty; /* [B,3,..]   or NULL */
  const float* tracking;          /* [B,2,..]   or NULL */
  const float* tracking_hp;       /* [B,2J,..]  or NULL */
} cp_heads;

typedef struct cp_decode_params {
  int32_t batch, out_h, out_w;
  int32_t num_classes;     /* opt.num_classes = hm channels, 1..CP_MAX_CLASSES (Objectron models: 1, opts.py:434): per-class
                            * top-K, then the K best of the num_classes x K candidates (decode.py:52-68)               */
  int32_t num_joints;      /* 8                                                            */
  int32_t K;               /* opt.K = 100, <= CP_MAX_K                                     */
  int32_t rep_mode;        /* opt.rep_mode: 0,1,3,4 (2 = random GMM sampling, unsupported) */
  int32_t use_moments;     /* opt.tracking_task || opt.refined_Kalman (decode.py:222)      */
  int32_t nms;             /* opt.nms (demo.py:114 sets True)                              */
  int32_t visible_thresh;  /* cuboid_pnp_shell.py:59-66: 6 book/chair/cereal_box, 3 camera/bottle/cup, 0 bike/laptop/shoe */
  int32_t opencv_return;   /* opt.show_axes: return the OpenCV pose instead of OpenGL      */
  int32_t apply_sigmoid;   /* 0: hm / hm_hp are probabilities; 1: both are logits; 2: only hm is a logit
                            * (opt.mse_loss: hm_hp is decoded raw, object_pose.py:136-138)  */
  int32_t use_pnp;         /* opt.use_pnp                                                  */
  float vis_thresh;        /* opt.vis_thresh (0.3)                                         */
  float balance;           /* opt.balance_coefficient[opt.c] (2)                           */
  int32_t modern_bool_semantics; /* 0 (default): the pinned torch==1.1.0 meaning of models/decode.py:183-188, where the
                            * seven comparison results are ADDED as integers and `mask_2 == 7` = "all seven gates hold".
                            * 1: what the unmodified reference computes on torch >= 1.2 (bool + bool is a logical OR, so
                            * `== 7` is never true): the heat-map keypoint representation is never used, kps_heatmap_* stay
                            * at the -10000 sentinel and the PnP sees the 8 displacement points only.                 */
  float test_scale;        /* opt.test_scales[0] (1; 0 is read as 1): the scale the frame was resized by in pre_process; != 1 divides bbox,
                            * kps, kps_displacement_mean / _std, kps_heatmap_mean, tracking and tracking_hp by it in
                            * float32 before soft-NMS and the PnP (object_pose.py:171-177)                              */
  int32_t num_scales;      /* len(opt.test_scales): > 1 forces the soft-NMS (object_pose.py:193); merge_outputs keeps the
                            * detections of test_scales[0] only (object_pose.py:188 reads detections[0])               */
} cp_decode_params;

/* meta: device fp64 [batch, CP_META_DOUBLES] per image:
 *   [0] c_x  [1] c_y  [2] s (src width of the affine, base_detector.py:114)
 *   [3] image width  [4] image height  [5..13] camera matrix row-major  [14,15] unused
 * dets:  device fp32 [batch, K, CP_DETS_RECORD] or NULL -- the 13 arrays of
 *        decode.py:348-361 in output-map pixels (layout: cp_dets_field).
 * poses: device fp32 [batch, K, CP_POSE_RECORD] -- slots [0, n_valid[b]) hold the
 *        reference's `results` (after score filter + soft-NMS) in order, image pixels,
 *        with the PnP output of each (layout: cp_pose_field).
 * n_valid: device int32 [batch].
 * workspace: device scratch of at least cp_decode_workspace_bytes(prm) bytes. */
size_t cp_decode_workspace_bytes(const cp_decode_params* prm);
int cp_decode_pnp(const cp_decode_params* prm, const cp_heads* heads, const double* meta,
                  float* dets, float* poses, int32_t* n_valid,
                  void* workspace, size_t workspace_bytes, void* stream);

/* forward + decode in one call; head maps stay in plan-owned buffers.
 * `heads_out` may be NULL, or an array of num_heads device pointers that
 * additionally receive the head logits (NCHW). */
int cp_infer(cp_plan* plan, int32_t batch, const float* images, const float* pre_img,
             const float* pre_hm, const float* pre_hm_hp, const cp_decode_params* prm,
             const double* meta, float* const* heads_out, float* dets, float* poses,
             int32_t* n_valid, void* stream);

/* cp_infer for every model of a multi-model plan: one forward and one decode for all of them.  prms[num_models]: the
 * decode parameters of each model; they may differ in visible_thresh and balance only (else CP_ERR_INVALID).  meta is
 * [batch] (the frames); heads_out[i] (optional) is [num_models, batch, C, H/4, W/4]; dets (optional)
 * [num_models, batch, K, CP_DETS_RECORD]; poses [num_models, batch, K, CP_POSE_RECORD]; n_valid [num_models, batch]. */
int cp_infer_multi(cp_plan* plan, int32_t batch, const float* images, const cp_decode_params* prms, const double* meta,
                   float* const* heads_out, float* dets, float* poses, int32_t* n_valid, void* stream);
/* cp_infer_multi for a plan of cp_plan_create_multi_track, with its four tracking inputs (images / pre_img [batch, ...],
 * pre_hm / pre_hm_hp [num_models, batch, ...]).  prms, meta [batch] and the outputs as in cp_infer_multi: the pose records
 * are [num_models, batch, K, CP_POSE_RECORD], which is the stream order of a cp_tracker_create_multi tracker of
 * num_models categories x batch streams.  cp_infer_multi refuses tracking plans. */
int cp_infer_multi_track(cp_plan* plan, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
                         const float* pre_hm_hp, const cp_decode_params* prms, const double* meta, float* const* heads_out,
                         float* dets, float* poses, int32_t* n_valid, void* stream);

/* Offsets (in floats) inside one CP_POSE_RECORD slot. */
enum cp_pose_field {
  CP_P_SCORE = 0, CP_P_CLS = 1, CP_P_STATUS = 2, CP_P_NPTS = 3,
  CP_P_BBOX = 4,            /* 4  */
  CP_P_CT = 8,              /* 2  */
  CP_P_KPS = 10,            /* 16 */
  CP_P_KPS_DISP_MEAN = 26,  /* 16 */
  CP_P_KPS_HM_MEAN = 42,    /* 16 */
  CP_P_KPS_HM_STD = 58,     /* 16 */
  CP_P_KPS_HM_HEIGHT = 74,  /* 8  */
  CP_P_KPS_DISP_STD = 82,   /* 16 */
  CP_P_OBJ_SCALE = 98,      /* 3  */
  CP_P_OBJ_SCALE_UNC = 101, /* 3  */
  CP_P_TRACKING = 104,      /* 2  */
  CP_P_TRACKING_HP = 106,   /* 16 */
  CP_P_LOCATION = 122,      /* 3  */
  CP_P_QUAT = 125,          /* 4 xyzw */
  CP_P_REPROJ = 129,        /* 1  */
  CP_P_PROJ_CUBOID = 130,   /* 16 */
  CP_P_KPS_3D_CAM = 146,    /* 27 */
  CP_P_KPS_PNP = 173,       /* 18 */
  CP_P_SRC_INDEX = 191      /* index k of the candidate in the top-K list */
};

/* PnP status stored in CP_P_STATUS (mirrors the reference's None paths). */
enum cp_pnp_status {
  CP_PNP_NOT_RUN = 0,
  CP_PNP_OK = 1,          /* pnp_shell returned a tuple -> goes into `boxes`                    */
  CP_PNP_INVISIBLE = 2,   /* pose stored in the result, visibility gate returned None (:59-79)  */
  CP_PNP_BEHIND = 3,      /* z < 0 (cuboid_pnp_solver.py:208-220)                               */
  CP_PNP_FEW_POINTS = 4,  /* < 4 valid points (cuboid_pnp_solver.py:157-160); 4-5 points are solved by EPnP   */
  CP_PNP_SOLVER_FAIL = 5
};

/* Offsets inside one CP_DETS_RECORD slot (output-map pixel units). */
enum cp_dets_field {
  CP_D_BBOX = 0, CP_D_SCORE = 4, CP_D_CLS = 5,
  CP_D_KPS = 6,             /* 16 */
  CP_D_OBJ_SCALE = 22,      /* 3  */
  CP_D_OBJ_SCALE_UNC = 25,  /* 3  */
  CP_D_TRACKING = 28,       /* 2  */
  CP_D_TRACKING_HP = 30,    /* 16 */
  CP_D_KPS_DISP_MEAN = 46,  /* 16 */
  CP_D_KPS_DISP_STD = 62,   /* 16 */
  CP_D_KPS_HM_MEAN = 78,    /* 16 */
  CP_D_KPS_HM_STD = 94,     /* 16 */
  CP_D_KPS_HM_HEIGHT = 110, /* 8  */
  CP_D_IND = 118            /* flat index of the centre cell */
};

/* ---- CenterPoseTrack state on the device (SURVEY.md rows a-T / f-2) ----------- */
/* Replaces utils/tracker.py:15-302 (Tracker: association, 32-state Kalman filter per object, scale pool, second PnP
 * with the filtered keypoints), the gaussian_fusion closure of detectors/base_detector.py:502-544 and the rendering of
 * the previous-frame heat maps, base_detector.py:150-388 (_get_additional_inputs, default options: use_pnp,
 * render_hm_mode 1, render_hmhp_mode 0-3).  One tracker holds `streams` independent videos (the batch dimension);
 * state lives in device memory, every call is enqueued on `stream`, calls on one tracker must be issued in frame order
 * on one stream.  Association is greedy (tracker.py:305-314) or, with `hungarian`, the minimum-cost assignment that
 * scipy.optimize.linear_sum_assignment returns (ties included).  Tracks can be seeded from ground truth
 * (Tracker.init_track with meta['pre_dets'], cp_tracker_seed) and the previous-frame heat maps drawn from that ground
 * truth (opt.gt_pre_hm_hmhp / gt_pre_hm_hmhp_first) or left empty (opt.empty_pre_hm), see cp_tracker_render_ex.
 *
 * Streams are stepped independently: each stream keeps its own current buffer of the double-buffered track state, so a
 * stream that a step does not list is left bit-for-bit as it was (tracks, ids, ages, filters, scale pool) and resumes
 * from there.  The _ex variants (cp_tracker_step_ex, cp_tracker_render_ex2, cp_tracker_seed_ex) take a stream map:
 * `stream_ids` is a HOST int32 [batch], owned by the caller and read before the call returns; batch row i reads and
 * advances tracker stream stream_ids[i].  Every id must lie in 0..streams-1 and appear once, otherwise the call returns
 * CP_ERR_INVALID before any work is enqueued.  stream_ids == NULL is the identity (row i = stream i), which is what the
 * entry points without a map do. */
#define CP_TRACK_RECORD 320
typedef struct cp_tracker cp_tracker;
typedef struct cp_tracker_config {
  int32_t streams;            /* independent videos = max batch of cp_tracker_step                         */
  int32_t max_tracks;         /* per stream, <= CP_MAX_K                                                    */
  int32_t kalman;             /* opt.kalman                                                                 */
  int32_t scale_pool;         /* opt.scale_pool                                                             */
  int32_t use_pnp;            /* opt.use_pnp                                                                */
  int32_t hps_uncertainty;    /* opt.hps_uncertainty                                                        */
  int32_t max_age;            /* opt.max_age (5)                                                            */
  int32_t visible_thresh;     /* as in cp_decode_params                                                     */
  int32_t opencv_return;      /* opt.show_axes                                                              */
  int32_t render_hm_mode;     /* opt.render_hm_mode (1: centre heat = score)                                */
  int32_t render_hmhp_mode;   /* opt.render_hmhp_mode (2: PnP keypoints, heat = filter confidence)          */
  int32_t device;
  float new_thresh;           /* opt.new_thresh                                                             */
  float pre_thresh;           /* opt.pre_thresh                                                             */
  float R;                    /* opt.R (20)                                                                 */
  float conf_lo, conf_hi;     /* opt.conf_border[opt.c] (3, 9)                                              */
  int32_t hungarian;          /* opt.hungarian: optimal instead of greedy association (tracker.py:154-177)  */
} cp_tracker_config;

int cp_tracker_create(const cp_tracker_config* cfg, cp_tracker** out);
/* One tracker for `models` object categories (1..CP_MAX_MODELS) of cfgs[0].streams streams each: tracker stream m * S + s
 * (S = cfgs[0].streams) is stream s of category m and uses cfgs[m].visible_thresh, conf_lo and conf_hi; the configs may
 * differ in those three fields only (else CP_ERR_INVALID, before anything is allocated).  Every other call sees a tracker
 * of models * S streams: cp_tracker_step advances all of them in one launch (two with hungarian), the stream maps of the
 * _ex calls address them as m * S + s, and the meta rows stay one per batch row (a frame's row repeated per category).
 * cp_tracker_create is this call with models = 1. */
int cp_tracker_create_multi(const cp_tracker_config* cfgs, int32_t models, cp_tracker** out);
int cp_tracker_destroy(cp_tracker* trk);
/* Tracker.reset(): forget every track of stream `index` (or of all streams when index < 0). */
int cp_tracker_reset(cp_tracker* trk, int32_t index, void* stream);
/* Tracker.step(results, boxes) for `batch` streams (stream b <- poses[b]).  poses / n_valid / meta as produced by
 * cp_decode_pnp / cp_infer (K slots per image).  tracks_out: device fp32 [batch, max_tracks, CP_TRACK_RECORD], slots
 * [0, n_tracks[b]) = the reference's self.tracker.tracks in order (layout: cp_track_field); n_tracks: device int32. */
int cp_tracker_step(cp_tracker* trk, int32_t batch, const float* poses, const int32_t* n_valid, int32_t K,
                    const double* meta, float* tracks_out, int32_t* n_tracks, void* stream);
/* cp_tracker_step with a stream map: batch row i (poses[i], meta[i], tracks_out[i], n_tracks[i]) is tracker stream
 * stream_ids[i].  Only the listed streams are stepped. */
int cp_tracker_step_ex(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, const float* poses,
                       const int32_t* n_valid, int32_t K, const double* meta, float* tracks_out, int32_t* n_tracks,
                       void* stream);
/* _get_additional_inputs(): render the tracks of every stream into pre_hm [batch,1,inp_h,inp_w] and pre_hm_hp
 * [batch,8,inp_h,inp_w] (device fp32, overwritten).  trans_input: device fp64 [batch,6] = the row-major 2x3 affine
 * meta['trans_input'] (original image -> network input). */
int cp_tracker_render(cp_tracker* trk, int32_t batch, const double* meta, const double* trans_input, int32_t inp_h,
                      int32_t inp_w, float* pre_hm, float* pre_hm_hp, void* stream);
/* Per-stream render modes of cp_tracker_render_ex. */
enum cp_render_mode {
  CP_RENDER_TRACKS = 0,  /* the tracks (what cp_tracker_render draws)                                              */
  CP_RENDER_GT = 1,      /* the ground-truth branch of _get_additional_inputs (base_detector.py:166-209): every track,
                          * no pre_thresh test, centre heat 1, the 8 points of kps_gt[1:] with heat 1 and no
                          * visibility or in-input gate.  Tracks that were not seeded draw their centre only.          */
  CP_RENDER_EMPTY = 2    /* all zeros (opt.empty_pre_hm)                                                            */
};
/* cp_tracker_render with a mode per stream: `modes` is a HOST int32 [batch] of cp_render_mode values, or NULL for all
 * CP_RENDER_TRACKS (then identical to cp_tracker_render).  An unknown mode returns CP_ERR_INVALID. */
int cp_tracker_render_ex(cp_tracker* trk, int32_t batch, const double* meta, const double* trans_input, int32_t inp_h,
                         int32_t inp_w, const int32_t* modes, float* pre_hm, float* pre_hm_hp, void* stream);
/* cp_tracker_render_ex with a stream map: image i (meta[i], trans_input[i], modes[i], pre_hm[i], pre_hm_hp[i]) draws the
 * tracks of tracker stream stream_ids[i]. */
int cp_tracker_render_ex2(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, const double* meta,
                          const double* trans_input, int32_t inp_h, int32_t inp_w, const int32_t* modes, float* pre_hm,
                          float* pre_hm_hp, void* stream);

/* Graph-safe forms: every per-step input is in device memory and read when the kernels run, nothing is allocated and
 * no host memory is read after the call returns, so a CUDA graph that captured the call replays it as issued.  Bad
 * arguments return CP_ERR_INVALID before any work is enqueued; a failure inside a capture (a cudaErrorStreamCapture*
 * status) returns CP_ERR_CUDA with its text in cp_last_error.  cp_tracker_step (greedy or Hungarian) is graph-safe as
 * it is.
 *
 * cp_tracker_reset_dev: flags is a DEVICE int32 [batch] (batch in 1..streams); every stream b with flags[b] != 0 is
 * reset exactly as cp_tracker_reset(trk, b) does (tracks, ids, ages, filters and scale pool forgotten). */
int cp_tracker_reset_dev(cp_tracker* trk, int32_t batch, const int32_t* flags, void* stream);
/* cp_tracker_render_ex without a stream map and with `modes` a DEVICE int32 [batch] of cp_render_mode values (or NULL
 * for all CP_RENDER_TRACKS); the kernel reads them, so they are not checked: a value other than CP_RENDER_GT or
 * CP_RENDER_EMPTY draws the tracks. */
int cp_tracker_render_dev(cp_tracker* trk, int32_t batch, const double* meta, const double* trans_input, int32_t inp_h,
                          int32_t inp_w, const int32_t* modes, float* pre_hm, float* pre_hm_hp, void* stream);
/* cp_tracker_render_dev with a stream map: image i draws the tracks of tracker stream stream_ids[i].  stream_ids is a
 * DEVICE int32 [batch] (or NULL: the identity) that the kernel reads WITHOUT checking: the caller guarantees every id is
 * in 0..streams-1 and none appears twice (cp_tracker_render_ex2 checks a host map; this one cannot). */
int cp_tracker_render_dev2(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, const double* meta,
                           const double* trans_input, int32_t inp_h, int32_t inp_w, const int32_t* modes, float* pre_hm,
                           float* pre_hm_hp, void* stream);
/* cp_tracker_step_ex with the stream map in device memory: row i (poses[i], n_valid[i], meta[i], tracks_out[i],
 * n_tracks[i]) steps tracker stream stream_ids[i]; streams the map does not list keep their state.  stream_ids is a
 * DEVICE int32 [batch] (or NULL: the identity) that the kernels read WITHOUT checking: the caller guarantees every id is
 * in 0..streams-1 and none appears twice.  Greedy or Hungarian association as configured; the kernels are those of
 * cp_tracker_step_ex. */
int cp_tracker_step_dev(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, const float* poses,
                        const int32_t* n_valid, int32_t K, const double* meta, float* tracks_out, int32_t* n_tracks,
                        void* stream);

/* Offsets (in floats) inside one CP_SEED_RECORD: one dict of meta['pre_dets'] (eval_video_official.py:422-450). */
#define CP_SEED_RECORD 264
enum cp_seed_field {
  /* [0, CP_POSE_RECORD): the cp_pose_field layout, holding the dict keys of the same names (image pixels).  CP_P_STATUS
   * is CP_PNP_OK when the dict carries a pose ('location', 'quaternion_xyzw', ...), else CP_PNP_NOT_RUN. */
  CP_S_KPS_FUSION_MEAN = 192,  /* 16 */
  CP_S_KPS_FUSION_STD = 208,   /* 16 */
  CP_S_KPS_GT = 224,           /* 18, normalised, centre first */
  CP_S_HAS_CT = 242,           /* 0: 'ct' is absent and becomes the bbox centre                         */
  CP_S_HAS_KPS_GT = 243,       /* 0: no 'kps_gt' (CP_RENDER_GT then draws the centre only)              */
  CP_S_KPS_PNP_KF = 244,       /* 18, normalised: a 'kps_pnp_kf' the dict already carries               */
  CP_S_HAS_KPS_PNP_KF = 262
};
/* Tracker.init_track(meta) with meta['pre_dets'] (utils/tracker.py:21-48) for `batch` streams.  seeds: device fp32
 * [batch, S, CP_SEED_RECORD]; n_seeds: device int32 [batch].  n_seeds[b] < 0 leaves stream b untouched; otherwise
 * stream b is reset (id counter included) and the first min(n_seeds[b], S) seeds with score > new_thresh become tracks
 * 1, 2, ... in order, their filter initialised from the seed's own kps_fusion_mean / kps_fusion_std / tracking_hp and
 * their scale pool from obj_scale / obj_scale_uncertainty.  S must be in 0..max_tracks. */
int cp_tracker_seed(cp_tracker* trk, int32_t batch, const float* seeds, const int32_t* n_seeds, int32_t S, void* stream);
/* cp_tracker_seed with a stream map: row i (seeds[i], n_seeds[i]) seeds tracker stream stream_ids[i]. */
int cp_tracker_seed_ex(cp_tracker* trk, int32_t batch, const int32_t* stream_ids, const float* seeds,
                       const int32_t* n_seeds, int32_t S, void* stream);

/* Offsets (in floats) inside one CP_TRACK_RECORD slot.  [0, CP_POSE_RECORD) is the pose record of the detection the
 * track carries; its PnP fields hold the SECOND (filtered) solve whenever that produced a pose (pnp_shell mutates the
 * track dict, cuboid_pnp_shell.py:27-54). */
enum cp_track_field {
  CP_T_ID = 192, CP_T_AGE = 193, CP_T_ACTIVE = 194,
  CP_T_IN_BOXES = 195,         /* 1: the second PnP returned a tuple and conf_avg > 0.25 -> in `boxes` (tracker.py:278-281) */
  CP_T_PNP2_STATUS = 196,      /* cp_pnp_status of the second PnP                                          */
  CP_T_CONF_AVG = 197,
  CP_T_KPS_FUSION_MEAN = 200,  /* 16 */
  CP_T_KPS_FUSION_STD = 216,   /* 16 */
  CP_T_KPS_MEAN_KF = 232,      /* 16, -10000 where the filter confidence is < 0.15                         */
  CP_T_KPS_STD_KF = 248,       /* 16 */
  CP_T_OBJ_SCALE_KF = 264,     /* 3  */
  CP_T_OBJ_SCALE_UNC_KF = 267, /* 3  */
  CP_T_KPS_PNP_KF = 270,       /* 18 */
  CP_T_KPS_3D_CAM_KF = 288     /* 27 */
};

/* ---- stand-alone modulated deformable convolution (the `_ext` replacement) -- */
/* input [B,C,H,W], weight [Co,C,3,3], bias [Co], offset [B,18,H,W]
 * (channel 2k = dy, 2k+1 = dx of tap k), mask [B,9,H,W] (already sigmoid'ed),
 * output [B,Co,H,W]; all device fp32 NCHW.  3x3, stride 1, pad 1, dilation 1,
 * deformable_group 1 -- the only configuration CenterPose instantiates
 * (pose_dla_dcn.py:384).  Scratch is taken from the stream-ordered allocator. */
int cp_dcn_v2_forward(const float* input, const float* weight, const float* bias,
                      const float* offset, const float* mask, float* output,
                      int32_t B, int32_t C, int32_t H, int32_t W, int32_t Co, void* stream);

/* Same op with an explicit cp_precision (CP_PREC_FP32: CUDA cores; CP_PREC_TF32X3 / CP_PREC_BF16: wgmma). */
int cp_dcn_v2_forward_ex(const float* input, const float* weight, const float* bias, const float* offset,
                         const float* mask, float* output, int32_t B, int32_t C, int32_t H, int32_t W,
                         int32_t Co, int32_t precision, void* stream);

/* Backward of the same op: replaces `_ext.dcn_v2_backward` (DCNv2/dcn_v2.py:63-76 -> src/cuda/dcn_v2_cuda.cu:206-335,
 * kernels dcn_v2_im2col_cuda.cu:197-330).  Inputs as in the forward plus grad_output [B,Co,H,W]; the five gradients
 * (grad_input [B,C,H,W], grad_offset [B,18,H,W], grad_mask [B,9,H,W], grad_weight [Co,C,3,3], grad_bias [Co]) are
 * OVERWRITTEN (the reference returns fresh tensors).  `precision` selects the kernel family of the column-gradient GEMM
 * (CP_PREC_FP32: CUDA cores; CP_PREC_TF32X3: wgmma, fp32-equivalent); the sampling pass and the weight-gradient GEMM
 * run in fp32.  grad_input is accumulated with float atomics (as in the reference), everything else in a fixed order.
 * Scratch (about B*H*W*(11*C + Co + 32) floats) comes from the stream-ordered allocator. */
int cp_dcn_v2_backward(const float* input, const float* weight, const float* offset, const float* mask,
                       const float* grad_output, float* grad_input, float* grad_offset, float* grad_mask,
                       float* grad_weight, float* grad_bias, int32_t B, int32_t C, int32_t H, int32_t W, int32_t Co,
                       int32_t precision, void* stream);

/* ---- single fused convolution (building block of the plan, exposed for layer-level parity tests) ----
 * out = [relu]( conv2d(x, weight, stride, pad) + bias [+ residual] ); x / residual / out are device fp32
 * NHWC ([B,H,W,Cin] / [B,Ho,Wo,Cout]), weight is OIHW like nn.Conv2d (pose_dla_dcn.py:37-44);
 * Cin % 16 == 0, Cout % 4 == 0.  bias / residual may be NULL. */
int cp_conv2d(const float* x, const float* weight, const float* bias, const float* residual, float* out,
              int32_t B, int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t k, int32_t stride,
              int32_t pad, int32_t relu, int32_t precision, void* stream);

/* ---- batched pre-process (next-row f-1) ------------------------------------ */
/* frames: device uint8 [B, src_h, src_w, 3] (BGR as cv2.imread gives);
 * out: device fp32 NCHW [B,3,dst_h,dst_w] = (warpAffine(frame)/255 - mean)/std with the
 * reference's fix_res affine (c = src centre, s = max(src_h, src_w)).  The warp is a bit-for-bit restatement of
 * cv2.warpAffine(INTER_LINEAR) for 8-bit frames (OpenCV's fixed-point remap: AB_SCALE 1024, INTER_BITS 5,
 * 15-bit integer weights), so the batched path feeds the network exactly what base_detector.py:128-134 does. */
int cp_preprocess(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w,
                  int32_t dst_h, int32_t dst_w, const float mean[3], const float std[3], void* stream);
/* Same with an explicit forward affine: trans_input = HOST pointer to the row-major 2x3 double matrix
 * meta['trans_input'] (source frame -> network input), e.g. for fix_short / keep_res or rotated crops. */
int cp_preprocess_affine(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w, int32_t dst_h,
                         int32_t dst_w, const double trans_input[6], const float mean[3], const float std[3], void* stream);
/* cp_preprocess_affine of each frame resized first, as pre_process does at a test scale (base_detector.py:94-96,
 * :128): out = (warpAffine(cv2.resize(frame, (rs_w, rs_h)), trans_input, (dst_w, dst_h)) / 255 - mean) / std, bit for
 * bit.  The resize is cv2's INTER_LINEAR for 8-bit frames (11-bit integer weights), computed per tap inside the warp,
 * so the resized frame is never stored.  rs_h x rs_w == src_h x src_w makes exactly the launch of
 * cp_preprocess_affine (cv2.resize copies such a frame).  Any size <= 0 returns CP_ERR_INVALID before any work. */
int cp_preprocess_resize_affine(const uint8_t* frames, float* out, int32_t B, int32_t src_h, int32_t src_w,
                                int32_t rs_h, int32_t rs_w, int32_t dst_h, int32_t dst_w, const double trans_input[6],
                                const float mean[3], const float std[3], void* stream);
/* A ragged batch in one launch: B frames of different sizes packed into one device buffer.  Frame b is uint8
 * [src_hw[b][0], src_hw[b][1], 3] starting `offsets[b]` bytes into `frames` (frames_bytes long); out: device fp32 NCHW
 * [B,3,dst_h,dst_w].  offsets (int64 [B]), src_hw (int32 [B,2]) and trans_input (double [B,6], row-major 2x3 forward
 * affines, or NULL) are HOST arrays owned by the caller and read before the call returns.  Frame b's output equals, bit
 * for bit, cp_preprocess_affine on that frame alone with trans_input[b], or cp_preprocess on it when trans_input is
 * NULL.  A frame that does not fit inside frames_bytes returns CP_ERR_INVALID before any work is enqueued.  A few
 * hundred bytes of per-frame parameters come from the stream-ordered allocator. */
int cp_preprocess_ragged(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                         float* out, int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input,
                         const float mean[3], const float std[3], void* stream);

/* YUV 4:2:0 frames as video decoders and cameras produce them, in cv2's layouts: one uint8 [3H/2, W] buffer per frame,
 * the Y plane [H, W] first, then
 *   CP_PIX_NV12: interleaved chroma rows [H/2, W], U at even and V at odd bytes (NVDEC's and most cameras' output);
 *   CP_PIX_I420: the U plane [H/2, W/2], then the V plane [H/2, W/2] (ffmpeg's yuv420p). */
enum cp_pixel_format {
  CP_PIX_NV12 = 0,
  CP_PIX_I420 = 1,
  CP_PIX_BGR = 2,  /* interleaved uint8 [H, W, 3]; taken by cp_preprocess_slots_dev and cp_preprocess_slots_ragged_dev
                    * (cp_preprocess_yuv420 refuses it) */
  /* Camera formats, ffmpeg's pix_fmt names; one uint8 [H, W, C] buffer per frame.  Each is converted to BGR inside the
   * warp, per tap, bit for bit what cv2.cvtColor gives with the code named (taps outside the frame are BGR 0).  Taken by
   * cp_preprocess_formats, cp_preprocess_slots_dev, the frame tables and their launches; cp_preprocess_yuv420 refuses
   * them.  The values are grouped by family; those in between are not formats. */
  CP_PIX_RGB24 = 16,     /* [H, W, 3] R G B (ROS 2 / PIL / PyAV "rgb24"): COLOR_RGB2BGR */
  CP_PIX_RGBA = 17,      /* [H, W, 4] R G B A, alpha ignored: COLOR_RGBA2BGR */
  CP_PIX_BGRA = 18,      /* [H, W, 4] B G R A, alpha ignored: COLOR_BGRA2BGR */
  CP_PIX_YUYV422 = 32,   /* [H, W, 2], W even, Y0 U Y1 V per pixel pair (V4L2 YUYV, GStreamer YUY2): COLOR_YUV2BGR_YUYV */
  CP_PIX_UYVY422 = 33,   /* [H, W, 2], W even, U Y0 V Y1 per pixel pair (V4L2 / GStreamer UYVY): COLOR_YUV2BGR_UYVY */
  /* Sensor formats: one uint8 [H, W] plane per frame.  A Bayer mosaic is named after its pixels (0,0) (0,1) / (1,0)
   * (1,1) as ffmpeg, V4L2 and ROS name it; cv2 names the same mosaic after the block at (1,1), so the codes cross.  The
   * demosaic is cv2's bilinear one (an in-frame border pixel takes the BGR of the nearest interior pixel); a mosaic needs
   * at least 3 x 3 pixels (cv2 gives a black image below that; these refuse it). */
  CP_PIX_GRAY = 48,          /* Y (ROS mono8, V4L2 GREY, GStreamer GRAY8): COLOR_GRAY2BGR, B = G = R = Y */
  CP_PIX_BAYER_RGGB8 = 49,   /* R G / G B (V4L2 RGGB): COLOR_BayerBG2BGR */
  CP_PIX_BAYER_BGGR8 = 50,   /* B G / G R (V4L2 BA81): COLOR_BayerRG2BGR */
  CP_PIX_BAYER_GBRG8 = 51,   /* G B / R G (V4L2 GBRG): COLOR_BayerGR2BGR */
  CP_PIX_BAYER_GRBG8 = 52,   /* G R / B G (V4L2 GRBG): COLOR_BayerGB2BGR */
  /* not a frame format: a launch over a table of per-frame formats (cp_preprocess_frame_table_formats) */
  CP_PIX_PER_FRAME = 64,
  /* not a frame format: OR-ed into a format or CP_PIX_PER_FRAME, the launch code of a table with coordinate maps
   * (cp_preprocess_frame_table_maps) */
  CP_PIX_REMAP = 128
};
/* cp_preprocess_ragged on YUV 4:2:0 frames: frame b is [src_hw[b][0] * 3 / 2, src_hw[b][1]] uint8 in `format`, i.e.
 * src_hw[b][0] * src_hw[b][1] * 3 / 2 bytes starting `offsets[b]` bytes into `frames`; src_hw holds the IMAGE sizes
 * (H, W), which must be even.  Frame b's output equals, bit for bit, cp_preprocess_ragged on
 * cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / COLOR_YUV2BGR_I420) with the same trans_input (NULL: each frame's fix_res
 * affine).  The conversion (BT.601 limited range, 20-bit fixed point, one U, V per 2x2 block, as cv2) runs inside the
 * warp on the four taps of every output pixel; taps outside the frame are BGR 0, like warpAffine's border.  An odd size,
 * an unknown format or a frame that does not fit inside frames_bytes returns CP_ERR_INVALID before any work is enqueued.
 * A uniform batch is the case of equal sizes. */
int cp_preprocess_yuv420(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                         int32_t format, float* out, int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input,
                         const float mean[3], const float std[3], void* stream);
/* cp_preprocess_ragged with one pixel format per frame: frame b is in formats[b] (HOST int32 [B], any cp_pixel_format
 * but CP_PIX_PER_FRAME), its buffer shape given by that format and the image size src_hw[b] = (H, W) (4:2:0: both even;
 * 4:2:2: W even; a Bayer mosaic: both at least 3).  Frame b's output equals, bit for bit, cp_preprocess_ragged on
 * cv2.cvtColor(frame) to BGR with the same trans_input (NULL: each frame's fix_res affine).  One launch: one format's
 * walk when every frame has it, else a walk that reads each frame's format from the per-frame parameters.  An unknown
 * format, a size its format cannot have or a frame that does not fit inside frames_bytes at its format's size returns
 * CP_ERR_INVALID before any work is enqueued. */
int cp_preprocess_formats(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                          const int32_t* formats, float* out, int32_t B, int32_t dst_h, int32_t dst_w,
                          const double* trans_input, const float mean[3], const float std[3], void* stream);

/* The pre-process of one tracking step of B video slots, safe to capture in a CUDA graph: it reads no host memory and
 * allocates nothing once enqueued, so a replay runs it with the arguments it was captured with.  frames: device uint8, B
 * frames of one image size (src_h, src_w) in `format` (cp_pixel_format; YUV 4:2:0 needs an even size, a Bayer mosaic at
 * least 3 x 3), frame b at byte b * (bytes of one frame).  trans_input: HOST row-major 2x3 forward affine for every
 * frame, read before the call returns (NULL: the fix_res affine of the size, as cp_preprocess).  out: device fp32
 * [B,3,dst_h,dst_w], frame b bit for bit what cp_preprocess_affine (BGR), cp_preprocess_yuv420 (NV12 / I420) or
 * cp_preprocess_formats gives for it.  start: device int32 [B] read when the kernel runs, or NULL; where start[b] != 0
 * frame b's output is written to prev[b] (device fp32 [B,3,dst_h,dst_w]) as well: a slot whose video starts with this
 * frame takes it as its previous frame.  start and prev are both given or both NULL.  Bad arguments return CP_ERR_INVALID
 * before any work is enqueued. */
int cp_preprocess_slots_dev(const uint8_t* frames, int32_t format, int32_t B, int32_t src_h, int32_t src_w,
                            int32_t dst_h, int32_t dst_w, const double* trans_input, const float mean[3],
                            const float std[3], const int32_t* start, float* out, float* prev, void* stream);

/* The pre-process of one tracking step of B video slots whose frames differ in size, safe to capture in a CUDA graph.
 * It takes two calls:
 *   - cp_preprocess_frame_table, once, when the graph is built: the per-frame parameters (byte offset, size and
 *     inverted affine of every frame) are checked on the host and written to `table`, caller-owned DEVICE memory of
 *     cp_preprocess_frame_table_bytes(B) bytes (8-byte aligned).  offsets (int64 [B]), src_hw (int32 [B,2], image sizes
 *     (H, W)) and trans_input (double [B,6] row-major 2x3 forward affines, or NULL for each frame's fix_res affine) are
 *     HOST arrays read before the call returns.  It runs the checks of cp_preprocess_ragged / cp_preprocess_yuv420: a
 *     null pointer, B <= 0, a frame that does not fit inside frames_bytes, an odd size in a YUV 4:2:0 format or an
 *     unknown format return CP_ERR_INVALID before any work.  The table is uploaded on `stream` and the call waits for
 *     the copy, so it must not be called inside a capture.
 *   - cp_preprocess_slots_ragged_dev, the captured call: frames (a device buffer of at least frames_bytes bytes, laid out
 *     as the table says), the table and start are device memory read when the kernel runs, nothing is allocated and no
 *     host memory is read after the call returns.  `format` must be the one the table was built for.  out: device fp32
 *     [B,3,dst_h,dst_w], frame b bit for bit what cp_preprocess_ragged (CP_PIX_BGR) or cp_preprocess_yuv420 (NV12 /
 *     I420) gives for it with the same offsets, sizes and affines.  start / prev as in cp_preprocess_slots_dev: where
 *     start[b] != 0 frame b's output is written to prev[b] as well, other rows of prev are not touched; both given or
 *     both NULL.  Bad arguments return CP_ERR_INVALID before any work is enqueued. */
int64_t cp_preprocess_frame_table_bytes(int32_t B);
int cp_preprocess_frame_table(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int32_t format,
                              int32_t B, int32_t dst_h, int32_t dst_w, const double* trans_input, void* table,
                              void* stream);
int cp_preprocess_slots_ragged_dev(const uint8_t* frames, const void* table, int32_t format, int32_t B, int32_t dst_h,
                                   int32_t dst_w, const float mean[3], const float std[3], const int32_t* start,
                                   float* out, float* prev, void* stream);
/* A frame table with one pixel format per frame (cameras of different kinds in one step): cp_preprocess_frame_table
 * with formats[b] (HOST int32 [B], any cp_pixel_format but CP_PIX_PER_FRAME) for frame b, checked the same way (an
 * unknown format, an odd width in 4:2:2 or odd size in 4:2:0, a mosaic below 3 x 3, a frame overrunning frames_bytes at
 * its format's size return CP_ERR_INVALID before any work).  The table has cp_preprocess_frame_table_bytes(B) bytes
 * and is launched by cp_preprocess_slots_ragged_dev and cp_preprocess_slots_rows_dev with format CP_PIX_PER_FRAME
 * (and only so): frame b's output is then bit for bit what the launch of a one-format table gives for it. */
int cp_preprocess_frame_table_formats(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                                      const int32_t* formats, int32_t B, int32_t dst_h, int32_t dst_w,
                                      const double* trans_input, void* table, void* stream);
/* Lens distortion: frames resampled through a coordinate map instead of an affine.  maps is a HOST array of B DEVICE
 * pointers (8-byte aligned); maps[b] is float32 [dst_h, dst_w, 2], the (x, y) source position in frame b of every
 * output pixel, e.g. cv2.initUndistortRectifyMap(K, D, None, [A; 0 0 1] @ K_new, (dst_w, dst_h), CV_32FC1) stacked on
 * the last axis.  maps[b] NULL: frame b keeps its affine (trans_input[b], or its fix_res affine when trans_input is
 * NULL).  A mapped frame's output is, bit for bit, cv2.remap(cv2.cvtColor(frame) to BGR, map x, map y, INTER_LINEAR,
 * BORDER_CONSTANT, 0), then normalised as every pre-process; map entries that are NaN, +-inf or beyond the int range
 * give the border value 0, as cv2.remap.  The caller owns the maps: they must hold their values and stay allocated
 * until every launch that reads them has finished (for a table, as long as the table is launched).
 *   - cp_preprocess_remap: cp_preprocess_formats with maps; the table is uploaded per call.
 *   - cp_preprocess_frame_table_maps: a frame table of cp_preprocess_frame_table_bytes(B) bytes, built as
 *     cp_preprocess_frame_table (format a cp_pixel_format, formats NULL) or cp_preprocess_frame_table_formats (format
 *     CP_PIX_PER_FRAME, formats HOST int32 [B]), with the same checks.  Mapped and unmapped frames may share it.  It is
 *     launched by cp_preprocess_slots_ragged_dev and cp_preprocess_slots_rows_dev with the launch code
 *     format | CP_PIX_REMAP (and only so); an unmapped frame's output is then bit for bit that of the table without
 *     maps.
 * Null pointers, B <= 0, a format / formats pair other than those above, a map that is not 8-byte aligned and every
 * check of the tables without maps return CP_ERR_INVALID before any work. */
int cp_preprocess_remap(const uint8_t* frames, int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw,
                        const int32_t* formats, const float* const* maps, float* out, int32_t B, int32_t dst_h,
                        int32_t dst_w, const double* trans_input, const float mean[3], const float std[3], void* stream);
int cp_preprocess_frame_table_maps(int64_t frames_bytes, const int64_t* offsets, const int32_t* src_hw, int32_t format,
                                   const int32_t* formats, const float* const* maps, int32_t B, int32_t dst_h,
                                   int32_t dst_w, const double* trans_input, void* table, void* stream);
/* The pre-process of one tracking step in which only some of the S slots of a cp_preprocess_frame_table have a frame,
 * safe to capture in a CUDA graph.  Row n of the B live rows is slot rows[n]: out[n] (device fp32 [B,3,dst_h,dst_w]) is
 * bit for bit what cp_preprocess_slots_ragged_dev gives for that slot's frame.  rows (int32 [B]), start (int32 [S], per
 * SLOT) and the table are DEVICE memory read when the kernel runs, WITHOUT checking: the caller guarantees every
 * rows[n] is in 0..S-1 and none appears twice.  store (device fp32 [S,3,dst_h,dst_w], the previous frame of every slot)
 * and prev (device fp32 [B,3,dst_h,dst_w]) are both given or both NULL; with them the walk also sets
 *   prev[n] = start[rows[n]] ? out[n] : store[rows[n]],  then  store[rows[n]] = out[n],
 * so a slot that starts its video takes this frame as its previous frame, and an idle slot's stored frame is not
 * touched.  start NULL: no slot starts.  Bad arguments return CP_ERR_INVALID before any work is enqueued. */
int cp_preprocess_slots_rows_dev(const uint8_t* frames, const void* table, int32_t format, const int32_t* rows, int32_t B,
                                 int32_t dst_h, int32_t dst_w, const float mean[3], const float std[3],
                                 const int32_t* start, float* store, float* out, float* prev, void* stream);
/* A row gather, safe to capture in a CUDA graph: dst row i = src row map[i], or zeros where map[i] < 0, for i in 0..n-1,
 * rows of row_bytes bytes (a positive multiple of 4; src and dst 4-byte aligned).  map is a DEVICE int32 [n] read when
 * the kernel runs, WITHOUT checking: the caller guarantees every map[i] is below the rows of src.  Bad arguments return
 * CP_ERR_INVALID before any work is enqueued. */
int cp_gather_rows_dev(const void* src, void* dst, int64_t row_bytes, int32_t n, const int32_t* map, void* stream);

/* ---- JPEG decode (jpeg.cu) -------------------------------------------------
 * Baseline sequential JPEG (SOF0 / SOF1, 8-bit, one interleaved scan of 1 or 3 components, luma sampling 1x1, 2x1,
 * 1x2, 2x2 or 4x1 with chroma 1x1, any restart interval, 8- or 16-bit DQT, DHT present or absent -- absent tables are
 * the standard ones of T.81 Annex K.3, as MJPEG frames need) decoded on the device into uint8 BGR [H, W, 3], bit for bit
 * cv2.imdecode(bytes, IMREAD_COLOR): libjpeg-turbo's integer pipeline (islow IDCT, fancy chroma up-sampling, the
 * jdcolor.c fixed-point YCbCr -> BGR) and the EXIF orientation applied as cv2 applies it.  Everything else is refused by
 * cp_jpeg_parse with a cp_jpeg_refusal before any device work. */
enum cp_jpeg_refusal {
  CP_JPEG_OK = 0,
  CP_JPEG_NOT_JPEG = 1,       /* no SOI */
  CP_JPEG_TRUNCATED = 2,      /* the headers end before the scan */
  CP_JPEG_PROGRESSIVE = 3,    /* SOF2 / SOF6 / SOF10 / SOF14 */
  CP_JPEG_LOSSLESS = 4,       /* SOF3 / SOF7 / SOF11 / SOF15 */
  CP_JPEG_ARITHMETIC = 5,     /* SOF9 (and the other arithmetic SOFs), DAC */
  CP_JPEG_PRECISION = 6,      /* samples other than 8 bits */
  CP_JPEG_COMPONENTS = 7,     /* not 1 or 3 components */
  CP_JPEG_MULTI_SCAN = 8,     /* a scan without every component, or a second scan */
  CP_JPEG_DNL = 9,            /* the height comes from a DNL marker */
  CP_JPEG_SAMPLING = 10,      /* another sampling layout */
  CP_JPEG_RGB = 11,           /* RGB-coded (Adobe transform 0, or component ids 'R' 'G' 'B') */
  CP_JPEG_BAD_TABLE = 12,     /* a missing or malformed DQT / DHT */
  CP_JPEG_BAD_HEADER = 13,    /* any other malformed header */
  CP_JPEG_TOO_LARGE = 14      /* more than 2^30 pixels (cv2.imread refuses them too, CV_IO_MAX_IMAGE_PIXELS) */
};
#define CP_JPEG_MAX_COMPONENTS 3
/* One Huffman table, derived on the host: look[code of the next 9 bits] = (length << 8) | symbol for codes of at most
 * 9 bits (0 otherwise); longer codes through libjpeg's maxcode / valoffset (maxcode[l] = -1: no code of length l). */
typedef struct cp_jpeg_huff {
  uint16_t look[512];
  int32_t maxcode[18];
  int32_t valoffset[18];
  uint8_t vals[256];
} cp_jpeg_huff;
/* What cp_jpeg_parse reads from a file.  width x height is the coded frame, out_h x out_w the decoded image after the
 * EXIF orientation (1..8).  The scan's entropy-coded bytes are [scan_begin, scan_end) of the file. */
typedef struct cp_jpeg_header {
  int32_t status;                 /* cp_jpeg_refusal */
  int32_t width, height, out_h, out_w, orientation;
  int32_t ncomp;                  /* 1 (gray) or 3 (YCbCr) */
  int32_t hmax, vmax;             /* luma sampling; 1 x 1 for gray */
  int32_t mcux, mcuy, blocks_per_mcu, restart_interval;
  int64_t scan_begin, scan_end;
  int32_t comp_h[CP_JPEG_MAX_COMPONENTS], comp_v[CP_JPEG_MAX_COMPONENTS];
  int16_t quant[CP_JPEG_MAX_COMPONENTS][64];          /* natural order, as the IDCT multiplies (libjpeg's short) */
  cp_jpeg_huff dc[CP_JPEG_MAX_COMPONENTS], ac[CP_JPEG_MAX_COMPONENTS];
} cp_jpeg_header;
/* Host only, no GPU: parses the n bytes of a JPEG file and fills *h.  Returns 0 when the file is supported, else
 * CP_ERR_INVALID with the reason in h->status (and cp_last_error). */
int cp_jpeg_parse(const uint8_t* bytes, int64_t n, cp_jpeg_header* h);
/* Device workspace bytes cp_jpeg_decode needs for these B parsed headers at any subseq_words; 0 for bad arguments. */
size_t cp_jpeg_workspace_bytes(const cp_jpeg_header* headers, int32_t B);
/* Decodes B parsed JPEGs in one launch per phase.  headers: HOST [B]; file b's bytes start byte_offsets[b] (HOST int64)
 * into the DEVICE buffer d_bytes; its BGR image (uint8 [out_h, out_w, 3]) is written at DEVICE d_bgr + out_offsets[b]
 * (HOST int64).  d_errors: DEVICE int32 [B], set to 0 for a frame decoded exactly and to a cp_jpeg_error mask for a
 * corrupt stream; every read is bounded by its restart segment, so a corrupt frame touches nothing but its error word
 * and its own output.  subseq_words: the length in 32-bit words of the subsequences of the parallel Huffman decode (0
 * = the library's default).  The call waits on `stream` once per synchronisation round of the Huffman decode.  Bad
 * arguments (a refused header, a small workspace) return CP_ERR_INVALID before any work. */
enum cp_jpeg_error {
  CP_JPEG_ERR_CODE = 1,       /* a Huffman code that is in no table */
  CP_JPEG_ERR_RUN = 2,        /* an AC run past coefficient 63 */
  CP_JPEG_ERR_SHORT = 4,      /* a restart segment ends before its MCU count */
  CP_JPEG_ERR_RESTART = 8,    /* a missing or misnumbered RST marker */
  CP_JPEG_ERR_SYNC = 16       /* cp_jpeg_decode_slots_dev: a CTA waited about a second for its predecessor's state */
};
int cp_jpeg_decode(const cp_jpeg_header* headers, int32_t B, const uint8_t* d_bytes, const int64_t* byte_offsets,
                   uint8_t* d_bgr, const int64_t* out_offsets, void* workspace, size_t ws_bytes, int32_t* d_errors,
                   int32_t subseq_words, void* stream);
/* The synchronisation rounds the last cp_jpeg_decode of this thread took (1 when every subsequence started exact). */
int cp_jpeg_last_rounds(void);

/* The slot decode, safe to capture in a CUDA graph: S slots of fixed decoded size hw[s] = (out_h, out_w) (HOST int32
 * [S][2], after the EXIF orientation), each taking one encoded frame of at most max_bytes[s] bytes (HOST int64 [S]) per
 * call.  Every grid and workspace offset depends only on S, hw, max_bytes and subseq_words; what changes per frame
 * (sampling, quality, tables, restart interval, orientation, length) is read on the device from a control block.  A
 * call: cp_jpeg_slots_prepare fills the block on the host, the caller copies it to a DEVICE buffer of
 * cp_jpeg_slots_block_bytes(S) bytes and slot s's file to d_bytes + the sum of max_bytes[0..s-1], and the captured
 * cp_jpeg_decode_slots_dev decodes.  The result is bit for bit cp_jpeg_decode's (cv2.imdecode's) at any
 * subseq_words. */
/* Device workspace bytes of these slots at subseq_words (0 = the default); 0 for bad arguments.  Host only. */
size_t cp_jpeg_slots_workspace_bytes(int32_t S, const int32_t* hw, const int64_t* max_bytes, int32_t subseq_words);
/* Bytes of the control block of S slots: S cp_jpeg_header, then the per-slot jobs (256-byte aligned); 0 for S <= 0. */
size_t cp_jpeg_slots_block_bytes(int32_t S);
/* Host only, no GPU: fills host_block (cp_jpeg_slots_block_bytes(S) bytes) for one call.  headers[s]: slot s's file
 * parsed by cp_jpeg_parse; nbytes[s]: its length, 0 to skip the slot this call (its header in the block is zeroed, its
 * output is not written and its error word is 0); out_offsets[s]: where its BGR image [out_h, out_w, 3] goes in d_bgr.
 * A live slot whose header is refused, decodes to another size than hw[s], or has more than max_bytes[s] bytes (or a
 * scan past nbytes[s]) returns CP_ERR_INVALID naming the slot, and the block is left as it was. */
int cp_jpeg_slots_prepare(int32_t S, const int32_t* hw, const int64_t* max_bytes, int32_t subseq_words,
                          const cp_jpeg_header* headers, const int64_t* nbytes, const int64_t* out_offsets,
                          void* host_block);
/* Decodes the slots of the DEVICE block d_block with no host round trip: one launch per phase over capacity-sized
 * grids, the Huffman synchronisation in one chained launch.  d_errors: DEVICE int32 [S], each slot's cp_jpeg_error mask
 * (0 for a skipped slot).  A corrupt frame touches nothing but its own error word, workspace regions and output. */
int cp_jpeg_decode_slots_dev(const void* d_block, int32_t S, const int32_t* hw, const int64_t* max_bytes,
                             int32_t subseq_words, const uint8_t* d_bytes, uint8_t* d_bgr, void* workspace,
                             size_t ws_bytes, int32_t* d_errors, void* stream);
/* Safe to capture: d_n_valid[m * n + r] = 0 for m < M, r < n when d_errors[slot] != 0, slot = d_rows[r] (DEVICE int32
 * [n]) or r when d_rows is NULL.  A slot whose frame did not decode exactly detects nothing. */
int cp_jpeg_mask_counts_dev(const int32_t* d_errors, const int32_t* d_rows, int32_t n, int32_t M, int32_t* d_n_valid,
                            void* stream);

/* ---- misc ------------------------------------------------------------------ */
int cp_version(void);
const char* cp_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* CENTERPOSE_B200_H_ */

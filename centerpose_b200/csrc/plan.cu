// Plan = static layer schedule + activation arena + packed weights for one
// (arch, heads, batch, resolution) configuration.  The topology below follows
// the reference definitions (citations relative to
// /root/reference/src/lib/models/networks):
//   pose_dla_dcn.py:227-322  DLA-34 base    (dla34(): levels [1,1,1,2,2,1],
//                                            channels [16,32,64,128,256,512], :340-346)
//   pose_dla_dcn.py:171-224  Tree / Root / BasicBlock wiring and concat order
//   pose_dla_dcn.py:392-443  IDAUp / DLAUp  (proj DCN -> depthwise ConvT up -> + skip -> node DCN)
//   pose_dla_dcn.py:457-570  DLASeg: ida_up, heads (3x3 -> [GN] -> ReLU -> 1x1), convGRU routing
//   DCNv2/dcn_v2.py:97-128   DCN = 3x3 conv -> 27 ch (18 offsets + 9 mask logits) + deformable 3x3
//   convGRU.py:20-94, GN.py:4-9
// and the ResNet family (resnet() below, msra_resnet.py):
//   msra_resnet.py:116-124, 235-252  stem (7x7/2 conv, BN, ReLU, 3x3/2 max-pool), pre_* stems :126-147, layer1..4
//   msra_resnet.py:35-105, 178-193   BasicBlock / Bottleneck, downsample; resnet_spec :300-304
//   msra_resnet.py:150-154, 208-233  deconv_layers: 3 x (ConvTranspose2d 4x4/2/1, BN, ReLU)
//   msra_resnet.py:157-174, 256-257  heads (3x3 -> ReLU -> 1x1)
#include <stdlib.h>
#include <string.h>

#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "arena_pack.h"
#include "common.cuh"

namespace cp {

thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
thread_local long long g_launch_counter = 0;
thread_local int g_pdl = 0;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

namespace {

struct Act {
  size_t off = 0;  // floats into the activation arena
  int C = 0, H = 0, W = 0;
  int stride = 0;  // pixel stride in floats
  int ext = -1;    // >= 0: external NCHW input index (0 images, 1 pre_img, 2 pre_hm, 3 pre_hm_hp)
  int buf = -1;    // >= 0: the arena allocation it is a view of (cp_plan::bufs)
};

// the external inputs a multi-track plan takes once per model and frame: pre_hm and pre_hm_hp
constexpr unsigned kMultiTrackInputs = (1u << 2) | (1u << 3);

enum OpType { OP_IGEMM, OP_MAXPOOL, OP_UPADD, OP_GN_RELU, OP_GRU, OP_MAXPOOL3 };

struct Op {
  OpType type = OP_IGEMM;
  std::string name;
  // igemm (IGEMM_DECONV: kh = kw = 4, stride 2, pad 1 as the layer is declared; igemm_params maps it to its phases)
  // and OP_MAXPOOL3 (src[0], out, optional res)
  Act src[4];
  int nsrc = 0;
  int mode = IGEMM_NHWC_VEC;
  Act out;
  int out_head = -1;  // >= 0: result goes to head output `out_head` as NCHW
  bool has_res = false, res_after_relu = false, relu = false;
  Act res;
  int kh = 1, kw = 1, stride = 1, pad = 0, Cin = 0, Cout = 0, CoutPad = 0, Kpad = 0;
  size_t w_off = 0, b_off = 0;
  int w_ld = 0;            // leading dimension of the fp32 packed weight matrix
  ConvKernel kernel;       // chosen before the arena exists (select_kernels)
  int last_ksplit = 0, last_path = CP_KPATH_NONE;     // what the op's latest launch did (cp_plan_op_ksegments)
  size_t tile_off = 0;     // bytes into the plan's tensor-core weight-tile buffer
  TmaMaps maps;            // conv_tma / dcn_tma: encoded once the arena exists (encode_maps)
  std::vector<int> head_children;   // merged heads 3x3 conv: indices of the per-head 1x1 ops that read its slices
  bool fuse_heads = false;          // ... which run inside its epilogue (conv_tma.cu), never touching HBM
  bool fused_away = false;          // this 1x1 op is computed by its parent's epilogue
  Act om;
  // up-sample
  int f = 0;
  size_t upw_off = 0;
  bool has_skip = false;
  Act skip;
  // group-norm
  size_t gamma_off = 0, beta_off = 0;
  int groups = 0, chanOffset = 0;
  // gru
  Act gx, gh, gprev;
  bool first_step = false;
};

enum PackType { PACK_CONV, PACK_BIAS, PACK_UP, PACK_VEC, PACK_DECONV };

struct PackJob {
  PackType type;
  std::string key;       // main tensor key
  std::string bias_key;  // conv bias key ("" = none)
  std::string bn;        // BN prefix ("" = none)
  int Cout = 0, Cin = 0, kh = 0, kw = 0, CoutPad = 0, Kpad = 0, ld = 0, colOff = 0;
  size_t dst = 0;        // floats into the weight arena (weights / bias / up / vec)
  size_t scale = 0;      // scratch scale vector (PACK_BIAS writes, PACK_CONV reads); 0 = none
  bool use_scale = false;
};

struct WRef {
  const float* p;
  int64_t n;
};

// One OP_IGEMM op as the builder declares it (Builder::conv).
struct ConvSpec {
  std::vector<Act> src;             // concatenated along channels; an external NCHW source makes it an IGEMM_NCHW_SCALAR stem
  int k = 1, stride = 1, pad = 0;   // IGEMM_DECONV: 4, 2, 1, as the ConvTranspose2d is declared
  int Cout = 0;
  bool relu = false;
  const Act* res = nullptr;         // added before the ReLU, or after it with res_after_relu
  bool res_after_relu = false;
  int head = -1;                    // >= 0: the output is head `head`'s NCHW tensor, else a new allocation
  int mode = IGEMM_NHWC_VEC;        // or IGEMM_DCN, reading its offsets / mask logits from `om`, or IGEMM_DECONV
  Act om;
  std::string wkey, bias_key, bn;   // the state-dict weight, bias and BatchNorm prefix packed for this op ("": none) ...
  size_t w_off = 0, b_off = 0;      // ... or, with wkey empty, where Builder::merged_weights packed them
};

}  // namespace
}  // namespace cp

using namespace cp;

struct cp_plan {
  cp_config cfg;
  std::vector<std::string> head_names;
  int B = 0, H = 0, W = 0;
  std::vector<Op> ops;
  std::vector<PackJob> jobs;
  float* act = nullptr;
  size_t act_floats = 0;
  float* wts = nullptr;
  size_t w_floats = 0;
  std::vector<Act> head_bufs;  // plan-owned NCHW head logits (cp_infer)
  bool loaded = false;
  int launches = 0;
  void* decode_ws = nullptr;
  size_t decode_ws_bytes = 0;
  double* gn_stats = nullptr;
  bool no_dcn_tma = false;       // CP_NO_DCN_TMA=1: deformable convs on the global-gather kernel (A/B measurements)
  unsigned char* umma_wts = nullptr;
  size_t umma_bytes = 0;
  float* splitk_ws = nullptr;      // conv_tma / dcn_tma split-K partial sums (kSplitkWsFloats)
  // multi-model plans (cp_plan_create_multi): model m's fp32 weights are wts + m * w_floats, its weight tiles
  // umma_wts + m * umma_bytes; the arena holds models * B images, model m's at [m * batch, (m + 1) * batch)
  int models = 1;
  std::vector<char> model_loaded;
  // bit e set: external input e holds one image per model and frame ([models, batch, ...]) rather than one per frame
  // (cp_plan_create_multi_track: pre_hm and pre_hm_hp, which each category draws from its own tracks)
  unsigned ext_per_model = 0;
  // Every arena allocation of the schedule (Builder::new_act) with the ops over which it is live, and its offset in
  // floats.  Without CP_PLAN_REUSE_ACTIVATIONS the offsets are the bump allocation's: every allocation has its own
  // memory.  With it they come from arena_pack(), and an allocation no op touches has none.
  bool reuse = false;
  bool invariant = false;          // CP_PLAN_BATCH_INVARIANT: every split-capable launch has fixed K segments
  std::vector<ArenaAlloc> bufs;
  std::vector<size_t> buf_off;
};

namespace cp {
namespace {

struct Builder {
  cp_plan* P;
  size_t act_cur = 0, w_cur = 0;
  int B;

  size_t walloc(size_t n) {
    size_t o = w_cur;
    w_cur += (n + 63) / 64 * 64;
    return o;
  }
  Act new_act(int C, int H, int W) {
    Act a;
    a.off = act_cur;
    a.C = C;
    a.H = H;
    a.W = W;
    a.stride = C;
    a.buf = (int)P->bufs.size();
    ArenaAlloc al;
    al.floats = arena_align((size_t)B * H * W * C);
    P->bufs.push_back(al);
    P->buf_off.push_back(act_cur);
    act_cur += al.floats;
    return a;
  }

  // The OP_IGEMM op of `s`: its padded GEMM shape, its output allocation, its weight storage and their pack jobs.
  Act conv(const ConvSpec& s) {
    const bool deconv = s.mode == IGEMM_DECONV;      // four 2x2-tap phase GEMMs, one [Kpad][CoutPad] block each
    Op op;
    op.nsrc = (int)s.src.size();
    for (int i = 0; i < op.nsrc; ++i) {
      op.src[i] = s.src[i];
      op.Cin += s.src[i].C;
    }
    op.mode = s.src[0].ext >= 0 ? IGEMM_NCHW_SCALAR : s.mode;
    op.kh = op.kw = s.k;
    op.stride = s.stride;
    op.pad = s.pad;
    op.Cout = s.Cout;
    op.CoutPad = op.w_ld = conv_cout_pad(s.Cout);
    op.Kpad = round_up((deconv ? 4 : s.k * s.k) * op.Cin, 16);
    op.relu = s.relu;
    if (s.res) {
      op.has_res = true;
      op.res = *s.res;
      op.res_after_relu = s.res_after_relu;
    }
    op.om = s.om;
    const int Hin = s.src[0].H, Win = s.src[0].W;
    const int Ho = deconv ? 2 * Hin : (Hin + 2 * s.pad - s.k) / s.stride + 1;
    const int Wo = deconv ? 2 * Win : (Win + 2 * s.pad - s.k) / s.stride + 1;
    op.out_head = s.head;
    // padded channels are never stored (the kernels mask n >= Cout), but a new allocation's pixel stride spans them:
    // the 27-channel offset / mask tensor is read in rows of 32
    if (s.head < 0) op.out = new_act(op.CoutPad, Ho, Wo);
    op.out.C = s.Cout;
    op.out.H = Ho;
    op.out.W = Wo;
    if (s.wkey.empty()) {
      op.w_off = s.w_off;
      op.b_off = s.b_off;
    } else {
      op.w_off = walloc((size_t)(deconv ? 4 : 1) * op.Kpad * op.CoutPad);
      op.b_off = walloc(op.CoutPad);
      add_pack(deconv ? PACK_DECONV : PACK_CONV, s.wkey, s.bias_key, s.bn, s.Cout, op.Cin, s.k, op.CoutPad, op.Kpad,
               op.CoutPad, 0, op.w_off, op.b_off);
    }
    op.name = s.wkey.empty() ? "conv" + std::to_string(s.k) + "x" + std::to_string(s.k) + "_merged_" + std::to_string(s.Cout)
                             : s.wkey.substr(0, s.wkey.rfind('.'));
    if (op.mode == IGEMM_DCN) op.name += "(dcn)";
    P->ops.push_back(op);
    return op.out;
  }

  // Several convs over one input, side by side in one [Kpad][keys.size() * Cout] weight matrix and bias, for one
  // N-wide conv (ConvSpec w_off / b_off): the merged heads 3x3s and the convGRU gate convs.  Returns (w_off, b_off).
  std::pair<size_t, size_t> merged_weights(const std::vector<std::string>& keys, bool bias, int Cin, int k, int Cout) {
    const int N = (int)keys.size() * Cout, Kpad = round_up(k * k * Cin, 16);
    const size_t w = walloc((size_t)Kpad * N), b = walloc(N);
    for (size_t i = 0; i < keys.size(); ++i)
      add_pack(PACK_CONV, keys[i] + ".weight", bias ? keys[i] + ".bias" : "", "", Cout, Cin, k, Cout, Kpad, N,
               (int)i * Cout, w, b);
    return {w, b};
  }

  // The bias (+ folded BN) job and the weight job of a [Kpad][CoutPad] block at column `colOff` of a matrix `ld` wide
  void add_pack(PackType type, const std::string& wkey, const std::string& bias_key, const std::string& bn, int Cout,
                int Cin, int k, int CoutPad, int Kpad, int ld, int colOff, size_t w_off, size_t b_off) {
    PackJob jb;
    jb.type = PACK_BIAS;
    jb.key = bias_key;
    jb.bn = bn;
    jb.Cout = Cout;
    jb.CoutPad = CoutPad;
    jb.dst = b_off + colOff;
    jb.scale = walloc(CoutPad);
    P->jobs.push_back(jb);
    PackJob jw;
    jw.type = type;
    jw.key = wkey;
    jw.Cout = Cout;
    jw.Cin = Cin;
    jw.kh = jw.kw = k;
    jw.CoutPad = CoutPad;
    jw.Kpad = Kpad;
    jw.ld = ld;
    jw.colOff = colOff;
    jw.dst = w_off;
    jw.scale = jb.scale;
    jw.use_scale = !bn.empty();
    P->jobs.push_back(jw);
  }

  Act conv_bn(const Act& x, const std::string& convkey, const std::string& bnkey, int Cout, int k, int stride,
              int pad, bool relu, const Act* res = nullptr) {
    return conv({.src = {x}, .k = k, .stride = stride, .pad = pad, .Cout = Cout, .relu = relu, .res = res,
                 .wkey = convkey + ".weight", .bn = bnkey});
  }

  Act maxpool(const Act& x) {
    Op op;
    op.type = OP_MAXPOOL;
    op.src[0] = x;
    op.out = new_act(x.C, x.H / 2, x.W / 2);
    op.name = "maxpool2";
    P->ops.push_back(op);
    return op.out;
  }

  // MaxPool2d(3, 2, 1) [+ residual] (msra_resnet.py:120, 242-247)
  Act maxpool3(const Act& x, const Act* res, const std::string& name) {
    Op op;
    op.type = OP_MAXPOOL3;
    op.src[0] = x;
    if (res) {
      op.has_res = true;
      op.res = *res;
    }
    op.out = new_act(x.C, x.H / 2, x.W / 2);
    op.name = name;
    P->ops.push_back(op);
    return op.out;
  }

  // ConvTranspose2d(Cin, Cout, 4, stride 2, pad 1, bias=False) + folded BN + ReLU (msra_resnet.py:219-230)
  Act deconv_bn(const Act& x, const std::string& wkey, const std::string& bn, int Cout) {
    return conv({.src = {x}, .k = 4, .stride = 2, .pad = 1, .Cout = Cout, .relu = true, .mode = IGEMM_DECONV, .wkey = wkey,
                 .bn = bn});
  }

  // BasicBlock (msra_resnet.py:35-64) and Bottleneck (:67-105): out = relu(bn(conv) + residual), the stride on conv1 of
  // a BasicBlock and on the 3x3 conv2 of a Bottleneck; `downsample` (1x1 at that stride + BN) when the shape changes
  Act res_block(const Act& x, const std::string& p, int planes, int stride, bool bottleneck) {
    const int Cout = bottleneck ? 4 * planes : planes;
    Act residual = x;
    if (stride != 1 || x.C != Cout)
      residual = conv_bn(x, p + ".downsample.0", p + ".downsample.1", Cout, 1, stride, 0, false);
    if (!bottleneck) {
      Act y = conv_bn(x, p + ".conv1", p + ".bn1", planes, 3, stride, 1, true);
      return conv_bn(y, p + ".conv2", p + ".bn2", planes, 3, 1, 1, true, &residual);
    }
    Act y = conv_bn(x, p + ".conv1", p + ".bn1", planes, 1, 1, 0, true);
    y = conv_bn(y, p + ".conv2", p + ".bn2", planes, 3, stride, 1, true);
    return conv_bn(y, p + ".conv3", p + ".bn3", Cout, 1, 1, 0, true, &residual);
  }

  Act basic_block(const Act& x, const std::string& p, int Cout, int stride, const Act& residual) {
    Act y = conv_bn(x, p + ".conv1", p + ".bn1", Cout, 3, stride, 1, true);
    return conv_bn(y, p + ".conv2", p + ".bn2", Cout, 3, 1, 1, true, &residual);
  }

  // levels == 1 Tree
  Act tree1(const Act& x, const std::string& p, int Cin, int Cout, int stride, bool level_root,
            const std::vector<Act>& extra) {
    std::vector<Act> children = extra;
    Act bottom = stride > 1 ? maxpool(x) : x;
    Act residual = bottom;
    if (Cin != Cout) residual = conv_bn(bottom, p + ".project.0", p + ".project.1", Cout, 1, 1, 0, false);
    if (level_root) children.push_back(bottom);
    Act x1 = basic_block(x, p + ".tree1", Cout, stride, residual);
    Act x2 = basic_block(x1, p + ".tree2", Cout, 1, x1);
    std::vector<Act> cat = {x2, x1};
    for (auto& c : children) cat.push_back(c);
    return conv({.src = cat, .Cout = Cout, .relu = true, .wkey = p + ".root.conv.weight", .bn = p + ".root.bn"});
  }

  // levels == 2 Tree with level_root (level3 / level4); the outer `project` is dead compute
  Act tree2(const Act& x, const std::string& p, int Cin, int Cout, int stride) {
    Act bottom = maxpool(x);
    Act x1 = tree1(x, p + ".tree1", Cin, Cout, stride, false, {});
    return tree1(x1, p + ".tree2", Cout, Cout, 1, false, {bottom, x1});
  }

  // DCN (DCNv2/dcn_v2.py:97-128): the 3x3 offset / mask conv (18 offsets + 9 mask logits), then the deformable 3x3
  Act deform_conv(const Act& x, const std::string& p, int Cout) {
    const Act om = conv({.src = {x}, .k = 3, .pad = 1, .Cout = 27, .wkey = p + ".conv.conv_offset_mask.weight",
                         .bias_key = p + ".conv.conv_offset_mask.bias"});
    return conv({.src = {x}, .k = 3, .pad = 1, .Cout = Cout, .relu = true, .mode = IGEMM_DCN, .om = om,
                 .wkey = p + ".conv.weight", .bias_key = p + ".conv.bias", .bn = p + ".actf.0"});
  }

  Act up_add(const Act& x, const std::string& key, int f, const Act& skip) {
    Op op;
    op.type = OP_UPADD;
    op.src[0] = x;
    op.f = f;
    op.has_skip = true;
    op.skip = skip;
    op.out = new_act(x.C, x.H * f, x.W * f);
    op.upw_off = walloc((size_t)x.C * 4 * f * f);
    PackJob j;
    j.type = PACK_UP;
    j.key = key;
    j.Cout = x.C;
    j.kh = 2 * f;
    j.dst = op.upw_off;
    P->jobs.push_back(j);
    op.name = key.substr(0, key.rfind('.'));
    P->ops.push_back(op);
    return op.out;
  }

  // IDAUp.forward (pose_dla_dcn.py:411-417); up_f[j] = up-sampling factor of proj_j
  void ida_up(std::vector<Act>& layers, const std::string& p, int startp, int endp, int o,
              const std::vector<int>& up_f) {
    for (int i = startp + 1; i < endp; ++i) {
      int j = i - startp;
      Act t = deform_conv(layers[i], p + ".proj_" + std::to_string(j), o);
      Act u = up_add(t, p + ".up_" + std::to_string(j) + ".weight", up_f[j], layers[i - 1]);
      layers[i] = deform_conv(u, p + ".node_" + std::to_string(j), o);
    }
  }
};

bool is_res_arch(int arch) { return arch >= CP_ARCH_RES_18 && arch <= CP_ARCH_RES_152; }

// PoseResNet up to the heads (msra_resnet.py:235-254): stem, layer1..4 (resnet_spec :300-304), deconv_layers.
template <class Ext>
Act resnet(Builder& b, const cp_config& c, Ext ext) {
  static const int kBlocks[5][4] = {{2, 2, 2, 2}, {3, 4, 6, 3}, {3, 4, 6, 3}, {3, 4, 23, 3}, {3, 8, 36, 3}};
  const int d = c.arch - CP_ARCH_RES_18;
  const bool bottleneck = c.arch >= CP_ARCH_RES_50;
  Act x = b.conv({.src = {ext(0, 3)}, .k = 7, .stride = 2, .pad = 3, .Cout = 64, .relu = true, .wkey = "conv1.weight",
                  .bn = "bn1"});
  x = b.maxpool3(x, nullptr, "maxpool");
  if (c.tracking) {      // x = x + pre_img_layer(pre_img) + pre_hm_layer(pre_hm) + pre_hm_hp_layer(pre_hm_hp), in this order
    const char* keys[3] = {"pre_img_layer", "pre_hm_layer", "pre_hm_hp_layer"};
    const int cin[3] = {3, 1, 8};
    for (int e = 0; e < 3; ++e) {
      const std::string k = keys[e];
      Act t = b.conv({.src = {ext(e + 1, cin[e])}, .k = 7, .stride = 2, .pad = 3, .Cout = 64, .relu = true,
                      .wkey = k + ".0.weight", .bn = k + ".1"});
      x = b.maxpool3(t, &x, k + ".3");
    }
  }
  for (int l = 0; l < 4; ++l)
    for (int j = 0; j < kBlocks[d][l]; ++j)
      x = b.res_block(x, "layer" + std::to_string(l + 1) + "." + std::to_string(j), 64 << l, (l > 0 && j == 0) ? 2 : 1,
                      bottleneck);
  for (int i = 0; i < 3; ++i)
    x = b.deconv_bn(x, "deconv_layers." + std::to_string(3 * i) + ".weight", "deconv_layers." + std::to_string(3 * i + 1),
                    256);
  return x;
}

int build_graph(cp_plan* P) {
  const cp_config& c = P->cfg;
  Builder b;
  b.P = P;
  b.B = P->B * P->models;
  P->ops.clear();
  P->jobs.clear();
  P->bufs.clear();
  P->buf_off.clear();
  const int H = P->H, W = P->W;

  auto ext = [&](int idx, int C) {
    Act a;
    a.ext = idx;
    a.C = C;
    a.H = H;
    a.W = W;
    return a;
  };
  Act F;      // the stride-4 feature the heads read
  if (is_res_arch(c.arch)) {
    F = resnet(b, c, ext);
  } else {
    // ---- DLA-34 base (pose_dla_dcn.py:310-322)
    Act x = b.conv({.src = {ext(0, 3)}, .k = 7, .pad = 3, .Cout = 16, .relu = true, .wkey = "base.base_layer.0.weight",
                    .bn = "base.base_layer.1"});
    if (c.tracking) {      // x = x + relu(bn(conv(pre_*))) for pre_img, pre_hm, pre_hm_hp, in this order
      const char* keys[3] = {"base.pre_img_layer", "base.pre_hm_layer", "base.pre_hm_hp_layer"};
      const int cin[3] = {3, 1, 8};
      for (int e = 0; e < 3; ++e)
        x = b.conv({.src = {ext(e + 1, cin[e])}, .k = 7, .pad = 3, .Cout = 16, .relu = true, .res = &x,
                    .res_after_relu = true, .wkey = std::string(keys[e]) + ".0.weight", .bn = std::string(keys[e]) + ".1"});
    }
    std::vector<Act> lv(6);
    lv[0] = b.conv_bn(x, "base.level0.0", "base.level0.1", 16, 3, 1, 1, true);
    lv[1] = b.conv_bn(lv[0], "base.level1.0", "base.level1.1", 32, 3, 2, 1, true);
    lv[2] = b.tree1(lv[1], "base.level2", 32, 64, 2, false, {});
    lv[3] = b.tree2(lv[2], "base.level3", 64, 128, 2);
    lv[4] = b.tree2(lv[3], "base.level4", 128, 256, 2);
    lv[5] = b.tree1(lv[4], "base.level5", 256, 512, 2, true, {});

    // ---- DLAUp (pose_dla_dcn.py:420-443), first_level = 2
    const int first = 2;
    std::vector<int> channels = {64, 128, 256, 512};
    std::vector<int> in_channels = channels;
    std::vector<int> scales = {1, 2, 4, 8};
    struct Ida {
      int o;
      std::vector<int> up_f;
    };
    std::vector<Ida> idas;
    const int nch = (int)channels.size();
    for (int i = 0; i < nch - 1; ++i) {
      int j = nch - i - 2;
      Ida d;
      d.o = channels[j];
      for (int t = j; t < nch; ++t) d.up_f.push_back(scales[t] / scales[j]);
      idas.push_back(d);
      for (int t = j + 1; t < nch; ++t) {
        scales[t] = scales[j];
        in_channels[t] = channels[j];
      }
    }
    std::vector<Act> layers = lv;
    std::vector<Act> out = {layers.back()};
    for (int i = 0; i < (int)layers.size() - first - 1; ++i) {
      b.ida_up(layers, "dla_up.ida_" + std::to_string(i), (int)layers.size() - i - 2, (int)layers.size(), idas[i].o,
               idas[i].up_f);
      out.insert(out.begin(), layers.back());
    }
    // ---- ida_up over out[0:3] (pose_dla_dcn.py:487-488, 533-536), last_level = 5
    std::vector<Act> y(out.begin(), out.begin() + 3);
    b.ida_up(y, "ida_up", 0, 3, 64, {1, 2, 4});
    F = y.back();

  }

  // ---- optional convGRU (convGRU.py:72-94): the three input convs see the same x at every step -> hoisted
  std::vector<Act> feat_for_head(c.num_heads, F);
  const bool gru = c.arch == CP_ARCH_DLAV1_34;
  if (gru) {
    const int steps = c.tracking_task_gru ? 4 : 3;
    const int HC = 64;
    // xi = [Wir x + b | Wiz x + b | Win x + b], hh = [Whr h | Whz h | Whn h]
    const std::string cell = "convGRU.cell0.";
    const auto [wx, bx] = b.merged_weights({cell + "Wir", cell + "Wiz", cell + "Win"}, true, F.C, 3, HC);
    const Act xi = b.conv({.src = {F}, .k = 3, .pad = 1, .Cout = 3 * HC, .w_off = wx, .b_off = bx});
    const auto [wh, bh] = b.merged_weights({cell + "Whr", cell + "Whz", cell + "Whn"}, false, HC, 3, HC);
    std::vector<Act> hs;
    Act hprev;
    for (int s = 0; s < steps; ++s) {
      Act hh;
      if (s > 0) hh = b.conv({.src = {hprev}, .k = 3, .pad = 1, .Cout = 3 * HC, .w_off = wh, .b_off = bh});
      Op op;
      op.type = OP_GRU;
      op.gx = xi;
      op.gh = hh;
      op.gprev = hprev;
      op.first_step = (s == 0);
      op.out = b.new_act(HC, F.H, F.W);
      op.name = "convGRU.gates.step" + std::to_string(s);
      P->ops.push_back(op);
      hprev = op.out;
      hs.push_back(op.out);
    }
    for (int h = 0; h < c.num_heads; ++h) {
      const std::string& n = P->head_names[h];
      int r = -1;
      if (c.tracking_task_gru) {
        if (n == "tracking" || n == "tracking_hp") r = 0;
        else if (n == "hm" || n == "wh" || n == "reg") r = 1;
        else if (n == "hm_hp" || n == "hp_offset" || n == "hps" || n == "hps_uncertainty") r = 2;
        else if (n == "scale" || n == "scale_uncertainty") r = 3;
      } else {
        if (n == "hm" || n == "wh" || n == "reg") r = 0;
        else if (n == "hm_hp" || n == "hp_offset" || n == "hps") r = 1;
        else if (n == "scale") r = 2;
      }
      if (r < 0) return fail(CP_ERR_INVALID, "head '" + n + "' has no convGRU route (pose_dla_dcn.py:545-563)");
      feat_for_head[h] = hs[r];
    }
  }

  // ---- heads: all heads that read the same feature share one 3x3 conv launch (N = n_heads * head_conv)
  const int HCV = c.head_conv;
  std::vector<bool> done(c.num_heads, false);
  for (int h0 = 0; h0 < c.num_heads; ++h0) {
    if (done[h0]) continue;
    std::vector<int> grp;
    for (int h = h0; h < c.num_heads; ++h)
      if (!done[h] && feat_for_head[h].off == feat_for_head[h0].off) grp.push_back(h);
    const Act& f = feat_for_head[h0];
    const int N = (int)grp.size() * HCV;
    std::vector<std::string> keys;
    for (int h : grp) keys.push_back(P->head_names[h] + ".0");
    const auto [wm, bm] = b.merged_weights(keys, true, f.C, 3, HCV);
    const Act mid = b.conv({.src = {f}, .k = 3, .pad = 1, .Cout = N, .relu = !gru, .w_off = wm, .b_off = bm});
    const size_t merged_idx = P->ops.size() - 1;
    std::vector<int> children;
    for (size_t gi = 0; gi < grp.size(); ++gi) {
      int h = grp[gi];
      const std::string& n = P->head_names[h];
      done[h] = true;
      Act slice = mid;
      slice.off += gi * HCV;
      slice.C = HCV;
      slice.stride = N;
      std::string last = n + ".2";
      if (gru) {
        Op g;
        g.type = OP_GN_RELU;
        g.out = slice;
        g.groups = (HCV % 32 == 0) ? 32 : 16;
        g.gamma_off = b.walloc(HCV);
        g.beta_off = b.walloc(HCV);
        PackJob j1;
        j1.type = PACK_VEC;
        j1.key = n + ".1.weight";
        j1.Cout = HCV;
        j1.dst = g.gamma_off;
        P->jobs.push_back(j1);
        PackJob j2 = j1;
        j2.key = n + ".1.bias";
        j2.dst = g.beta_off;
        P->jobs.push_back(j2);
        g.name = n + ".1(groupnorm+relu)";
        P->ops.push_back(g);
        last = n + ".3";
      }
      b.conv({.src = {slice}, .Cout = c.head_channels[h], .head = h, .wkey = last + ".weight", .bias_key = last + ".bias"});
      children.push_back((int)P->ops.size() - 1);
    }
    if (!gru) P->ops[merged_idx].head_children = children;     // GroupNorm sits between the two convs in dlav1
  }
  // plan-owned head buffers (NCHW) for cp_infer
  P->head_bufs.clear();
  for (int h = 0; h < c.num_heads; ++h) {
    Act a = b.new_act(c.head_channels[h], H / 4, W / 4);
    P->head_bufs.push_back(a);
  }
  P->act_floats = b.act_cur;
  P->w_floats = b.w_cur;
  return CP_OK;
}

// Kernel parameters of conv op `op` at `batch` frames (x every model of the plan).  ext[] may hold nulls (family
// queries); run_op rejects them.
void igemm_params(const cp_plan* P, const Op& op, int batch, const float* const ext[4], float* const* head_out,
                  IgemmParams* pp) {
  IgemmParams& p = *pp;
  p = IgemmParams{};
  p.ipm = batch;
  p.wstride = (long long)P->w_floats;
  p.tstride = (long long)P->umma_bytes;
  batch *= P->models;
  p.nsrc = op.nsrc;
  for (int i = 0; i < op.nsrc; ++i) {
    const Act& a = op.src[i];
    p.src[i] = a.ext >= 0 ? ext[a.ext] : P->act + a.off;
    if (a.ext >= 0 && ((P->ext_per_model >> a.ext) & 1u)) p.nchw_per_model |= 1u << i;
    p.srcC[i] = a.C;
    p.srcStride[i] = a.stride;
  }
  p.B = batch;
  p.Hin = op.src[0].H;
  p.Win = op.src[0].W;
  p.Cin = op.Cin;
  p.kh = op.kh;
  p.kw = op.kw;
  p.stride = op.stride;
  p.pad = op.pad;
  p.Hout = (p.Hin + 2 * op.pad - op.kh) / op.stride + 1;
  p.Wout = (p.Win + 2 * op.pad - op.kw) / op.stride + 1;
  if (op.mode == IGEMM_DECONV) {      // the 4x4/2/1 transposed conv as four 2x2-tap phase GEMMs (common.cuh)
    p.kh = p.kw = 2;
    p.stride = 1;
    p.pad = 0;
    p.Hout = 2 * p.Hin;
    p.Wout = 2 * p.Win;
  }
  p.Cout = op.Cout;
  p.CoutPad = op.CoutPad;
  p.Kpad = op.Kpad;
  p.wgt = P->wts + op.w_off;
  p.bias = P->wts + op.b_off;
  p.residual = op.has_res ? P->act + op.res.off : nullptr;
  p.resStride = op.res.stride;
  p.relu = op.relu;
  p.res_after_relu = op.res_after_relu;
  if (op.out_head >= 0) {
    p.out = head_out ? head_out[op.out_head] : nullptr;
    p.out_nchw = 1;
    p.outStride = 0;
  } else {
    p.out = P->act + op.out.off;
    p.outStride = op.out.stride;
  }
  if (op.mode == IGEMM_DCN) {
    p.offmask = P->act + op.om.off;
    p.omStride = op.om.stride;
    p.mask_is_logit = 1;
  }
  p.mode = op.mode;
  if (op.fuse_heads) {
    p.fuse_n = (int)op.head_children.size();
    p.fuse_hidden = P->cfg.head_conv;
    for (int i = 0; i < p.fuse_n; ++i) {
      const Op& ch = P->ops[op.head_children[i]];
      p.fuse_w[i] = P->wts + ch.w_off;
      p.fuse_b[i] = P->wts + ch.b_off;
      p.fuse_out[i] = head_out ? head_out[ch.out_head] : nullptr;
      p.fuse_cout[i] = ch.Cout;
    }
  }
}

// igemm_params at the plan's batch with no inputs bound: what kernel selection, tensor maps and weight tiles read
void plan_params(const cp_plan* P, const Op& op, IgemmParams* p) {
  static const float* const no_ext[4] = {};
  igemm_params(P, op, P->B, no_ext, nullptr, p);
}

// The kernel of every conv op, its weight-tile offset, and which per-head 1x1 convs run inside the epilogue of their
// merged heads conv.  Runs before the arena exists (cp_plan_memory has no device at all): the choice reads shapes,
// strides and whether a residual is added, never an address.
void select_kernels(cp_plan* P) {
  // 16-channel layers (level0 / level1): 133 K single-tile CTAs of almost no MMA work are dominated by the fixed per-CTA
  // cost of a tensor-core kernel -> keep them, and the NCHW stems, on CUDA cores
  const ConvPolicy pol{true, !P->no_dcn_tma, true, true};
  static const float residual_present = 0.f;      // a residual at arena offset 0 of a null arena would read as none
  P->umma_bytes = 0;
  for (auto& op : P->ops) {
    if (op.type != OP_IGEMM) continue;
    IgemmParams p;
    plan_params(P, op, &p);
    if (op.has_res) p.residual = &residual_present;
    op.kernel = select_conv_kernel(p, P->cfg.precision, pol);
    op.tile_off = P->umma_bytes;
    P->umma_bytes += (op.kernel.wbytes + 1023) / 1024 * 1024;
  }
  // The per-head 1x1 convs move into the epilogue of the merged heads conv when that one runs on conv_tma: hidden =
  // relu(conv3x3) never reaches HBM (3.7 GB of writes + 3.7 GB of reads and seven launches at batch 32).  In both
  // tf32 modes the two epilogue threads that own an output row multiply its hidden channels with the head's [256][16]
  // 1x1 weights (read through __ldg) and combine their halves with one shuffle (conv_tma.cu).
  const int head_conv = P->cfg.head_conv;
  for (auto& op : P->ops) {
    if (op.head_children.empty() || op.kernel.family != CP_FAM_CONV_TMA) continue;
    const int bn = op.kernel.BN;
    bool ok = op.relu && !op.has_res && (head_conv % bn == 0) && (int)op.head_children.size() <= 16 &&
              op.CoutPad == (int)op.head_children.size() * head_conv && (!op.kernel.x3 || bn == 128);
    for (int ci : op.head_children) {
      const Op& ch = P->ops[ci];
      ok = ok && ch.CoutPad == 16 && ch.w_ld == 16 && ch.Cin == head_conv && ch.out_head >= 0 && !ch.relu && !ch.has_res;
    }
    if (!ok) continue;
    op.fuse_heads = true;
    for (int ci : op.head_children) P->ops[ci].fused_away = true;
  }
  // CP_PLAN_BATCH_INVARIANT: the K segments of every launch that may split, from the layer's shape alone (fixed_ksegments:
  // the tiles of one image of one model and the channel slabs).  The default's splits are the x3 conv_tma launches
  // without the fused 1x1 and every dcn_tma launch; every other launch keeps one segment.
  for (auto& op : P->ops) {
    if (op.type != OP_IGEMM) continue;
    ConvKernel& k = op.kernel;
    k.ksegments = 0;
    if (!P->invariant) continue;
    k.ksegments = 1;
    if (op.fused_away) continue;           // runs inside its parent's epilogue
    IgemmParams p;
    plan_params(P, op, &p);
    if (k.family == CP_FAM_DCN_TMA)
      k.ksegments = fixed_ksegments(dcn_tma_image_tiles(p, k.BN), p.Cin / k.cslab);
    else if (k.family == CP_FAM_CONV_TMA && k.x3 && !op.fuse_heads)
      k.ksegments = fixed_ksegments(conv_tma_image_tiles(p, k.BN), p.Cin / k.cslab);
  }
}

// Every arena tensor op `op` reads or writes when it runs, passed to f as an Act&: none for a fused-away 1x1, the plan's
// head buffer for a head output, and no hidden tile for a fused heads conv (its children's head buffers instead).
template <class F>
void for_each_act(cp_plan* P, Op& op, F f) {
  if (op.fused_away) return;
  switch (op.type) {
    case OP_IGEMM:
      for (int s = 0; s < op.nsrc; ++s) f(op.src[s]);
      if (op.has_res) f(op.res);
      if (op.mode == IGEMM_DCN) f(op.om);
      if (op.out_head >= 0) f(P->head_bufs[op.out_head]);
      else if (!op.fuse_heads) f(op.out);
      if (op.fuse_heads)
        for (int c : op.head_children) f(P->head_bufs[P->ops[c].out_head]);
      return;
    case OP_MAXPOOL:
    case OP_MAXPOOL3:
    case OP_UPADD:
      f(op.src[0]);
      if (op.has_res) f(op.res);
      if (op.has_skip) f(op.skip);
      break;
    case OP_GN_RELU:
      break;
    case OP_GRU:
      f(op.gx);
      if (!op.first_step) {
        f(op.gh);
        f(op.gprev);
      }
      break;
  }
  f(op.out);
}

// The op range over which each arena allocation is live, then, with CP_PLAN_REUSE_ACTIVATIONS, the packed offsets.  Both
// come from one list of uses, so no view can be moved without being live or live without being moved.  The head
// buffers stay live to the end of the call: cp_infer decodes them after the last op.
void layout_arena(cp_plan* P) {
  std::vector<std::pair<int, Act*>> uses;      // (op index, view)
  const int end = (int)P->ops.size();
  for (int i = 0; i < end; ++i) for_each_act(P, P->ops[i], [&](Act& a) { uses.push_back({i, &a}); });
  for (Act& h : P->head_bufs) uses.push_back({end, &h});
  for (auto& b : P->bufs) b.first = b.last = -1;
  for (const auto& [i, a] : uses) {
    if (a->buf < 0) continue;
    ArenaAlloc& b = P->bufs[a->buf];
    if (b.first < 0) b.first = i;
    b.last = std::max(b.last, i);
  }
  if (!P->reuse) return;
  std::vector<size_t> off;
  P->act_floats = arena_pack(P->bufs, &off);
  std::set<Act*> moved;      // a head buffer is listed by the op that writes it and again at the end
  for (const auto& [i, a] : uses)
    if (a->buf >= 0 && moved.insert(a).second) a->off = a->off - P->buf_off[a->buf] + off[a->buf];
  P->buf_off = off;
}

// False for an allocation that got no memory (a reuse plan's merged heads hidden tile when the 1x1s are fused).
bool has_memory(const cp_plan* P, const Act& a) { return a.buf < 0 || !P->reuse || P->bufs[a.buf].first >= 0; }

// The tensor maps of the TMA convolutions that launch: they hold the arena addresses.
int encode_maps(cp_plan* P) {
  for (auto& op : P->ops) {
    if (op.type != OP_IGEMM || op.fused_away) continue;
    IgemmParams p;
    plan_params(P, op, &p);
    if (int rc = conv_encode(op.kernel, p, P->B * P->models, &op.maps)) return rc;
  }
  return CP_OK;
}

}  // namespace
}  // namespace cp

// ------------------------------------------------------------------------------------
extern "C" {

int cp_version(void) { return CP_ABI_VERSION; }
const char* cp_last_error(void) { return cp::g_last_error.c_str(); }

int cp_plan_create(const cp_config* cfg, cp_plan** out) { return cp_plan_create_multi(cfg, 1, out); }

static int create_plan(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_plan** out);

int cp_plan_create_multi(const cp_config* cfg, int32_t num_models, cp_plan** out) {
  if (!cfg || !out) return fail(CP_ERR_INVALID, "cp_plan_create: null argument");
  if (num_models < 1 || num_models > CP_MAX_MODELS)
    return fail(CP_ERR_INVALID, "cp_plan_create_multi: num_models must be in 1..CP_MAX_MODELS");
  if (cfg->tracking && num_models > 1)
    return fail(CP_ERR_INVALID, "cp_plan_create_multi: a tracking plan made here holds one model; several tracking "
                                "models run through cp_plan_create_multi_track");
  return create_plan(cfg, num_models, 0u, out);
}

int cp_plan_create_multi_track(const cp_config* cfg, int32_t num_models, cp_plan** out) {
  if (!cfg || !out) return fail(CP_ERR_INVALID, "cp_plan_create_multi_track: null argument");
  if (cfg->tracking != 1) return fail(CP_ERR_INVALID, "cp_plan_create_multi_track: needs a tracking config (tracking = 1)");
  if (num_models < 1 || num_models > CP_MAX_MODELS)
    return fail(CP_ERR_INVALID, "cp_plan_create_multi_track: num_models must be in 1..CP_MAX_MODELS");
  return create_plan(cfg, num_models, CP_PLAN_MULTI_TRACK, out);
}

// the arguments cp_plan_create_ex and cp_plan_memory share (the config itself is checked by plan_layout)
static int check_ex_args(const cp_config* cfg, int32_t num_models, uint32_t flags, const char* fn) {
  const std::string f(fn);
  if (!cfg) return fail(CP_ERR_INVALID, f + ": null argument");
  if (flags & ~(uint32_t)(CP_PLAN_REUSE_ACTIVATIONS | CP_PLAN_MULTI_TRACK | CP_PLAN_BATCH_INVARIANT))
    return fail(CP_ERR_INVALID, f + ": unknown flags");
  if (num_models < 1 || num_models > CP_MAX_MODELS) return fail(CP_ERR_INVALID, f + ": num_models must be in 1..CP_MAX_MODELS");
  if ((flags & CP_PLAN_MULTI_TRACK) && cfg->tracking != 1)
    return fail(CP_ERR_INVALID, f + ": CP_PLAN_MULTI_TRACK needs a tracking config (tracking = 1)");
  if (cfg->tracking && num_models > 1 && !(flags & CP_PLAN_MULTI_TRACK))
    return fail(CP_ERR_INVALID, f + ": several tracking models need CP_PLAN_MULTI_TRACK");
  return CP_OK;
}

int cp_plan_create_ex(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_plan** out) {
  if (!out) return fail(CP_ERR_INVALID, "cp_plan_create_ex: null argument");
  if (int rc = check_ex_args(cfg, num_models, flags, "cp_plan_create_ex")) return rc;
  return create_plan(cfg, num_models, flags, out);
}

// Everything about a plan that needs no device: the checked config, the schedule, the kernel of every op, the weight
// and tile sizes and the arena layout.
static int plan_layout(cp_plan* P, const cp_config* cfg, int32_t num_models, uint32_t flags) {
  if (cfg->arch != CP_ARCH_DLA34 && cfg->arch != CP_ARCH_DLAV1_34 && !is_res_arch(cfg->arch))
    return fail(CP_ERR_INVALID, "cp_plan_create: unknown arch");
  if (is_res_arch(cfg->arch) && cfg->tracking_task_gru)
    return fail(CP_ERR_INVALID, "cp_plan_create: tracking_task_gru needs the dlav1 convGRU; ResNets have none");
  if (!known_precision(cfg->precision))
    return fail(CP_ERR_INVALID, "cp_plan_create: unknown precision");
  if (cfg->height % 32 || cfg->width % 32 || cfg->height <= 0 || cfg->width <= 0)
    return fail(CP_ERR_INVALID, "cp_plan_create: height/width must be positive multiples of 32");
  if (cfg->max_batch <= 0 || cfg->num_heads <= 0 || cfg->num_heads > CP_MAX_HEADS)
    return fail(CP_ERR_INVALID, "cp_plan_create: bad batch / head count");
  if (cfg->head_conv <= 0 || cfg->head_conv % 64)
    return fail(CP_ERR_INVALID, "cp_plan_create: head_conv must be a positive multiple of 64");
  if (cfg->arch == CP_ARCH_DLAV1_34 && cfg->head_conv != 256)
    return fail(CP_ERR_INVALID, "cp_plan_create: dlav1 GroupNorm path needs head_conv == 256");
  P->cfg = *cfg;
  for (int i = 0; i < cfg->num_heads; ++i) {
    if (!cfg->head_names[i] || cfg->head_channels[i] <= 0 || cfg->head_channels[i] > 16)
      return fail(CP_ERR_INVALID, "cp_plan_create: head channels must be in 1..16");
    P->head_names.push_back(cfg->head_names[i]);
  }
  for (int i = 0; i < cfg->num_heads; ++i) P->cfg.head_names[i] = P->head_names[i].c_str();
  P->B = cfg->max_batch;
  P->models = num_models;
  P->ext_per_model = (flags & CP_PLAN_MULTI_TRACK) ? kMultiTrackInputs : 0u;
  P->reuse = (flags & CP_PLAN_REUSE_ACTIVATIONS) != 0;
  P->invariant = (flags & CP_PLAN_BATCH_INVARIANT) != 0;
  P->model_loaded.assign(num_models, 0);
  P->H = cfg->height;
  P->W = cfg->width;
  if (const char* e = getenv("CP_NO_DCN_TMA")) P->no_dcn_tma = atoi(e) != 0;
  if (int rc = build_graph(P)) return rc;
  select_kernels(P);
  layout_arena(P);
  return CP_OK;
}

static void plan_memory(const cp_plan* P, cp_memory_info* m) {
  const bool splitk = P->cfg.precision == CP_PREC_TF32X3 || P->cfg.precision == CP_PREC_TF32;
  m->activation_bytes = (int64_t)(P->act_floats * sizeof(float));
  m->weight_bytes = (int64_t)(P->w_floats * P->models * sizeof(float));
  m->tile_bytes = (int64_t)(P->umma_bytes * P->models);
  m->workspace_bytes = (int64_t)(sizeof(double) * gn_workspace_doubles(P->B * P->models) +
                                 (splitk ? kSplitkWsFloats * sizeof(float) : 0));
}

static int create_plan(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_plan** out) {
  std::unique_ptr<cp_plan> P(new cp_plan());
  if (int rc = plan_layout(P.get(), cfg, num_models, flags)) return rc;
  // the plan lives on cfg->device; the caller's current device is restored on every exit path
  struct DeviceGuard {
    int prev = -1;
    ~DeviceGuard() {
      if (prev >= 0) cudaSetDevice(prev);
    }
  } guard;
  CP_CUDA_CHECK(cudaGetDevice(&guard.prev));
  CP_CUDA_CHECK(cudaSetDevice(cfg->device));
  CP_CUDA_CHECK(cudaMalloc(&P->act, P->act_floats * sizeof(float)));
  CP_CUDA_CHECK(cudaMalloc(&P->wts, P->w_floats * num_models * sizeof(float)));
  CP_CUDA_CHECK(cudaMemset(P->wts, 0, P->w_floats * num_models * sizeof(float)));
  CP_CUDA_CHECK(cudaMalloc(&P->gn_stats, sizeof(double) * gn_workspace_doubles(P->B * num_models)));
  if (int rc = encode_maps(P.get())) return rc;
  if (P->umma_bytes) CP_CUDA_CHECK(cudaMalloc(&P->umma_wts, P->umma_bytes * num_models));
  if (cfg->precision == CP_PREC_TF32X3 || cfg->precision == CP_PREC_TF32) {
    CP_CUDA_CHECK(cudaMalloc(&P->splitk_ws, kSplitkWsFloats * sizeof(float)));
  }
  int n = 0;
  for (auto& op : P->ops) n += op.fused_away ? 0 : ((op.type == OP_GN_RELU) ? 3 : 1);
  P->launches = n;
  *out = P.release();
  return CP_OK;
}

int cp_plan_memory(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_memory_info* out) {
  if (!out) return fail(CP_ERR_INVALID, "cp_plan_memory: null argument");
  if (int rc = check_ex_args(cfg, num_models, flags, "cp_plan_memory")) return rc;
  cp_plan P;      // host side only: nothing is allocated on a device
  if (int rc = plan_layout(&P, cfg, num_models, flags)) return rc;
  plan_memory(&P, out);
  return CP_OK;
}

int cp_plan_allocations(const cp_config* cfg, int32_t num_models, uint32_t flags, cp_act_alloc* out, int32_t max_allocs,
                        int32_t* n_allocs) {
  if (!out || !n_allocs) return fail(CP_ERR_INVALID, "cp_plan_allocations: null argument");
  if (int rc = check_ex_args(cfg, num_models, flags, "cp_plan_allocations")) return rc;
  cp_plan P;
  if (int rc = plan_layout(&P, cfg, num_models, flags)) return rc;
  const int n = (int)std::min(P.bufs.size(), (size_t)std::max(max_allocs, 0));
  for (int i = 0; i < n; ++i) {
    const ArenaAlloc& b = P.bufs[i];
    const bool mem = !P.reuse || b.first >= 0;
    out[i].floats = mem ? (int64_t)b.floats : 0;
    out[i].off = mem ? (int64_t)P.buf_off[i] : -1;
    out[i].first = b.first;
    out[i].last = b.last;
  }
  *n_allocs = (int32_t)P.bufs.size();
  return CP_OK;
}

int cp_plan_ksegments(const cp_config* cfg, int32_t num_models, uint32_t flags, int32_t* segments, int32_t max_ops,
                      int32_t* n_ops) {
  if (!segments || !n_ops) return fail(CP_ERR_INVALID, "cp_plan_ksegments: null argument");
  if (int rc = check_ex_args(cfg, num_models, flags, "cp_plan_ksegments")) return rc;
  cp_plan P;
  if (int rc = plan_layout(&P, cfg, num_models, flags)) return rc;
  const int n = (int)std::min(P.ops.size(), (size_t)std::max(max_ops, 0));
  for (int i = 0; i < n; ++i) segments[i] = P.ops[i].type == OP_IGEMM ? P.ops[i].kernel.ksegments : (P.invariant ? 1 : 0);
  *n_ops = (int32_t)P.ops.size();
  return CP_OK;
}

int cp_plan_op_ksegments(const cp_plan* P, int32_t i, int32_t* segments, int32_t* last_segments, int32_t* last_path) {
  if (!P || !segments) return fail(CP_ERR_INVALID, "cp_plan_op_ksegments: null argument");
  if (i < 0 || i >= (int)P->ops.size()) return fail(CP_ERR_INVALID, "cp_plan_op_ksegments: op index out of range");
  const Op& op = P->ops[i];
  *segments = op.type == OP_IGEMM ? op.kernel.ksegments : (P->invariant ? 1 : 0);
  if (last_segments) *last_segments = op.last_ksplit;
  if (last_path) *last_path = op.last_path;
  return CP_OK;
}

int cp_plan_destroy(cp_plan* P) {
  if (!P) return CP_OK;
  cudaFree(P->act);
  cudaFree(P->wts);
  cudaFree(P->gn_stats);
  if (P->umma_wts) cudaFree(P->umma_wts);
  if (P->splitk_ws) cudaFree(P->splitk_ws);
  if (P->decode_ws) cudaFree(P->decode_ws);
  delete P;
  return CP_OK;
}

int64_t cp_plan_bytes(const cp_plan* P) {
  return P ? (int64_t)((P->act_floats + P->w_floats * P->models) * sizeof(float)) : 0;
}
int32_t cp_plan_num_models(const cp_plan* P) { return P ? P->models : 0; }
int32_t cp_plan_forward_launches(const cp_plan* P) { return P ? P->launches : 0; }

int cp_plan_load_weights(cp_plan* P, const char* const* names, const void* const* ptrs, const int64_t* numel,
                         int32_t n, void* stream_) {
  return cp_plan_load_weights_model(P, 0, names, ptrs, numel, n, stream_);
}

int cp_plan_load_weights_model(cp_plan* P, int32_t model, const char* const* names, const void* const* ptrs,
                               const int64_t* numel, int32_t n, void* stream_) {
  if (!P || !names || !ptrs || !numel) return fail(CP_ERR_INVALID, "cp_plan_load_weights: null argument");
  if (model < 0 || model >= P->models) return fail(CP_ERR_INVALID, "cp_plan_load_weights_model: model index out of range");
  cudaStream_t s = (cudaStream_t)stream_;
  float* const wts = P->wts + (size_t)model * P->w_floats;      // this model's copy of the weight storage
  std::map<std::string, WRef> m;
  for (int i = 0; i < n; ++i) {
    std::string k = names[i];
    if (k.rfind("module.", 0) == 0 && k.rfind("module_list", 0) != 0) k = k.substr(7);
    m[k] = WRef{(const float*)ptrs[i], numel[i]};
  }
  auto get = [&](const std::string& k, int64_t want, const float** out) -> int {
    auto it = m.find(k);
    if (it == m.end()) return fail(CP_ERR_MISSING_KEY, "state_dict key missing: " + k);
    if (it->second.n != want)
      return fail(CP_ERR_SHAPE, "state_dict key " + k + " has " + std::to_string(it->second.n) + " elements, plan needs " +
                                    std::to_string(want));
    *out = it->second.p;
    return CP_OK;
  };
  int rc;
  for (auto& j : P->jobs) {
    switch (j.type) {
      case PACK_BIAS: {
        const float *cb = nullptr, *g = nullptr, *be = nullptr, *mu = nullptr, *var = nullptr;
        if (!j.key.empty() && (rc = get(j.key, j.Cout, &cb))) return rc;
        if (!j.bn.empty()) {
          if ((rc = get(j.bn + ".weight", j.Cout, &g))) return rc;
          if ((rc = get(j.bn + ".bias", j.Cout, &be))) return rc;
          if ((rc = get(j.bn + ".running_mean", j.Cout, &mu))) return rc;
          if ((rc = get(j.bn + ".running_var", j.Cout, &var))) return rc;
        }
        if ((rc = launch_pack_bias(cb, g, be, mu, var, wts + j.scale, wts + j.dst, j.Cout, j.CoutPad, 1e-5f, s)))
          return rc;
        break;
      }
      case PACK_CONV: {
        const float* w = nullptr;
        if ((rc = get(j.key, (int64_t)j.Cout * j.Cin * j.kh * j.kw, &w))) return rc;
        if ((rc = launch_pack_conv_weight(w, j.use_scale ? wts + j.scale : nullptr, wts + j.dst, j.Cout, j.Cin,
                                          j.kh, j.kw, j.CoutPad, j.Kpad, j.ld, j.colOff, s)))
          return rc;
        break;
      }
      case PACK_UP: {
        const float* w = nullptr;
        if ((rc = get(j.key, (int64_t)j.Cout * j.kh * j.kh, &w))) return rc;
        if ((rc = launch_pack_up_weight(w, wts + j.dst, j.Cout, j.kh, s))) return rc;
        break;
      }
      case PACK_DECONV: {
        const float* w = nullptr;
        if ((rc = get(j.key, (int64_t)j.Cin * j.Cout * 16, &w))) return rc;
        if ((rc = launch_pack_deconv_weight(w, wts + j.scale, wts + j.dst, j.Cin, j.Cout, j.CoutPad, j.Kpad, s))) return rc;
        break;
      }
      case PACK_VEC: {
        const float* w = nullptr;
        if ((rc = get(j.key, j.Cout, &w))) return rc;
        CP_CUDA_CHECK(cudaMemcpyAsync(wts + j.dst, w, sizeof(float) * j.Cout, cudaMemcpyDeviceToDevice, s));
        break;
      }
    }
  }
  // second pass: tensor-core weight tiles are cut from the finished fp32 matrices (merged matrices are complete now)
  for (auto& op : P->ops) {
    if (op.type != OP_IGEMM || !op.kernel.wbytes) continue;
    IgemmParams p;
    plan_params(P, op, &p);
    p.wgt += (size_t)model * P->w_floats;
    if ((rc = conv_pack(op.kernel, p, op.w_ld, P->umma_wts + (size_t)model * P->umma_bytes + op.tile_off, s))) return rc;
  }
  P->model_loaded[model] = 1;
  P->loaded = true;
  for (char l : P->model_loaded) P->loaded = P->loaded && l;
  return CP_OK;
}

struct ProfCtx {
  std::vector<cudaEvent_t> ev;
};

// PDL hides launch latency + prologue per kernel, which matters when the kernels are short (small batches); once they
// run for 100s of us the early CTAs of the next launch only add scheduling work, so it is switched on by the amount of
// work.  The threshold below has not been re-chosen for the H100 (scripts/pdl_sweep.py sweeps it); results are
// bit-identical either way.  CP_PDL=1 / CP_NO_PDL=1 force it.
static bool pdl_wanted(long long pixels) {
  if (getenv("CP_NO_PDL")) return false;
  if (const char* e = getenv("CP_PDL")) return atoi(e) != 0;
  return pixels <= 8ll * 512 * 512;
}

// One op of the schedule, as cp_forward runs it.  `info` (may be null) receives what the launcher decided.
static int run_op(cp_plan* P, size_t idx, int batch, const float* const ext[4], float* const* head_out, cudaStream_t s,
                  cp_op_launch* info) {
  int rc;
  const Op& op = P->ops[idx];
  const int images = batch * P->models;       // every model's images go through one launch
  const long long wstride = (long long)P->w_floats;
  cp_op_launch li{};
  li.ksplit = 1;
  if (op.fused_away) {          // computed inside the epilogue of the merged heads conv
    if (info) *info = li;
    return CP_OK;
  }
  switch (op.type) {
    case OP_IGEMM: {
      for (int i = 0; i < op.nsrc; ++i)
        if (op.src[i].ext >= 0 && !ext[op.src[i].ext]) return fail(CP_ERR_INVALID, "cp_forward: a tracking input tensor is null");
      IgemmParams p;
      igemm_params(P, op, batch, ext, head_out, &p);
      p.wgt_umma = P->umma_wts + op.tile_off;
      p.splitk_ws = P->splitk_ws;
      p.splitk_ws_floats = P->splitk_ws ? kSplitkWsFloats : 0;
      LaunchInfo tc;
      li.family = op.kernel.family;
      if ((rc = conv_launch(op.kernel, p, &op.maps, s, &tc))) return rc;
      li.BN = tc.BN;
      li.ksplit = tc.ksplit;
      li.grid = (int32_t)tc.grid;
      P->ops[idx].last_ksplit = tc.ksplit;
      P->ops[idx].last_path = tc.path;
      break;
    }
    case OP_MAXPOOL:
      li.family = CP_FAM_MAXPOOL;
      if ((rc = launch_maxpool2(P->act + op.src[0].off, P->act + op.out.off, images, op.src[0].H, op.src[0].W,
                                op.src[0].C, s)))
        return rc;
      break;
    case OP_MAXPOOL3:
      li.family = CP_FAM_MAXPOOL;
      if ((rc = launch_maxpool3s2(P->act + op.src[0].off, op.has_res ? P->act + op.res.off : nullptr, P->act + op.out.off,
                                  images, op.src[0].H, op.src[0].W, op.src[0].C, s)))
        return rc;
      break;
    case OP_UPADD:
      li.family = CP_FAM_UPADD;
      if ((rc = launch_upsample_add(P->act + op.src[0].off, P->wts + op.upw_off,
                                    op.has_skip ? P->act + op.skip.off : nullptr, P->act + op.out.off, images,
                                    op.src[0].H, op.src[0].W, op.src[0].C, op.f, s, batch, wstride)))
        return rc;
      break;
    case OP_GN_RELU:
      li.family = CP_FAM_GN_RELU;
      if ((rc = launch_group_norm_relu(P->act + op.out.off, P->wts + op.gamma_off, P->wts + op.beta_off, images,
                                       op.out.H * op.out.W, op.out.C, op.out.stride, 0, op.groups, 1e-5f,
                                       P->gn_stats, s, batch, wstride)))
        return rc;
      break;
    case OP_GRU:
      li.family = CP_FAM_GRU;
      if ((rc = launch_gru_gates(P->act + op.gx.off, op.first_step ? nullptr : P->act + op.gh.off,
                                 op.first_step ? nullptr : P->act + op.gprev.off, P->act + op.out.off,
                                 images * op.out.H * op.out.W, op.out.C, op.first_step, s)))
        return rc;
      break;
  }
  if (info) *info = li;
  return CP_OK;
}

static int run_forward(cp_plan* P, int batch, const float* const ext[4], float* const* head_out, cudaStream_t s,
                       ProfCtx* prof = nullptr) {
  int rc;
  const long long launches0 = g_launch_counter;
  // programmatic dependent launch for the whole schedule (common.cuh); off while profiling (events sit between the ops)
  struct PdlScope {
    explicit PdlScope(int on) { g_pdl = on; }
    ~PdlScope() { g_pdl = 0; }
  } pdl_scope(!prof && pdl_wanted((long long)batch * P->models * P->H * P->W));
  for (size_t i = 0; i < P->ops.size(); ++i) {
    if (prof) {
      cudaEvent_t e;
      CP_CUDA_CHECK(cudaEventCreate(&e));
      CP_CUDA_CHECK(cudaEventRecord(e, s));
      prof->ev.push_back(e);
    }
    if ((rc = run_op(P, i, batch, ext, head_out, s, nullptr))) return rc;
  }
  if (prof) {
    cudaEvent_t e;
    CP_CUDA_CHECK(cudaEventCreate(&e));
    CP_CUDA_CHECK(cudaEventRecord(e, s));
    prof->ev.push_back(e);
  }
  P->launches = (int)(g_launch_counter - launches0);      // measured, replaces the estimate of cp_plan_create
  return CP_OK;
}

// cp_op_stat.kind / cp_op_desc.kind: op type * 10 + igemm mode; the 3x3/2 max-pool is 11 (10 is the 2x2 DLA pool)
static int op_kind(const Op& op) {
  if (op.type == OP_MAXPOOL3) return 11;
  return (int)op.type * 10 + (op.type == OP_IGEMM ? op.mode : 0);
}

// Algorithmic work of one op at batch `batch` (2*MAC; fp32 bytes of the tensors it must touch once).
static void op_work(const Op& op, int batch, double* flops, double* bytes) {
  *flops = 0;
  *bytes = 0;
  const double B = batch;
  switch (op.type) {
    case OP_IGEMM: {
      int Hin = op.src[0].H, Win = op.src[0].W;
      int Ho = (Hin + 2 * op.pad - op.kh) / op.stride + 1, Wo = (Win + 2 * op.pad - op.kw) / op.stride + 1;
      double M = B * Ho * Wo;
      *flops = 2.0 * M * op.kh * op.kw * op.Cin * op.Cout;
      if (op.mode == IGEMM_DECONV) {      // 16 taps per input pixel: 4 per output pixel
        M = B * op.out.H * op.out.W;
        *flops = 2.0 * M * 4 * op.Cin * op.Cout;
      }
      *bytes = 4.0 * (B * Hin * Win * op.Cin + (double)op.kh * op.kw * op.Cin * op.Cout + (op.fuse_heads ? 0.0 : M * op.Cout) +
                      (op.has_res ? M * op.Cout : 0.0) + (op.mode == IGEMM_DCN ? M * 27 : 0.0));
      if (op.fused_away) {      // accounted to the parent below
        *flops = 0;
        *bytes = 0;
      }
      break;
    }
    case OP_MAXPOOL:
      *bytes = 4.0 * B * op.src[0].H * op.src[0].W * op.src[0].C * 1.25;
      break;
    case OP_MAXPOOL3:
      *bytes = 4.0 * B * op.src[0].H * op.src[0].W * op.src[0].C * (op.has_res ? 1.5 : 1.25);
      break;
    case OP_UPADD: {
      double o = B * op.out.H * op.out.W * op.out.C;
      *flops = 2.0 * o * 4;
      *bytes = 4.0 * (o * 2 + B * op.src[0].H * op.src[0].W * op.src[0].C);
      break;
    }
    case OP_GN_RELU:
      *bytes = 4.0 * B * op.out.H * op.out.W * op.out.C * 3;
      break;
    case OP_GRU:
      *bytes = 4.0 * B * op.out.H * op.out.W * op.out.C * 8;
      break;
  }
}

// The checks every call that runs the schedule starts with: `given` is false when a pointer `fn` needs is null, `load`
// names the call that loads the weights.
static int check_run(const cp_plan* P, bool given, int32_t batch, const char* fn, const char* load = "cp_plan_load_weights") {
  if (!P || !given) return fail(CP_ERR_INVALID, std::string(fn) + ": null argument");
  if (!P->loaded) return fail(CP_ERR_NOT_LOADED, std::string(fn) + ": call " + load + " first");
  if (batch <= 0 || batch > P->B) return fail(CP_ERR_INVALID, std::string(fn) + ": batch exceeds the plan's max_batch");
  return CP_OK;
}
static const char* const kLoadEveryModel = "cp_plan_load_weights_model for every model";

int cp_forward(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
               const float* pre_hm_hp, float* const* head_out, void* stream) {
  if (int rc = check_run(P, images && head_out, batch, "cp_forward")) return rc;
  const float* ext[4] = {images, pre_img, pre_hm, pre_hm_hp};
  return run_forward(P, batch, ext, head_out, (cudaStream_t)stream);
}

int cp_plan_num_ops(const cp_plan* P) { return P ? (int)P->ops.size() : 0; }

int cp_plan_profile(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
                    const float* pre_hm_hp, float* const* head_out, void* stream, cp_op_stat* stats, int32_t max_stats,
                    int32_t* n_stats) {
  if (int rc = check_run(P, images && head_out && stats && n_stats, batch, "cp_plan_profile")) return rc;
  const float* ext[4] = {images, pre_img, pre_hm, pre_hm_hp};
  ProfCtx ctx;
  int rc = run_forward(P, batch, ext, head_out, (cudaStream_t)stream, &ctx);
  if (rc == CP_OK) {
    CP_CUDA_CHECK(cudaEventSynchronize(ctx.ev.back()));
    int n = 0;
    for (size_t i = 0; i + 1 < ctx.ev.size() && n < max_stats; ++i, ++n) {
      const Op& op = P->ops[i];
      cp_op_stat& st = stats[n];
      memset(&st, 0, sizeof(st));
      snprintf(st.name, sizeof(st.name), "%s", op.name.c_str());
      st.kind = op_kind(op);
      cudaEventElapsedTime(&st.ms, ctx.ev[i], ctx.ev[i + 1]);
      op_work(op, batch * P->models, &st.flops, &st.bytes);
    }
    *n_stats = n;
  }
  for (auto e : ctx.ev) cudaEventDestroy(e);
  return rc;
}

// `first`: the arena offset of the image the description starts at (model m of a multi-model plan: m * max_batch)
static void act_desc(const Act& a, cp_act_desc* d, size_t first = 0) {
  d->off = a.ext >= 0 || a.C == 0 ? -1 : (int64_t)(a.off + first * a.H * a.W * a.stride);
  d->ext = a.ext;
  d->C = a.C;
  d->H = a.H;
  d->W = a.W;
  d->stride = a.stride;
}

int cp_plan_op_desc(const cp_plan* P, int32_t i, cp_op_desc* d) { return cp_plan_op_desc_model(P, 0, i, d); }

int cp_plan_op_desc_model(const cp_plan* P, int32_t model, int32_t i, cp_op_desc* d) {
  if (!P || !d) return fail(CP_ERR_INVALID, "cp_plan_op_desc: null argument");
  if (model < 0 || model >= P->models) return fail(CP_ERR_INVALID, "cp_plan_op_desc_model: model index out of range");
  if (i < 0 || i >= (int)P->ops.size()) return fail(CP_ERR_INVALID, "cp_plan_op_desc: op index out of range");
  const Op& op = P->ops[i];
  const float* const wts = P->wts + (size_t)model * P->w_floats;
  const size_t first = (size_t)model * P->B;
  auto act_desc = [P, first](const Act& a, cp_act_desc* ad) {
    ::act_desc(a, ad, first);
    if (!has_memory(P, a)) ad->off = -1;
  };
  memset(d, 0, sizeof(*d));
  snprintf(d->name, sizeof(d->name), "%s", op.name.c_str());
  d->kind = op_kind(op);
  d->nsrc = op.nsrc;
  for (int k = 0; k < 4; ++k) act_desc(op.src[k], &d->src[k]);
  if (op.type != OP_IGEMM) act_desc(op.src[0], &d->src[0]);
  act_desc(op.out, &d->out);
  d->out_head = op.out_head;
  if (op.out_head >= 0) d->out.off = -1;
  d->kh = op.kh;
  d->stride = op.stride;
  d->pad = op.pad;
  d->Cin = op.Cin;
  d->Cout = op.Cout;
  d->CoutPad = op.CoutPad;
  d->Kpad = op.Kpad;
  d->relu = op.relu;
  d->has_res = op.has_res;
  d->res_after_relu = op.res_after_relu;
  act_desc(op.res, &d->res);
  act_desc(op.om, &d->om);
  act_desc(op.skip, &d->skip);
  act_desc(op.gx, &d->gx);
  act_desc(op.gh, &d->gh);
  act_desc(op.gprev, &d->gprev);
  d->parent = -1;
  switch (op.type) {
    case OP_IGEMM: {
      d->w = wts + op.w_off;
      d->w_ld = op.w_ld;
      d->bias = wts + op.b_off;
      d->family = op.kernel.family;
      d->x3 = op.kernel.x3;
      break;
    }
    case OP_MAXPOOL: d->family = CP_FAM_MAXPOOL; break;
    case OP_MAXPOOL3: d->family = CP_FAM_MAXPOOL; break;
    case OP_UPADD:
      d->family = CP_FAM_UPADD;
      d->up_w = wts + op.upw_off;
      d->f = op.f;
      d->has_skip = op.has_skip;
      break;
    case OP_GN_RELU:
      d->family = CP_FAM_GN_RELU;
      d->gamma = wts + op.gamma_off;
      d->beta = wts + op.beta_off;
      d->groups = op.groups;
      break;
    case OP_GRU:
      d->family = CP_FAM_GRU;
      d->first_step = op.first_step;
      break;
  }
  d->fuse_heads = op.fuse_heads;
  d->fused_away = op.fused_away;
  d->n_children = (int)op.head_children.size();
  for (int k = 0; k < d->n_children && k < CP_MAX_HEADS; ++k) d->children[k] = op.head_children[k];
  if (op.fused_away) {
    d->family = CP_FAM_NONE;
    for (int j = 0; j < (int)P->ops.size(); ++j)
      for (int c : P->ops[j].head_children)
        if (c == i) d->parent = j;
  }
  return CP_OK;
}

int cp_plan_arena(const cp_plan* P, float** act, int64_t* floats) {
  if (!P || !act || !floats) return fail(CP_ERR_INVALID, "cp_plan_arena: null argument");
  *act = P->act;
  *floats = (int64_t)P->act_floats;
  return CP_OK;
}

int cp_plan_run_ops(cp_plan* P, int32_t batch, int32_t first, int32_t last, const float* images, const float* pre_img,
                    const float* pre_hm, const float* pre_hm_hp, float* const* head_out, void* stream,
                    cp_op_launch* info) {
  if (int rc = check_run(P, images && head_out, batch, "cp_plan_run_ops")) return rc;
  if (first < 0 || last < first || last > (int)P->ops.size())
    return fail(CP_ERR_INVALID, "cp_plan_run_ops: op range outside the schedule");
  const float* ext[4] = {images, pre_img, pre_hm, pre_hm_hp};
  g_pdl = 0;
  for (int32_t i = first; i < last; ++i) {
    int rc = run_op(P, (size_t)i, batch, ext, head_out, (cudaStream_t)stream, info ? info + (i - first) : nullptr);
    if (rc) return rc;
  }
  return CP_OK;
}

static int infer_models(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
                        const float* pre_hm_hp, const cp_decode_params* prm, const double* meta, float* const* heads_out,
                        float* dets, float* poses, int32_t* n_valid, void* stream);

int cp_infer(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
             const float* pre_hm_hp, const cp_decode_params* prm, const double* meta, float* const* heads_out,
             float* dets, float* poses, int32_t* n_valid, void* stream) {
  if (int rc = check_run(P, images && prm && meta && poses && n_valid, batch, "cp_infer")) return rc;
  if (P->models > 1)
    return fail(CP_ERR_INVALID, P->cfg.tracking ? "cp_infer: a multi-model tracking plan runs through cp_infer_multi_track"
                                                : "cp_infer: a multi-model plan runs through cp_infer_multi");
  return infer_models(P, batch, images, pre_img, pre_hm, pre_hm_hp, prm, meta, heads_out, dets, poses, n_valid, stream);
}

// the decode parameters of a multi-model call: the models may differ in their per-category constants only
static int check_model_prms(const cp_plan* P, const cp_decode_params* prms, const char* fn) {
  for (int m = 1; m < P->models; ++m) {
    cp_decode_params a = prms[0], b = prms[m];
    a.visible_thresh = b.visible_thresh = 0;      // the per-category constants (cuboid_pnp_shell.py:59-66, balance)
    a.balance = b.balance = 0.f;
    a.batch = b.batch = a.out_h = b.out_h = a.out_w = b.out_w = 0;      // set by the call
    if (memcmp(&a, &b, sizeof(a)))
      return fail(CP_ERR_INVALID, std::string(fn) + ": the models' decode parameters may differ in visible_thresh and balance only");
  }
  return CP_OK;
}

int cp_infer_multi(cp_plan* P, int32_t batch, const float* images, const cp_decode_params* prms, const double* meta,
                   float* const* heads_out, float* dets, float* poses, int32_t* n_valid, void* stream) {
  if (int rc = check_run(P, images && prms && meta && poses && n_valid, batch, "cp_infer_multi", kLoadEveryModel))
    return rc;
  if (P->cfg.tracking)
    return fail(CP_ERR_INVALID, "cp_infer_multi: tracking plans run through cp_infer or cp_infer_multi_track");
  if (int rc = check_model_prms(P, prms, "cp_infer_multi")) return rc;
  return infer_models(P, batch, images, nullptr, nullptr, nullptr, prms, meta, heads_out, dets, poses, n_valid, stream);
}

int cp_infer_multi_track(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
                         const float* pre_hm_hp, const cp_decode_params* prms, const double* meta, float* const* heads_out,
                         float* dets, float* poses, int32_t* n_valid, void* stream) {
  const bool given = images && pre_img && pre_hm && pre_hm_hp && prms && meta && poses && n_valid;
  if (P && given && (!P->cfg.tracking || P->ext_per_model != kMultiTrackInputs))
    return fail(CP_ERR_INVALID, "cp_infer_multi_track: the plan was not made by cp_plan_create_multi_track");
  if (int rc = check_run(P, given, batch, "cp_infer_multi_track", kLoadEveryModel)) return rc;
  if (int rc = check_model_prms(P, prms, "cp_infer_multi_track")) return rc;
  return infer_models(P, batch, images, pre_img, pre_hm, pre_hm_hp, prms, meta, heads_out, dets, poses, n_valid, stream);
}

}  // extern "C"

// forward + one decode over every model's heads; prm[0 .. P->models)
static int infer_models(cp_plan* P, int32_t batch, const float* images, const float* pre_img, const float* pre_hm,
                        const float* pre_hm_hp, const cp_decode_params* prm, const double* meta, float* const* heads_out,
                        float* dets, float* poses, int32_t* n_valid, void* stream) {
  float* hp[CP_MAX_HEADS];
  for (int h = 0; h < P->cfg.num_heads; ++h)
    hp[h] = (heads_out && heads_out[h]) ? heads_out[h] : P->act + P->head_bufs[h].off;
  const float* ext[4] = {images, pre_img, pre_hm, pre_hm_hp};
  int rc = run_forward(P, batch, ext, hp, (cudaStream_t)stream);
  if (rc) return rc;
  cp_heads hd{};
  for (int h = 0; h < P->cfg.num_heads; ++h) {
    const std::string& n = P->head_names[h];
    if (n == "hm" && P->cfg.head_channels[h] != prm->num_classes)
      return fail(CP_ERR_INVALID, "cp_infer: prm->num_classes differs from the plan's hm channels");
    if (n == "hm") hd.hm = hp[h];
    else if (n == "wh") hd.wh = hp[h];
    else if (n == "hps") hd.hps = hp[h];
    else if (n == "reg") hd.reg = hp[h];
    else if (n == "hm_hp") hd.hm_hp = hp[h];
    else if (n == "hp_offset") hd.hp_offset = hp[h];
    else if (n == "scale") hd.scale = hp[h];
    else if (n == "hps_uncertainty") hd.hps_uncertainty = hp[h];
    else if (n == "scale_uncertainty") hd.scale_uncertainty = hp[h];
    else if (n == "tracking") hd.tracking = hp[h];
    else if (n == "tracking_hp") hd.tracking_hp = hp[h];
  }
  std::vector<cp_decode_params> qs(prm, prm + P->models);
  cp_decode_params& q = qs[0];
  q.batch = batch * P->models;
  q.out_h = P->H / 4;
  q.out_w = P->W / 4;
  q.apply_sigmoid = prm->apply_sigmoid == 2 ? 2 : 1;     // the plan's heads are logits; 2 = opt.mse_loss (raw hm_hp)
  size_t need = cp_decode_workspace_bytes(&q);
  if (need > P->decode_ws_bytes) {
    // grows only on the first call for a given K / batch (not steady state)
    if (P->decode_ws) cudaFree(P->decode_ws);
    cp_decode_params qmax = q;
    qmax.batch = P->B * P->models;
    size_t cap = cp_decode_workspace_bytes(&qmax);
    CP_CUDA_CHECK(cudaMalloc(&P->decode_ws, cap));
    P->decode_ws_bytes = cap;
  }
  return decode_pnp_models(qs.data(), P->models, &hd, meta, dets, poses, n_valid, P->decode_ws, P->decode_ws_bytes,
                           stream);
}

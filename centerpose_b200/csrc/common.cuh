// Shared declarations for libcenterpose_b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/centerpose_b200.h"
#include "ksegments.h"        // fixed_ksegments: the K segments of batch-invariant plans

namespace cp {

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
extern thread_local long long g_launch_counter;      // kernels launched by this thread (every CP_LAUNCH_CHECK)

#define CP_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return ::cp::fail(CP_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

#define CP_LAUNCH_CHECK(what)                                                            \
  do {                                                                                   \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess)                                                               \
      return ::cp::fail(CP_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(_e));  \
    ++::cp::g_launch_counter;                                                            \
  } while (0)

// ---------------------------------------------------------------------------
// Implicit-GEMM convolution, fp32 CUDA-core path (parity mode).
//   out[m, n] = epilogue( sum_k A[m, k] * Wp[k, n] )
//   m = (b, oy, ox) output pixel, n = output channel, k = (ky, kx, ci).
// A is never materialised: it is gathered on the fly from up to 4 NHWC sources
// (channel concatenation, Root nodes), from an NCHW tensor (stems), or by
// bilinear deformable sampling driven by an offset/mask tensor (DCNv2).
// ---------------------------------------------------------------------------
enum IgemmMode {
  IGEMM_NCHW_SCALAR = 0,  // generic k -> (tap, c) decode, NCHW input (7x7 stems, Cin = 1/3/8)
  IGEMM_NHWC_VEC = 1,     // Cin of every source % 16 == 0, float4 gathers
  IGEMM_DCN = 2,          // 3x3 s1 p1 modulated deformable sampling, single NHWC source
  // Dense ConvTranspose2d(k 4, stride 2, pad 1) over one NHWC source (msra_resnet.py:208-233), by sub-pixel phases:
  // output pixel (2y + py, 2x + px) only sees input rows y + dy(py, a) and columns x + dx(px, b), a, b in {0, 1}, with
  // dy(0, a) = -a (ky = 1 + 2a) and dy(1, a) = 1 - a (ky = 2a), the same for columns.  Each phase (py, px) is an
  // implicit GEMM over the INPUT grid with kh = kw = 2 taps, K = 4 Cin (row (2a + b) Cin + ci); the weight matrix is
  // the four phases' [Kpad][CoutPad] blocks in the order py * 2 + px (launch_pack_deconv_weight), and Hout / Wout are
  // the output's 2 Hin / 2 Win.  The phase is a grid coordinate.
  IGEMM_DECONV = 3
};
// deconv phases: input offset and kernel row of tap a of phase p (the same for columns)
__host__ __device__ __forceinline__ int deconv_dy(int p, int a) { return p ? 1 - a : -a; }
__host__ __device__ __forceinline__ int deconv_ky(int p, int a) { return p ? 2 * a : 1 + 2 * a; }

struct IgemmParams {
  const float* src[4];
  int srcC[4];       // channels contributed by each source
  int srcStride[4];  // pixel stride (floats) of each NHWC source (>= srcC)
  int nsrc;
  int B, Hin, Win, Cin;
  int Hout, Wout, Cout, CoutPad;
  int kh, kw, stride, pad;
  int Kpad;              // rows of the packed weight matrix (multiple of 16)
  const float* wgt;      // [Kpad][CoutPad], BN scale folded in
  const float* bias;     // [CoutPad], conv bias + BN shift folded
  const float* residual; // NHWC, Cout channels, pixel stride resStride; or null
  int resStride;
  int relu;
  int res_after_relu;    // 1: out = relu(acc + bias) + residual  (tracking stems)
  float* out;
  int outStride;         // NHWC pixel stride
  int out_nchw;          // 1: write NCHW [B, Cout, Hout, Wout]
  const float* offmask;  // DCN: NHWC [.., omStride] raw conv_offset_mask output (27 used)
  int omStride;
  int mask_is_logit;     // 1: apply sigmoid to channels 18..26
  int mode;
  const void* wgt_umma;  // tensor-core path: pre-swizzled weight tiles (igemm_umma.cu, conv_tma.cu, dcn_tma.cu), else null
  // conv_tma / dcn_tma split-K workspace (plan-owned; null = no split-K): partial sums
  float* splitk_ws;
  size_t splitk_ws_floats;
  // conv_tma only: the per-head 1x1 convolutions fused into the epilogue of the merged heads 3x3 conv.  Head h owns the
  // output columns [h * fuse_hidden, (h + 1) * fuse_hidden); its 1x1 weights are [fuse_hidden][16] fp32 (rows = hidden
  // channel, 16 padded outputs), bias [16], output NCHW [B, fuse_cout[h], Hout, Wout].  fuse_n == 0: not fused.
  int fuse_n, fuse_hidden;
  const float* fuse_w[16];
  const float* fuse_b[16];
  float* fuse_out[16];
  int fuse_cout[16];
  // Several models of one architecture behind one launch (multi-model plans, plan.cu): image n belongs to model
  // n / ipm, whose fp32 weights and biases (wgt, bias, fuse_w, fuse_b) sit (n / ipm) * wstride floats and whose weight
  // tiles sit (n / ipm) * tstride bytes after the pointers above.  NCHW sources (the plan's input frames) are shared by
  // the models: image n reads source image n % ipm.  ipm == 0: one model.
  int ipm;
  long long wstride, tstride;
  // Bit i set: NCHW source src[i] holds one image per launch image (multi-category tracking plans: every model's own
  // previous-frame heat maps), so image n reads its source image n, not n % ipm.  Honoured by the kernels that read NCHW
  // sources (stem_conv7_kernel, the NCHW mode of igemm_fp32).
  unsigned nchw_per_model;
};
// images per model of a launch (model_ipm > 0 everywhere in the kernels)
inline int model_ipm(const IgemmParams& p) { return p.ipm > 0 ? p.ipm : p.B; }

int launch_igemm_fp32(const IgemmParams& p, cudaStream_t stream);

// cp_decode_pnp over the heads of `models` models (decode.cu): prm[0].batch = models x frames, image b is frame
// b % frames of model b / frames and decodes with prm[b / frames].visible_thresh / .balance; meta holds the frames' rows
int decode_pnp_models(const cp_decode_params* prm, int models, const cp_heads* heads, const double* meta, float* dets,
                      float* poses, int32_t* n_valid, void* workspace, size_t workspace_bytes, void* stream);

// What a tensor-core launcher decided for one launch (reported to cp_plan_run_ops; null = not wanted).
struct LaunchInfo {
  int BN = 0;           // N tile
  int ksplit = 1;       // split-K factor (1 = off)
  long long grid = 0;   // CTAs of the main kernel
  int path = 0;         // cp_kpath: how the K segments were summed
};

// dedicated 7x7 stem kernel (stem_conv.cu); consumes the same packed fp32 weights as the generic kernel
bool conv3_c16_supported(const IgemmParams& p);     // direct 3x3 16 -> 16 NHWC convolution (stem_conv.cu)
int launch_conv3_c16(const IgemmParams& p, cudaStream_t stream);
bool stem_supported(const IgemmParams& p);
int launch_stem_conv(const IgemmParams& p, cudaStream_t s);

// The kernel that runs one convolution and its arithmetic (conv_select.cu).
struct ConvKernel {
  int family = CP_FAM_IGEMM_FP32;   // cp_op_family; CP_FAM_NONE: no kernel takes the shape under the policy
  bool x3 = false;                  // tf32 3-term split (fp32-equivalent); otherwise igemm_umma runs bf16 and the TMA
                                    // kernels a single tf32 pass
  bool round_out = false;           // conv_tma / dcn_tma round the stored outputs to tf32
  int BN = 0;                       // N tile (tensor-core families)
  int cslab = 0;                    // channels per activation slab (conv_tma / dcn_tma)
  size_t wbytes = 0;                // bytes of the pre-swizzled weight tiles (0: the kernel reads the fp32 matrix)
  // conv_tma / dcn_tma K segments of a batch-invariant plan (fixed_ksegments, set at plan time); 0: the launcher picks
  // split-K from the launch's tiles and the SM count (splitk_factor)
  int ksegments = 0;
};
// Where the callers of select_conv_kernel differ.
struct ConvPolicy {
  bool small_on_cuda_cores;   // NCHW inputs and Cin < 32 stay on CUDA cores
  bool dcn_tma;               // deformable convs may run on dcn_tma
  bool round_out;             // single-pass tf32 TMA kernels round their outputs to tf32
  bool cuda_core_fallback;    // a tensor-core precision no tensor-core kernel takes runs on CUDA cores (else CP_FAM_NONE)
};
inline bool known_precision(int32_t precision) {
  return precision == CP_PREC_FP32 || precision == CP_PREC_TF32X3 || precision == CP_PREC_BF16 || precision == CP_PREC_TF32;
}
// tf32 and tf32x3 run the gather kernel in tf32x3, bf16 in bf16
inline bool gather_x3(int32_t precision) { return precision == CP_PREC_TF32 || precision == CP_PREC_TF32X3; }
ConvKernel select_conv_kernel(const IgemmParams& p, int32_t precision, const ConvPolicy& pol);
// CUtensorMaps of a TMA family, encoded on the host and passed by value at launch
struct alignas(64) TmaMaps {
  unsigned char map[4][128];
};
int conv_encode(const ConvKernel& k, const IgemmParams& p, int Bmax, TmaMaps* maps);
int conv_pack(const ConvKernel& k, const IgemmParams& p, int ld, void* tiles, cudaStream_t s);
int conv_launch(const ConvKernel& k, const IgemmParams& p, const TmaMaps* maps, cudaStream_t s, LaunchInfo* info = nullptr);
// one stand-alone convolution: select, encode, pack into stream-ordered scratch tiles, launch
int run_conv(IgemmParams& p, int32_t precision, const ConvPolicy& pol, cudaStream_t s);

// Split-K of the persistent TMA kernels: the largest divisor S of `slabs` such that tiles x S CTAs fit the SMs and their
// partial sums (tile_floats each) fit the workspace; 1 = off.  CP_NO_SPLITK=1 turns it off; it is read at every launch.
int splitk_factor(long long tiles, int slabs, int num_sms, size_t tile_floats, size_t ws_floats);
// How a launch of conv_tma / dcn_tma sums the K slabs of its (m, n) tiles.
struct KSplit {
  int ksplit = 1;            // K segments per tile (1: one)
  int sps = 0;               // slabs per segment
  bool fold = false;         // one CTA per tile runs the segments back to back (the FOLD kernel instances)
  long long total_tiles = 0; // tiles of the persistent grid: (m, n) tiles, times ksplit unless folded
  unsigned grid = 0;         // CTAs: min(total_tiles, SMs)
};
// Batch-invariant plans (k.ksegments > 0) take the plan's segments, split over CTAs where the partial sums fit the
// workspace and folded otherwise; other plans split as splitk_factor says.  can_split: the launch has split-K and fold
// instances.  Fails (CP_ERR_INVALID, messages prefixed with `who`) where the segments do not fit the launch.
int ksplit_for(const ConvKernel& k, long long mn_tiles, int slabs, size_t tile_floats, size_t ws_floats, bool can_split,
               const char* who, KSplit* out);

// wgmma tensor-core gather path (igemm_umma.cu).  prec: 0 = bf16, 1 = tf32 x 3 (fp32-equivalent)
bool umma_supported(const IgemmParams& p, int prec);
int umma_tile_n(int CoutPad, int prec);
size_t umma_weight_bytes(int Kreal, int CoutPad, int prec);
int launch_pack_umma_weight(const float* src_k_by_ld, int ld, int Kreal, int Cout, int CoutPad, int prec, void* dst,
                            cudaStream_t s);
int launch_igemm_umma(const IgemmParams& p, int prec, cudaStream_t stream, LaunchInfo* info = nullptr);

// elementwise / data-movement kernels (elementwise.cu)
int launch_maxpool2(const float* in, float* out, int B, int H, int W, int C, cudaStream_t s);
// MaxPool2d(3, 2, 1) over NHWC (msra_resnet.py:120), out = [residual +] maxpool(in); H, W even, C % 4 == 0
int launch_maxpool3s2(const float* in, const float* residual, float* out, int B, int H, int W, int C, cudaStream_t s);
// ConvTranspose2d weight [Cin][Cout][4][4] -> the four phase blocks of IGEMM_DECONV, [4][Kpad][CoutPad], times scale
int launch_pack_deconv_weight(const float* w_io44, const float* scale, float* out, int Cin, int Cout, int CoutPad, int Kpad,
                              cudaStream_t s);
// upsample_add / group_norm_relu: image n uses the weights at (n / ipm) * wstride floats (multi-model plans; ipm = B:
// one model)
int launch_upsample_add(const float* in, const float* wgt_kkc, const float* skip, float* out, int B,
                        int Hin, int Win, int C, int f, cudaStream_t s, int ipm = 0, long long wstride = 0);
// writes the [Kpad x CoutPad] block at column `colOff` of a row-major matrix with leading dimension `ld`
int launch_pack_conv_weight(const float* w_oihw, const float* scale, float* out, int Cout, int Cin,
                            int kh, int kw, int CoutPad, int Kpad, int ld, int colOff, cudaStream_t s,
                            int CinPad = 0);
int launch_pack_bias(const float* conv_bias, const float* bn_w, const float* bn_b, const float* bn_mean,
                     const float* bn_var, float* scale_out, float* bias_out, int C, int CPad, float eps,
                     cudaStream_t s);
int launch_pack_up_weight(const float* w_c1kk, float* out_kkc, int C, int k, cudaStream_t s);
int launch_nchw_to_nhwc(const float* in, float* out, int B, int C, int H, int W, int outStride,
                        int chanOffset, cudaStream_t s);
int launch_nhwc_to_nchw(const float* in, float* out, int B, int C, int H, int W, int inStride, cudaStream_t s);
// GroupNorm+ReLU workspace: gn_workspace_doubles(B) doubles (statistics + per-block partial sums)
constexpr int kGnBlocks = 64, kGnMaxGroups = 64;
inline size_t gn_workspace_doubles(int B) { return (size_t)B * kGnMaxGroups * 2 * (1 + kGnBlocks); }
int launch_group_norm_relu(float* x, const float* gamma, const float* beta, int B, int HW, int C,
                           int stride, int chanOffset, int groups, float eps, double* ws, cudaStream_t s, int ipm = 0,
                           long long wstride = 0);
int launch_gru_gates(const float* xi, const float* hh, const float* hprev, float* hout, int B_HW, int C,
                     int first_step, cudaStream_t s);

// tf32x3: 32-channel K blocks per accumulation group (the tensor core chains them in its accumulator before they are
// added, with round-to-nearest, into fp32 running sums in registers)
constexpr int kX3GroupBlocks = 1;

// TMA-fed shifted-window wgmma convolution (conv_tma.cu): stride-1 1x1 / 3x3 over NHWC fp32, tf32 operands
// x3 = 1: 3-term split with two-level accumulation (fp32-equivalent); x3 = 0: single tf32 pass
bool tma_conv_supported(const IgemmParams& p, int x3);
size_t tma_weight_bytes(int Cin, int taps, int CoutPad, int x3);
int tma_tile_n(int CoutPad, int x3);             // N tile of conv_tma for this output width
int tma_cslab(const IgemmParams& p, int x3);     // channels per activation slab (32 or 16); needs Cin, kh, Win, CoutPad
int launch_pack_tma_weight(const float* src_k_by_ld, int ld, int Cin, int taps, int Cout, int CoutPad, int x3, int cslab,
                           int bn, void* dst, cudaStream_t s);
int tma_encode_nhwc_box(const float* base, int C, int W, int H, int B, int strideFloats, int boxC, int boxW, int boxH,
                        CUtensorMapSwizzle swizzle, void* map_out /* 128 bytes, 64-byte aligned */);
int tma_conv_encode(const IgemmParams& p, int Bmax, int cslab, void* maps_out /* 4 x 128 bytes */);
int launch_conv_tma(const IgemmParams& p, const void* maps, const ConvKernel& k, cudaStream_t stream, LaunchInfo* info);
long long conv_tma_image_tiles(const IgemmParams& p, int BN);     // (m, n) tiles of one image of one model

// TMA-staged deformable convolution (dcn_tma.cu): DCNv2 3x3 stride 1 pad 1 over one NHWC fp32 source, kind::tf32.
// x3 = 1: 3-term split + promoted accumulation (fp32-equivalent);  x3 = 0: single pass.
bool dcn_tma_supported(const IgemmParams& p, int x3);
int dcn_tma_tile_n(int CoutPad, int x3);
int dcn_tma_encode(const IgemmParams& p, int Bmax, void* map_out /* 128 bytes, 64-byte aligned */);
int launch_dcn_tma(const IgemmParams& p, const void* map, const ConvKernel& k, cudaStream_t stream, LaunchInfo* info);
long long dcn_tma_image_tiles(const IgemmParams& p, int BN);      // (m, n) tiles of one image of one model

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
// Output columns of a convolution's packed weight matrix: 16, 32, then multiples of 64 (27 offset/mask channels -> 32)
inline int conv_cout_pad(int Cout) { return round_up(Cout, Cout > 32 ? 64 : (Cout > 16 ? 32 : 16)); }

// ---------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  The forward is ~90 dependent launches; at batch 1 a launch is ~25 us of which the
// launch latency + the fixed prologue of a tensor-core CTA (barrier init, first weight tiles) is a large share.
// Every kernel of the forward schedule therefore (a) signals `launch_dependents` at its very start, so the NEXT kernel's
// CTAs are placed on an SM the moment a CTA of this one retires, and (b) executes `griddep_wait()` before its first
// read of an activation / first global write.  What runs before the wait touches only per-plan constants (weights,
// biases) and the CTA's own shared memory.  A plan that reuses arena memory (CP_PLAN_REUSE_ACTIVATIONS) relies on this: the
// next launch may overwrite what this one reads (DESIGN §4).  Kernels launched without the attribute see both instructions as no-ops.
// g_pdl is set by run_forward (plan.cu) around the op loop; stand-alone ops (cp_conv2d ...) pack their weights on the
// stream right before the launch and therefore never use it.  CP_NO_PDL=1 disables it (A/B runs).
extern thread_local int g_pdl;
#ifdef __CUDACC__
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif
constexpr size_t kSplitkWsFloats = (size_t)160 * 256 * 128;     // >= (#SMs) tile-splits of 256 positions x 128 columns

// Launch attributes (cudaFuncSetAttribute) and the SM count are properties of the CURRENT DEVICE, not of the calling
// thread: the caches below are indexed by cudaGetDevice() so that a process which runs plans on cuda:0 and cuda:1
// configures the > 48 KB shared-memory kernels on both.  (Two threads racing on the same slot set the same attribute
// twice, which is harmless.)
constexpr int kMaxDevices = 64;
inline int current_device_slot() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= kMaxDevices) d = 0;
  return d;
}
template <typename T>
struct PerDevice {
  T v[kMaxDevices] = {};
  T& here() { return v[current_device_slot()]; }
};
inline int device_sm_count(int* out) {
  static PerDevice<int> cache;
  int& n = cache.here();
  if (!n) {
    int dev = 0;
    CP_CUDA_CHECK(cudaGetDevice(&dev));
    CP_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  }
  *out = n;
  return CP_OK;
}
#ifdef __CUDACC__
// A kernel instance and its opt-in to the 227 KB of dynamic shared memory of an SM, made once per device and instance:
// opt_in_smem<Kernel> keeps its own per-device flag.  Null fn: no such instance.
template <class Fn>
struct SmemKernel {
  Fn fn = nullptr;
  int (*opt_in)() = nullptr;
};
template <auto Kernel>
int opt_in_smem() {
  static PerDevice<bool> configured;
  if (!configured.here()) {
    CP_CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured.here() = true;
  }
  return CP_OK;
}
template <auto Kernel>
SmemKernel<decltype(Kernel)> smem_kernel() {
  return {Kernel, opt_in_smem<Kernel>};
}
#endif

}  // namespace cp

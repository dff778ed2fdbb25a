// Which kernel runs a convolution, and the host steps that kernel needs (tensor maps, weight tiles, launch).  The plan
// (plan.cu) and the stand-alone ops (cp_conv2d, cp_dcn_v2_forward_ex, cp_dcn_v2_backward) both choose here; they differ
// only in the ConvPolicy they pass.
#include <stdlib.h>

#include "common.cuh"

namespace cp {

// Tried in this order: dcn_tma, conv_tma (tf32 / tf32x3 only), the wgmma gather kernel, then the CUDA-core kernels.
ConvKernel select_conv_kernel(const IgemmParams& p, int32_t precision, const ConvPolicy& pol) {
  const bool small = p.mode == IGEMM_NCHW_SCALAR || p.Cin < 32;
  if (precision != CP_PREC_FP32 && !(pol.small_on_cuda_cores && small)) {
    const bool tma = precision == CP_PREC_TF32 || precision == CP_PREC_TF32X3;
    const bool x3 = precision == CP_PREC_TF32X3;
    if (tma && pol.dcn_tma && dcn_tma_supported(p, x3))
      return {CP_FAM_DCN_TMA, x3, pol.round_out && !x3, dcn_tma_tile_n(p.CoutPad, x3), 16,
              tma_weight_bytes(p.Cin, 9, p.CoutPad, x3)};
    if (tma && tma_conv_supported(p, x3))
      return {CP_FAM_CONV_TMA, x3, pol.round_out && !x3, tma_tile_n(p.CoutPad, x3), tma_cslab(p, x3),
              tma_weight_bytes(p.Cin, p.kh * p.kw, p.CoutPad, x3)};
    const bool gx3 = gather_x3(precision);
    const int phases = p.mode == IGEMM_DECONV ? 4 : 1;      // a transposed conv has one tile set per phase
    if (umma_supported(p, gx3))
      return {CP_FAM_IGEMM_UMMA, gx3, false, umma_tile_n(p.CoutPad, gx3), 0,
              phases * umma_weight_bytes(p.kh * p.kw * p.Cin, p.CoutPad, gx3)};
    if (!pol.cuda_core_fallback) return {CP_FAM_NONE};
  }
  return {stem_supported(p) ? CP_FAM_STEM : (conv3_c16_supported(p) ? CP_FAM_CONV3_C16 : CP_FAM_IGEMM_FP32)};
}

int conv_encode(const ConvKernel& k, const IgemmParams& p, int Bmax, TmaMaps* maps) {
  if (k.family == CP_FAM_DCN_TMA) return dcn_tma_encode(p, Bmax, maps->map);
  if (k.family == CP_FAM_CONV_TMA) return tma_conv_encode(p, Bmax, k.cslab, maps->map);
  return CP_OK;
}

// Cuts the kernel's weight tiles from the fp32 matrix p.wgt ([Kpad][ld], BN scale folded).
int conv_pack(const ConvKernel& k, const IgemmParams& p, int ld, void* tiles, cudaStream_t s) {
  switch (k.family) {
    case CP_FAM_DCN_TMA:
    case CP_FAM_CONV_TMA:
      return launch_pack_tma_weight(p.wgt, ld, p.Cin, p.kh * p.kw, p.Cout, p.CoutPad, k.x3, k.cslab, k.BN, tiles, s);
    case CP_FAM_IGEMM_UMMA: {
      // IGEMM_DECONV: the phases' [Kpad][ld] blocks follow each other, and so do their tile sets
      const int phases = p.mode == IGEMM_DECONV ? 4 : 1;
      const size_t phase_bytes = k.wbytes / phases;
      for (int ph = 0; ph < phases; ++ph)
        if (int rc = launch_pack_umma_weight(p.wgt + (size_t)ph * p.Kpad * ld, ld, p.kh * p.kw * p.Cin, p.Cout, p.CoutPad,
                                             k.x3, (unsigned char*)tiles + ph * phase_bytes, s))
          return rc;
      return CP_OK;
    }
    default:
      return CP_OK;
  }
}

int conv_launch(const ConvKernel& k, const IgemmParams& p, const TmaMaps* maps, cudaStream_t s, LaunchInfo* info) {
  switch (k.family) {
    case CP_FAM_DCN_TMA: return launch_dcn_tma(p, maps->map, k, s, info);
    case CP_FAM_CONV_TMA: return launch_conv_tma(p, maps->map, k, s, info);
    case CP_FAM_IGEMM_UMMA: return launch_igemm_umma(p, k.x3, s, info);
    case CP_FAM_STEM: return launch_stem_conv(p, s);
    case CP_FAM_CONV3_C16: return launch_conv3_c16(p, s);
    case CP_FAM_IGEMM_FP32: return launch_igemm_fp32(p, s);
    default: return fail(CP_ERR_INVALID, "conv: no kernel selected");
  }
}

// The stand-alone ops pack their tiles on the stream right before the launch and free them after it (stream-ordered).
int run_conv(IgemmParams& p, int32_t precision, const ConvPolicy& pol, cudaStream_t s) {
  const ConvKernel k = select_conv_kernel(p, precision, pol);
  if (k.family == CP_FAM_NONE) return fail(CP_ERR_INVALID, "shape not supported by the wgmma kernel");
  if (!k.wbytes) return conv_launch(k, p, nullptr, s);
  void* tiles = nullptr;
  CP_CUDA_CHECK(cudaMallocAsync(&tiles, k.wbytes, s));
  TmaMaps maps;
  int rc = conv_encode(k, p, p.B, &maps);
  if (!rc) rc = conv_pack(k, p, p.CoutPad, tiles, s);
  if (!rc) {
    p.wgt_umma = tiles;
    rc = conv_launch(k, p, &maps, s);
  }
  cudaFreeAsync(tiles, s);
  return rc;
}

int splitk_factor(long long tiles, int slabs, int num_sms, size_t tile_floats, size_t ws_floats) {
  const char* off = getenv("CP_NO_SPLITK");
  if (!ws_floats || (off && atoi(off) != 0)) return 1;
  int S = 1;
  for (int cand = 2; cand <= slabs; ++cand)
    if (slabs % cand == 0 && tiles * cand <= num_sms && (size_t)tiles * cand * tile_floats <= ws_floats) S = cand;
  return S;
}

int ksplit_for(const ConvKernel& k, long long mn_tiles, int slabs, size_t tile_floats, size_t ws_floats, bool can_split,
               const char* who, KSplit* out) {
  int num_sms = 0;
  if (int rc = device_sm_count(&num_sms)) return rc;
  KSplit r;
  if (k.ksegments > 0) {
    if (slabs % k.ksegments || (k.ksegments > 1 && !can_split))
      return fail(CP_ERR_INVALID, std::string(who) + ": K segments do not fit the launch");
    r.ksplit = k.ksegments;
    r.fold = r.ksplit > 1 && (size_t)mn_tiles * r.ksplit * tile_floats > ws_floats;
  } else {
    r.ksplit = can_split ? splitk_factor(mn_tiles, slabs, num_sms, tile_floats, ws_floats) : 1;
  }
  r.sps = slabs / r.ksplit;
  r.total_tiles = r.fold ? mn_tiles : mn_tiles * r.ksplit;
  if (r.total_tiles >= (1ll << 31)) return fail(CP_ERR_INVALID, std::string(who) + ": too many tiles");
  r.grid = (unsigned)(r.total_tiles < num_sms ? r.total_tiles : num_sms);
  *out = r;
  return CP_OK;
}

}  // namespace cp

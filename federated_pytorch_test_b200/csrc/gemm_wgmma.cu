// Host side of the wgmma implicit-GEMM and weight-gradient kernels: TMA tensor-map construction, tile selection, launch.
// (Kernels: igemm_wgmma.cuh, wgrad_wgmma.cuh.)  Torch-free translation unit: raw pointers + cudaStream_t.
#include "fedb200.h"
#include "igemm_wgmma.cuh"
#include "wgrad_wgmma.cuh"

#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <stdexcept>
#include <string>

namespace fedb200 {

// ------------------------------------------------------------------------------------------------
// cuTensorMapEncodeTiled is a driver entry point; resolve it at run time (no link-time libcuda:
// the build container has no driver).
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr)
      throw std::runtime_error("fedb200: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// TFLOAT32 makes the TMA unit round fp32 -> tf32 (nearest) on the way into shared memory; FLOAT32 copies the bits and
// the tensor core truncates the low 13 mantissa bits.  FEDB200_TMAP_F32=1 selects the latter (experiments).
static CUtensorMapDataType tmap_dtype() {
  const char* v = std::getenv("FEDB200_TMAP_F32");
  return (v && std::atoi(v) == 1) ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;
}

static void check_cu(CUresult r, const char* what) {
  if (r != CUDA_SUCCESS) throw std::runtime_error(std::string("fedb200: ") + what + " failed with CUresult " + std::to_string(int(r)));
}

// fp32 matrix [rows, cols] with row pitch ld (elements): box = [box_rows x 32 cols], 128B swizzle,
// loaded as TF32 (round-to-nearest on the way into shared memory), out-of-bounds zero-filled.
// cw = channels (K elements) per operand row: 32 (one tap per k-block) or 16 / 8 (tap packing, IgemmParams::cw)
static CUtensorMapSwizzle swizzle_for(int cw) {
  return cw == 8 ? CU_TENSOR_MAP_SWIZZLE_32B : (cw == 16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B);
}
static CUtensorMap make_tmap_2d(const float* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, int cw = IG_BLOCK_K) {
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(float)};
  cuuint32_t box[2] = {uint32_t(cw), box_rows};
  cuuint32_t estr[2] = {1, 1};
  check_cu(encode_fn()(&m, tmap_dtype(),2, const_cast<float*>(ptr), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(cw), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
           "cuTensorMapEncodeTiled(2d)");
  return m;
}

// Output map for bulk stores / reduce-adds: plain FLOAT32 elements (the operand maps may use the TF32 element type)
static CUtensorMap make_tmap_out(float* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(float)};
  cuuint32_t box[2] = {32, box_rows};
  cuuint32_t estr[2] = {1, 1};
  check_cu(encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
           "cuTensorMapEncodeTiled(out)");
  return m;
}

// NHWC activation viewed as [C, W, H, N]; a box covers boxN x boxH x boxW output pixels (traversal stride = conv
// stride) x 32 channels and lands in shared memory as a [128 pixels x 128 B] K-major swizzled tile.
static CUtensorMap make_tmap_nhwc(const float* ptr, uint64_t N, uint64_t H, uint64_t W, uint64_t C, uint32_t boxN,
                                  uint32_t boxH, uint32_t boxW, uint32_t stride, int cw = IG_BLOCK_K) {
  CUtensorMap m;
  cuuint64_t dims[4] = {C, W, H, N};
  cuuint64_t strides[3] = {C * sizeof(float), W * C * sizeof(float), H * W * C * sizeof(float)};
  cuuint32_t box[4] = {uint32_t(cw), boxW * stride, boxH * stride, boxN};
  cuuint32_t estr[4] = {1, stride, stride, 1};
  check_cu(encode_fn()(&m, tmap_dtype(),4, const_cast<float*>(ptr), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(cw), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
           "cuTensorMapEncodeTiled(nhwc)");
  return m;
}

static int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return v ? std::atoi(v) : dflt;
}

static int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

static const CUtensorMap* g_out_map_override = nullptr;     // set (and cleared) by conv2d_nhwc_shuffle_tf32 around its dispatch

template <int BN, int ST>
static void launch(const CUtensorMap& ta, const CUtensorMap& tb, IgemmParams p, cudaStream_t stream) {
  using S = IgemmSmem<BN, ST>;
  auto kernel = igemm_wgmma_kernel<BN, ST>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: cudaFuncSetAttribute(igemm): ") + cudaGetErrorString(e));
    configured = true;
  }
  p.m_tiles = (p.M + IG_BLOCK_M - 1) / IG_BLOCK_M;
  p.n_tiles = (p.N + BN - 1) / BN;
  p.total_tiles = p.m_tiles * p.n_tiles * p.k_splits;
  // output map: box = 32 columns x 32 rows (one staging box), 128B swizzle like the operand maps
  p.tma_store = ((p.ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 && env_int("FEDB200_TMA_STORE", 1) != 0) ? 1 : 0;
  if (g_out_map_override != nullptr) p.tma_store = 1;
  const CUtensorMap tc = g_out_map_override != nullptr ? *g_out_map_override : (p.tma_store ? make_tmap_out(p.out, p.M, p.N, p.ldo, 32) : ta);
  // persistent: one CTA per SM walks the tiles; FEDB200_PERSIST=0 launches one CTA per tile (A/B runs)
  const int sms = num_sms();
  const int grid = (p.total_tiles < sms || env_int("FEDB200_PERSIST", 1) == 0) ? p.total_tiles : sms;
  cudaError_t e = launch_pdl(kernel, dim3(grid), dim3(IG_THREADS), S::TOTAL, stream, ta, tb, tc, p);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: igemm launch: ") + cudaGetErrorString(e));
  count_launch();
}

// Stages: as many k-blocks in flight as fit next to the epilogue buffers (~192 KB of the 227 KB a block may use).
static void dispatch(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const IgemmParams& p, cudaStream_t s) {
  switch (bn) {
    case 32: launch<32, 8>(ta, tb, p, s); break;
    case 64: launch<64, 8>(ta, tb, p, s); break;
    default: launch<128, 6>(ta, tb, p, s); break;
  }
}

// The widest N tile that N allows (fewer passes over the activations), up to 128 columns: a 64 x 128 fp32 accumulator
// is 64 registers per thread of a consumer warpgroup.  FEDB200_BLOCK_N overrides for experiments.
int pick_block_n(int M, int N) {
  (void)M;
  const int forced = env_int("FEDB200_BLOCK_N", 0);
  if (forced == 32 || forced == 64 || forced == 128) return forced;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  return 128;
}

// Split-K: slice K until ~one full wave of tiles exists; partial tiles are reduce-added into a zeroed output and the
// BatchNorm statistics come from a separate column pass.  FEDB200_SPLITK forces the number of slices.
static int pick_k_splits(int M, int N, int bn, int num_k_blocks) {
  const int ctas = ((M + IG_BLOCK_M - 1) / IG_BLOCK_M) * ((N + bn - 1) / bn);
  int splits = env_int("FEDB200_SPLITK", 0);
  if (splits <= 0) {
    const int wave = num_sms() + num_sms() / 8;
    splits = 1;
    while (splits < 8 && ctas * splits * 2 <= wave && num_k_blocks / (splits * 2) >= 6) splits *= 2;
  }
  return splits;
}

// ------------------------------------------------------------------------------------------------
void linear_tf32(const float* x, const float* w, const float* bias, float* out, int M, int N, int K, int ldx, int ldw,
                 int ldo, int act, cudaStream_t stream) {
  if ((ldx & 3) || (ldw & 3) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15))
    throw std::runtime_error("fedb200: linear_tf32 needs 16-byte aligned rows");
  const int bn = pick_block_n(M, N);
  CUtensorMap ta = make_tmap_2d(x, M, K, ldx, IG_BLOCK_M);
  CUtensorMap tb = make_tmap_2d(w, N, K, ldw, bn);
  IgemmParams p{};
  p.M = M; p.N = N;
  p.cblocks = (K + IG_BLOCK_K - 1) / IG_BLOCK_K;
  p.num_k_blocks = p.cblocks;
  p.taps_w = 1; p.b_cols_per_tap = 0; p.is_conv = 0;
  p.out = out; p.ldo = ldo; p.bias = bias; p.act = act; p.stats = nullptr;
  p.k_splits = 1; p.kb_per_split = p.num_k_blocks;
  dispatch(bn, ta, tb, p, stream);
}

bool conv_geometry_supported(int H_out, int W_out, int C_in, int stride) {
  if (W_out <= 0 || H_out <= 0 || W_out > 128 || (128 % W_out) != 0) return false;
  const int rows = 128 / W_out;                 // image rows (possibly spanning images) per 128-pixel tile
  if (rows <= H_out ? (H_out % rows) != 0 : (rows % H_out) != 0) return false;
  if ((C_in & 3) != 0) return false;            // 16-byte pixel pitch for TMA
  if (stride < 1 || stride > 2) return false;
  if (W_out * stride > 256) return false;
  return true;
}

// Generic implicit-GEMM convolution.  bias / act (ELU) are applied in the epilogue (VAE / CPC convolutions, SURVEY G6;
// no BatchNorm statistics and no split-K in that case).
static void conv2d_generic(const float* x, const float* w, float* y, float* stats, const float* bias, int act, int NB, int H,
                           int W, int C_in, int C_out, int kh, int kw, int stride, int pad, int dil, int H_out, int W_out,
                           cudaStream_t stream, int accumulate = 0);

void conv2d_nhwc_tf32(const float* x, const float* w, float* y, float* stats, int NB, int H, int W, int C_in, int C_out,
                      int kh, int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream) {
  conv2d_generic(x, w, y, stats, nullptr, 0, NB, H, W, C_in, C_out, kh, kw, stride, pad, dil, H_out, W_out, stream);
}

void conv2d_nhwc_bias_act_tf32(const float* x, const float* w, const float* bias, int act, float* y, int NB, int H, int W,
                               int C_in, int C_out, int kh, int kw, int stride, int pad, int dil, int H_out, int W_out,
                               cudaStream_t stream) {
  conv2d_generic(x, w, y, nullptr, bias, act, NB, H, W, C_in, C_out, kh, kw, stride, pad, dil, H_out, W_out, stream);
}

// y += conv(x, w): the residual-gradient accumulation of an identity-shortcut block fused into the data-gradient
// convolution (experimental, FEDB200_SKIP_FUSED=1): bulk tensor reduce-add epilogue.
void conv2d_nhwc_accumulate_tf32(const float* x, const float* w, float* y, int NB, int H, int W, int C_in, int C_out, int kh,
                                 int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream) {
  conv2d_generic(x, w, y, nullptr, nullptr, 0, NB, H, W, C_in, C_out, kh, kw, stride, pad, dil, H_out, W_out, stream, 1);
}

// Tap packing (IgemmParams::cw): with C_in <= 16 a 32-wide k-block holds 4 (C_in <= 8) or 2 taps instead of one tap padded with
// zeros.  FEDB200_TAP_PACK=0 switches it off (A/B runs).
static int pick_tap_pack(int C_in) {
  if (env_int("FEDB200_TAP_PACK", 1) == 0 || C_in > 16 || (C_in & 3)) return IG_BLOCK_K;
  return C_in <= 8 ? 8 : 16;
}

static void conv2d_generic(const float* x, const float* w, float* y, float* stats, const float* bias, int act, int NB, int H,
                           int W, int C_in, int C_out, int kh, int kw, int stride, int pad, int dil, int H_out, int W_out,
                           cudaStream_t stream, int accumulate) {
  if (!conv_geometry_supported(H_out, W_out, C_in, stride))
    throw std::runtime_error("fedb200: conv geometry not supported by the wgmma path");
  const int rows = 128 / W_out;
  const int boxH = rows <= H_out ? rows : H_out;
  const int boxN = rows <= H_out ? 1 : rows / H_out;
  const int M = NB * H_out * W_out;
  const int bn = pick_block_n(M, C_out);
  const int cw = pick_tap_pack(C_in);
  CUtensorMap ta = make_tmap_nhwc(x, NB, H, W, C_in, boxN, boxH, W_out, stride, cw);
  CUtensorMap tb = make_tmap_2d(w, C_out, uint64_t(kh) * kw * C_in, uint64_t(kh) * kw * C_in, bn, cw);
  IgemmParams p{};
  p.M = M; p.N = C_out;
  p.cblocks = (C_in + IG_BLOCK_K - 1) / IG_BLOCK_K;
  p.num_k_blocks = kh * kw * p.cblocks;
  p.taps_total = kh * kw;
  if (cw != IG_BLOCK_K) {
    p.cw = cw;
    p.num_k_blocks = (kh * kw + IG_BLOCK_K / cw - 1) / (IG_BLOCK_K / cw);
  }
  p.taps_w = kw; p.b_cols_per_tap = C_in; p.is_conv = 1;
  p.HW_out = H_out * W_out; p.W_out = W_out;
  p.stride = stride; p.pad = pad; p.dil = dil;
  p.out = y; p.ldo = C_out; p.bias = bias; p.act = act; p.stats = stats;
  p.k_splits = 1; p.kb_per_split = p.num_k_blocks;
  p.accumulate = accumulate;
  if (bias == nullptr && act == 0) {   // bias / activation must see the complete sum
    const int splits = pick_k_splits(M, C_out, bn, p.num_k_blocks);
    if (splits > 1) {
      p.kb_per_split = (p.num_k_blocks + splits - 1) / splits;
      p.k_splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;   // no empty slices
      p.stats = nullptr;
      if (!accumulate) cudaMemsetAsync(y, 0, size_t(M) * C_out * sizeof(float), stream);
    }
  }
  dispatch(bn, ta, tb, p, stream);
  if (p.k_splits > 1 && stats != nullptr) col_stats(y, stats, M, C_out, stream);
}

// ------------------------------------------------------------------------------------------------
// Stride-2 data gradient / transposed convolution WITHOUT a pixel-shuffle pass: the phase-packed stride-1 convolution
// (ops/conv_math.py: output channels (ph, pw, ci)) stores every 32 x 32 epilogue box straight to
// out[n, 2 ho + ph, 2 wo + pw, ci0 ..] through a 5-D tensor map {ci, pw, wo, ph, n * Ho + ho} over the [N, 2Ho, 2Wo, Ci] result.
// ------------------------------------------------------------------------------------------------
bool conv_shuffle_supported(int H_out, int W_out, int C_in, int Ci_out) {
  if (env_int("FEDB200_SHUFFLE_STORE", 1) == 0) return false;
  if (!conv_geometry_supported(H_out, W_out, C_in, 1)) return false;
  if (Ci_out % 32 != 0) return false;                         // a 32-column box must stay inside one phase
  if (W_out > 32 || (32 % W_out) != 0) return false;          // a 32-row box = whole output rows
  return true;
}

void conv2d_nhwc_shuffle_tf32(const float* x, const float* w, float* out, int NB, int H, int W, int C_in, int C4, int kh, int kw,
                              int pad, int H_out, int W_out, cudaStream_t stream) {
  const int Ci = C4 / 4;
  if (!conv_shuffle_supported(H_out, W_out, C_in, Ci)) throw std::runtime_error("fedb200: shuffled conv store not supported for this shape");
  const int rows = 128 / W_out;
  const int boxH = rows <= H_out ? rows : H_out;
  const int boxN = rows <= H_out ? 1 : rows / H_out;
  const int M = NB * H_out * W_out;
  const int bn = pick_block_n(M, C4);
  CUtensorMap ta = make_tmap_nhwc(x, NB, H, W, C_in, boxN, boxH, W_out, 1);
  CUtensorMap tb = make_tmap_2d(w, C4, uint64_t(kh) * kw * C_in, uint64_t(kh) * kw * C_in, bn);
  CUtensorMap tc;
  {
    cuuint64_t dims[5] = {cuuint64_t(Ci), 2, cuuint64_t(W_out), 2, cuuint64_t(NB) * H_out};
    cuuint64_t strides[4] = {cuuint64_t(Ci) * 4, cuuint64_t(2) * Ci * 4, cuuint64_t(2) * W_out * Ci * 4, cuuint64_t(4) * W_out * Ci * 4};
    cuuint32_t box[5] = {32, 1, cuuint32_t(W_out), 1, cuuint32_t(32 / W_out)};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    check_cu(encode_fn()(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE),
             "cuTensorMapEncodeTiled(shuffle)");
  }
  IgemmParams p{};
  p.M = M; p.N = C4;
  p.cblocks = (C_in + IG_BLOCK_K - 1) / IG_BLOCK_K;
  p.num_k_blocks = kh * kw * p.cblocks;
  p.taps_w = kw; p.b_cols_per_tap = C_in; p.is_conv = 1;
  p.HW_out = H_out * W_out; p.W_out = W_out;
  p.stride = 1; p.pad = pad; p.dil = 1;
  p.out = out; p.ldo = C4; p.bias = nullptr; p.act = 0; p.stats = nullptr;
  p.k_splits = 1; p.kb_per_split = p.num_k_blocks;
  p.shuffle_ci = Ci;
  {   // split-K exactly as conv2d_generic: partial tiles are reduce-added (5-D) into the zeroed result
    const int splits = pick_k_splits(M, C4, bn, p.num_k_blocks);
    if (splits > 1) {
      p.kb_per_split = (p.num_k_blocks + splits - 1) / splits;
      p.k_splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;
      cudaMemsetAsync(out, 0, size_t(M) * C4 * sizeof(float), stream);
    }
  }
  g_out_map_override = &tc;
  try {
    dispatch(bn, ta, tb, p, stream);
  } catch (...) {
    g_out_map_override = nullptr;
    throw;
  }
  g_out_map_override = nullptr;
}

// ------------------------------------------------------------------------------------------------
// Multi-dilation convolution: `branches` convolutions of the SAME input with the same kh x kw / stride but their own dilation and
// padding, each producing its own slice of the output channels, as ONE implicit GEMM (IgemmParams::ms_*): filter rows are
// (branch, row) pairs, the weight matrix w [C_out_total, branches * kh, kw, C_in] is block diagonal.  The CPC encoder's five
// dilated 4x4 / stride-2 stem convolutions + bias + ELU + concatenation.
// ------------------------------------------------------------------------------------------------
bool conv_multidil_supported(int H_out, int W_out, int C_in, int stride, int branches) {
  if (branches < 1 || branches > 8) return false;
  return conv_geometry_supported(H_out, W_out, C_in, stride);
}

void conv2d_nhwc_multidil_tf32(const float* x, const float* w, const float* bias, int act, float* y, int NB, int H, int W, int C_in,
                               int C_out, int branches, int kh, int kw, int stride, const int* dils, const int* pads, int H_out,
                               int W_out, cudaStream_t stream) {
  if (!conv_multidil_supported(H_out, W_out, C_in, stride, branches))
    throw std::runtime_error("fedb200: multi-dilation convolution not supported for this shape");
  const int rows = 128 / W_out;
  const int boxH = rows <= H_out ? rows : H_out;
  const int boxN = rows <= H_out ? 1 : rows / H_out;
  const int M = NB * H_out * W_out;
  const int bn = pick_block_n(M, C_out);
  const int kh_all = branches * kh;
  const int cw = pick_tap_pack(C_in);
  CUtensorMap ta = make_tmap_nhwc(x, NB, H, W, C_in, boxN, boxH, W_out, stride, cw);
  CUtensorMap tb = make_tmap_2d(w, C_out, uint64_t(kh_all) * kw * C_in, uint64_t(kh_all) * kw * C_in, bn, cw);
  IgemmParams p{};
  p.M = M; p.N = C_out;
  p.cblocks = (C_in + IG_BLOCK_K - 1) / IG_BLOCK_K;
  p.num_k_blocks = kh_all * kw * p.cblocks;
  p.taps_total = kh_all * kw;
  if (cw != IG_BLOCK_K) {
    p.cw = cw;
    p.num_k_blocks = (kh_all * kw + IG_BLOCK_K / cw - 1) / (IG_BLOCK_K / cw);
  }
  p.taps_w = kw; p.b_cols_per_tap = C_in; p.is_conv = 1;
  p.HW_out = H_out * W_out; p.W_out = W_out;
  p.stride = stride; p.pad = 0; p.dil = 1;
  p.out = y; p.ldo = C_out; p.bias = bias; p.act = act; p.stats = nullptr;
  p.k_splits = 1; p.kb_per_split = p.num_k_blocks;
  p.ms_kh = kh;
  for (int b = 0; b < branches; ++b) {
    if (dils[b] < 1 || dils[b] > 255 || pads[b] < 0 || pads[b] > 255) throw std::runtime_error("fedb200: multi-dilation: dilation / padding out of range");
    p.ms_dil |= (unsigned long long)(dils[b]) << (8 * b);
    p.ms_pad |= (unsigned long long)(pads[b]) << (8 * b);
  }
  dispatch(bn, ta, tb, p, stream);
}

// ------------------------------------------------------------------------------------------------
// Weight gradient (wgrad_wgmma.cuh)
// ------------------------------------------------------------------------------------------------
bool conv_wgrad_supported(int C_x, int C_out, int stride, int W_out, int H_out) {
  if ((C_x & 3) || (C_out & 3)) return false;
  if (stride < 1 || stride > 8) return false;
  return W_out > 0 && H_out > 0;
}

template <int BN>
static void launch_wgrad(const float* x, const float* dy, const WgradParams& p, int grid, cudaStream_t stream) {
  constexpr int smem = 2 * (WG_A_BYTES + BN * WG_BK * 4);
  auto kernel = wgrad_wgmma_kernel<BN>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: cudaFuncSetAttribute(wgrad): ") + cudaGetErrorString(e));
    configured = true;
  }
  cudaError_t e = launch_pdl(kernel, dim3(grid), dim3(WG_THREADS), size_t(smem), stream, x, dy, p);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: wgrad launch: ") + cudaGetErrorString(e));
  count_launch();
}

// dw [C_out, kh, kw, C_w] += wgrad(x [NB,H,W,C_x], dy [NB,H_out,W_out,C_out]); only the first C_w input channels are
// produced (C_w < C_x when the activation was channel-padded for TMA, e.g. the 3 -> 4 channel stem input).
void conv_wgrad_tf32(const float* x, const float* dy, float* dw, int NB, int H, int W, int C_x, int C_w, int C_out, int kh,
                     int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream) {
  if (!conv_wgrad_supported(C_x, C_out, stride, W_out, H_out))
    throw std::runtime_error("fedb200: wgrad geometry not supported by the wgmma path");
  WgradParams p{};
  p.H = H; p.W = W; p.Cx = C_x; p.Cw = C_w; p.Co = C_out;
  p.kw = kw; p.stride = stride; p.pad = pad; p.dil = dil; p.H_out = H_out; p.W_out = W_out;
  p.J = kh * kw * C_w;
  p.P = NB * H_out * W_out;
  p.dw = dw;
  const int bn = C_out <= 32 ? 32 : (C_out <= 64 ? 64 : 128);   // all output channels in one tile when they fit
  p.j_tiles = (p.J + WG_BM - 1) / WG_BM;
  p.co_tiles = (C_out + bn - 1) / bn;
  // Split the pixel range until ~two CTAs per SM exist (every split adds a full |dW| of red.add traffic in the
  // epilogue), keeping >= 8 k-blocks per CTA.
  const int kb_total = (p.P + WG_BK - 1) / WG_BK;
  const int base = p.j_tiles * p.co_tiles;
  int splits = env_int("FEDB200_WGRAD_SPLITS", 0);
  if (splits <= 0) {
    splits = std::max(1, 2 * num_sms() / base);
    splits = std::min(splits, std::max(1, kb_total / 8));
  }
  splits = std::max(1, std::min(splits, kb_total));
  p.kb_per_split = (kb_total + splits - 1) / splits;
  splits = (kb_total + p.kb_per_split - 1) / p.kb_per_split;       // no empty slices
  const int grid = base * splits;
  switch (bn) {
    case 32: launch_wgrad<32>(x, dy, p, grid, stream); break;
    case 64: launch_wgrad<64>(x, dy, p, grid, stream); break;
    default: launch_wgrad<128>(x, dy, p, grid, stream); break;
  }
}

}  // namespace fedb200

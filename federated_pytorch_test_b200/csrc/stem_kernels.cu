// The ResNet stem: 3 x 3 convolution of the 3-channel input to 64 channels (stride 1, padding 1, no bias) with training-mode
// BatchNorm and ELU, at 32 pixels per image row.
//
// The convolution is tiny (K = 27) next to its 64-channel fp32 output, so the stem is bound by the bytes it writes, not by
// the tensor cores: the wgmma implicit GEMM pads K to 36 with a 4th input channel, and its fp32 pre-BatchNorm tensor y is
// written by the convolution, read back by bn_elu_fwd and written again as the layer output.  stem_conv_bn_kernel instead
// recomputes the convolution from the 2 MB input wherever that saves a pass over y:
//   STEM_STORE_Y     y and the batch statistics (the training forward: bn_elu_fwd and the backward keep using y);
//   STEM_STATS_ONLY  the batch statistics alone;
//   STEM_APPLY       out = ELU(BN(conv(x))) from the complete statistics, plus everything bn_elu_fwd does besides the
//                    output: save_mean / save_invstd, the running-statistics update and the reset of the statistics buffer.
// Without a gradient to take, STATS_ONLY + APPLY replace conv + bn_elu_fwd and y is never stored.
//
// Band = STEM_ROWS output rows of one image (4 x 32 pixels x 64 channels), one warp per row; a CTA walks an equal share of
// the bands (grid sized for STEM_CTAS_PER_SM resident CTAs per SM), so the filter is staged once per CTA and the next band's
// input window is loaded while the current one computes.  The (rows + 2) x 34 x 3 window with its zero halo and the
// 64 x 27 filter sit in shared memory, both rounded to tf32 with cvt.rn (round to nearest, ties to even): the rounding the
// TFLOAT32 tensor maps give the wgmma convolution's operands, so y differs from that path by fp32 summation order only.  The warp computes its 32 x 64 tile with mma.sync.m16n8k8 tf32 (K = 27 padded to 32)
// into fp32 accumulators, one 16-pixel m-tile at a time.  The statistics go into the layer's [sum | sumsq | counter] buffer
// with one atomicAdd per channel and CTA, as the wgmma epilogue adds its tiles.  The tile leaves through a swizzled
// shared-memory row (conflict-free fragment writes) as 16-byte stores of whole 256-byte pixel rows: a warp writes 8 KB of
// contiguous NHWC memory per band.
#include "fedb200.h"

#include <stdexcept>
#include <string>

namespace fedb200 {

namespace {

constexpr int STEM_ROWS = 4;                       // output rows per band, one warp each
constexpr int STEM_THREADS = 32 * STEM_ROWS;
constexpr int STEM_W = 32;                         // output row width (one warp = two m16 tiles)
constexpr int STEM_CI = 3, STEM_CO = 64, STEM_K = 27;
constexpr int STEM_WIN_W = STEM_W + 2;
constexpr int STEM_WIN = (STEM_ROWS + 2) * STEM_WIN_W * STEM_CI;
constexpr int STEM_CTAS_PER_SM = 4;                // resident CTAs per SM the grid is sized for

int stem_sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

__device__ __forceinline__ float stem_tf32(float v) {
  uint32_t r;
  asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}
__device__ __forceinline__ float stem_elu(float v) { return v > 0.f ? v : (__expf(v) - 1.f); }   // as bn_elu_fwd

__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const float (&a)[4], float b0, float b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b0)), "r"(__float_as_uint(b1)));
}

struct StemParams {
  const float* x;          // [N, H, 32, 3]
  const float* w;          // [64, 3, 3, 3] (KRSC)
  float* out;              // [N, H, 32, 64]: y (STORE_Y) or the layer output (APPLY)
  float* stats;            // [sum 64 | sumsq 64 | counter]
  const float* gamma;
  const float* beta;
  float* running_mean;     // may be nullptr
  float* running_var;
  float* save_mean;
  float* save_invstd;
  int H;
  int bands;               // N * H / STEM_ROWS
  float eps, momentum;
  int act, self_clean;
};

}  // namespace

template <int MODE>
__global__ void __launch_bounds__(STEM_THREADS, STEM_CTAS_PER_SM)
stem_conv_bn_kernel(const StemParams p) {
  constexpr bool STORE = MODE != STEM_STATS_ONLY;
  constexpr int WIN_PER = (STEM_WIN + STEM_THREADS - 1) / STEM_THREADS;   // window elements per thread
  __shared__ float xs[2][STEM_WIN];                                      // double-buffered input window
  __shared__ __align__(16) float wf[8 * 4 * 32 * 2];                  // B fragments: [n-tile][k-step][lane][2]
  __shared__ __align__(16) float stage[STORE ? STEM_ROWS * STEM_W * STEM_CO : 4];
  __shared__ float red[STEM_ROWS][2 * STEM_CO];
  __shared__ float bn_sc[STEM_CO], bn_sh[STEM_CO];
  __shared__ int last_block;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int per_img = p.H / STEM_ROWS;
  const int M = p.bands * STEM_ROWS * STEM_W;

  // input window of a band: image rows h0 - 1 .. h0 + ROWS, columns -1 .. 32, zero outside the image; fetched into registers
  // after the current band's MMAs, stored (tf32-rounded) after its stores are issued
  float pre[WIN_PER];
  auto fetch = [&](int band) {
    const int n = band / per_img, h0 = (band - n * per_img) * STEM_ROWS;
    const float* xn = p.x + size_t(n) * p.H * STEM_W * STEM_CI;
#pragma unroll
    for (int u = 0; u < WIN_PER; ++u) {
      const int i = tid + u * STEM_THREADS;
      const int r = i / (STEM_WIN_W * STEM_CI), rem = i - r * (STEM_WIN_W * STEM_CI);
      const int c = rem / STEM_CI, ci = rem - c * STEM_CI;
      const int h = h0 - 1 + r, w = c - 1;
      pre[u] = (i < STEM_WIN && h >= 0 && h < p.H && w >= 0 && w < STEM_W) ? __ldg(xn + (h * STEM_W + w) * STEM_CI + ci) : 0.f;
    }
  };
  auto put = [&](int buf) {
#pragma unroll
    for (int u = 0; u < WIN_PER; ++u) {
      const int i = tid + u * STEM_THREADS;
      if (i < STEM_WIN) xs[buf][i] = stem_tf32(pre[u]);
    }
  };

  pdl_prologue();
  int band = blockIdx.x;                         // the host launches at most p.bands CTAs
  fetch(band);
  // filter as mma B fragments: element e of lane (g, t) in (n-tile j, k-step kk) is W[8 j + g][8 kk + t + 4 e], 0 for k >= 27
  for (int i = tid; i < 8 * 4 * 32 * 2; i += STEM_THREADS) {
    const int e = i & 1, l = (i >> 1) & 31, kk = (i >> 6) & 3, j = i >> 8;
    const int k = 8 * kk + (l & 3) + 4 * e;
    wf[i] = k < STEM_K ? stem_tf32(__ldg(p.w + (8 * j + (l >> 2)) * STEM_K + k)) : 0.f;
  }
  if constexpr (MODE == STEM_APPLY) {
    if (tid < STEM_CO) {            // exactly bn_elu_fwd's arithmetic on the complete sums
      const float invM = 1.f / float(M);
      const float mean = p.stats[tid] * invM;
      float var = fmaf(-mean, mean, p.stats[STEM_CO + tid] * invM);
      var = var > 0.f ? var : 0.f;
      const float invstd = rsqrtf(var + p.eps);
      const float sc = p.gamma[tid] * invstd;
      bn_sc[tid] = sc;
      bn_sh[tid] = fmaf(-mean, sc, p.beta[tid]);
      if (blockIdx.x == 0) {
        p.save_mean[tid] = mean;
        p.save_invstd[tid] = invstd;
        if (p.running_mean != nullptr) {
          const float unbiased = M > 1 ? var * float(M) / float(M - 1) : var;
          p.running_mean[tid] = fmaf(p.momentum, mean - p.running_mean[tid], p.running_mean[tid]);
          p.running_var[tid] = fmaf(p.momentum, unbiased - p.running_var[tid], p.running_var[tid]);
        }
      }
    }
  }
  put(0);
  __syncthreads();
  if constexpr (MODE == STEM_APPLY) {
    if (p.self_clean) {
      // every thread of every block reads the statistics before its block counts itself: the last block zeroes them
      unsigned int* counter = reinterpret_cast<unsigned int*>(p.stats + 2 * STEM_CO);
      if (tid == 0) {
        __threadfence();
        last_block = atomicAdd(counter, 1u) == gridDim.x - 1;
      }
      __syncthreads();
      if (last_block) {
        for (int c = tid; c < 2 * STEM_CO; c += STEM_THREADS) p.stats[c] = 0.f;
        if (tid == 0) *counter = 0u;
      }
    }
  }

  // A element (pixel column col, k) of this warp's row = xs[(warp * 34 + col) * 3 + koff(k)], koff(k) = (r * 34 + s) * 3 + ci
  int koff[4][2];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int k = 8 * kk + t + 4 * e, tap = k / STEM_CI, ci = k - tap * STEM_CI;
      koff[kk][e] = k < STEM_K ? ((tap / 3) * STEM_WIN_W + tap % 3) * STEM_CI + ci : -1;
    }
  // per-warp statistics of this CTA's bands, red[warp][c] / red[warp][64 + c], owned by lane (g = 0, t = (c % 8) / 2)
  if constexpr (MODE != STEM_APPLY) {
    for (int c = lane; c < 2 * STEM_CO; c += 32) red[warp][c] = 0.f;
    __syncwarp();
  }

  for (int it = 0; band < p.bands; band += gridDim.x, ++it) {
    const int buf = it & 1;
    const int next = band + gridDim.x;
    const float* xw = xs[buf];
    float* st = stage + warp * STEM_W * STEM_CO;   // this warp's staging row (STORE modes)
    if constexpr (STORE) __syncwarp();             // the previous band's reads of it are done
    // one 16-pixel m-tile at a time: 32 accumulators live, not 64 (4 CTAs per SM without spills)
#pragma unroll 1
    for (int mt = 0; mt < 2; ++mt) {
      float acc[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[j][q] = 0.f;
      const int p0 = (warp * STEM_WIN_W + 16 * mt + g) * STEM_CI;       // pixel column 16 mt + g; + 8 columns = + 24 floats
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        float a[4];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = koff[kk][e] >= 0;
          a[2 * e] = ok ? xw[p0 + koff[kk][e]] : 0.f;
          a[2 * e + 1] = ok ? xw[p0 + 8 * STEM_CI + koff[kk][e]] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 b = *reinterpret_cast<const float2*>(&wf[((j * 4 + kk) * 32 + lane) * 2]);
          mma_tf32_16x8x8(acc[j], a, b.x, b.y);
        }
      }

      // n-tile by n-tile, so that each accumulator dies once it is counted and staged
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if constexpr (MODE != STEM_APPLY) {
          // channel 8 j + 2 t + e: this thread's 2 pixels, then the 8 lanes g of the warp, into the warp's partial
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v0 = acc[j][e], v1 = acc[j][2 + e];
            float a1 = v0 + v1, a2 = fmaf(v1, v1, v0 * v0);
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
              a1 += __shfl_xor_sync(0xffffffffu, a1, o);
              a2 += __shfl_xor_sync(0xffffffffu, a2, o);
            }
            if (g == 0) {
              red[warp][8 * j + 2 * t + e] += a1;
              red[warp][STEM_CO + 8 * j + 2 * t + e] += a2;
            }
          }
        }
        if constexpr (STORE) {
          // element (px, c) of the staging row at px * 64 + ((c / 4) ^ (px % 16)) * 4 + c % 4
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int px = 16 * mt + g + 8 * hh, c = 8 * j + 2 * t;
            float v0 = acc[j][2 * hh], v1 = acc[j][2 * hh + 1];
            if constexpr (MODE == STEM_APPLY) {
              v0 = fmaf(v0, bn_sc[c], bn_sh[c]);
              v1 = fmaf(v1, bn_sc[c + 1], bn_sh[c + 1]);
              if (p.act) { v0 = stem_elu(v0); v1 = stem_elu(v1); }
            }
            *reinterpret_cast<float2*>(st + px * STEM_CO + (((c >> 2) ^ (px & 15)) << 2) + (c & 3)) = make_float2(v0, v1);
          }
        }
      }
    }
    if (next < p.bands) fetch(next);               // in flight while this band's stores issue
    if constexpr (STORE) {
      // 16-byte stores of whole 256-byte pixel rows: the warp's image row is 8 KB of contiguous NHWC memory
      __syncwarp();
      const int n = band / per_img, h0 = (band - n * per_img) * STEM_ROWS;
      float4* dst = reinterpret_cast<float4*>(p.out + ((size_t(n) * p.H + h0 + warp) * STEM_W) * STEM_CO);
      const float4* src = reinterpret_cast<const float4*>(st);
#pragma unroll
      for (int i = 0; i < STEM_W * STEM_CO / 4 / 32; ++i) {
        const int idx = 32 * i + lane, px = idx >> 4, q = idx & 15;
        dst[idx] = src[px * 16 + (q ^ (px & 15))];
      }
    }
    if (next < p.bands) put(buf ^ 1);              // its last readers passed the previous iteration's barrier
    __syncthreads();
  }

  if constexpr (MODE != STEM_APPLY) {
    // over the warps (the loop's last barrier made their partials visible): one atomicAdd per channel and CTA
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < STEM_ROWS; ++w) a += red[w][tid];
    atomicAdd(p.stats + tid, a);                   // tid < 128 = [sum 64 | sumsq 64]
  }
}

bool stem_conv_supported(int H, int W, int C_in, int C_out) {
  return W == STEM_W && H > 0 && H % STEM_ROWS == 0 && C_in == STEM_CI && C_out == STEM_CO;
}

void stem_conv_bn(int mode, const float* x, const float* w, float* out, float* stats, const float* gamma, const float* beta,
                  float* running_mean, float* running_var, float* save_mean, float* save_invstd, int NB, int H, float eps,
                  float momentum, int act, int self_clean, cudaStream_t stream) {
  if (!stem_conv_supported(H, STEM_W, STEM_CI, STEM_CO) || NB <= 0)
    throw std::runtime_error("fedb200: stem_conv_bn needs [N, H, 32, 3] input with H % 4 == 0 and 64 output channels");
  if ((mode == STEM_STORE_Y || mode == STEM_APPLY) && (reinterpret_cast<uintptr_t>(out) & 15))
    throw std::runtime_error("fedb200: stem_conv_bn needs a 16-byte aligned output");
  if (mode == STEM_APPLY && (gamma == nullptr || beta == nullptr || save_mean == nullptr || save_invstd == nullptr))
    throw std::runtime_error("fedb200: stem_conv_bn APPLY needs gamma, beta, save_mean and save_invstd");
  const int bands = NB * (H / STEM_ROWS);
  StemParams p{x, w, out, stats, gamma, beta, running_mean, running_var, save_mean, save_invstd, H, bands, eps, momentum, act,
               self_clean};
  // up to STEM_CTAS_PER_SM CTAs per SM, each taking the same number of bands (the filter is staged once per CTA, and the
  // statistics leave it in one atomicAdd per channel)
  const int per_cta = (bands + STEM_CTAS_PER_SM * stem_sm_count() - 1) / (STEM_CTAS_PER_SM * stem_sm_count());
  const dim3 grid((bands + per_cta - 1) / per_cta);
  cudaError_t e;
  switch (mode) {
    case STEM_STORE_Y: e = launch_pdl(stem_conv_bn_kernel<STEM_STORE_Y>, grid, dim3(STEM_THREADS), 0, stream, p); break;
    case STEM_STATS_ONLY: e = launch_pdl(stem_conv_bn_kernel<STEM_STATS_ONLY>, grid, dim3(STEM_THREADS), 0, stream, p); break;
    case STEM_APPLY: e = launch_pdl(stem_conv_bn_kernel<STEM_APPLY>, grid, dim3(STEM_THREADS), 0, stream, p); break;
    default: throw std::runtime_error("fedb200: stem_conv_bn: unknown mode");
  }
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: stem_conv_bn launch: ") + cudaGetErrorString(e));
  count_launch();
}

}  // namespace fedb200

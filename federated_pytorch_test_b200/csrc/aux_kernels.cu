// Hand-written fp32 kernels for the small / awkward operators of the model zoo — everything that is NOT a large
// convolution (those are on wgmma: gemm_wgmma.cu, wgrad_wgmma.cuh):
//
//  * gemm_f32_kernel        true-fp32 strided GEMM with bias / ELU / accumulate epilogue: nn.Linear forward, data and
//                           weight gradients (SURVEY G5; the reference runs nn.Linear in true fp32, and so does this)
//  * act_bwd_bias_kernel    dz = dout * ELU'(z) (from the saved output) and db = column sums of dz in one pass
//  * maxpool2x2 fwd / bwd   NCHW (Net / Net1 / Net2, SURVEY G4)
//  * argmax_count_kernel    evaluation: argmax over classes, compare with the label, count — on the device (G21)
//  * info_nce fwd / bwd     normalised P x P Gram over R rows + diagonal log-softmax (+ closed-form gradient), G12
//  * gauss_nll_rows fwd/bwd per-(cluster, sample) Gaussian negative log-likelihood sums of the VAE-CL cost 1, G11
//  * smallconv fwd/dgrad/wgrad   direct convolutions for channel counts / map sizes the TMA path cannot tile
//                           (Net: 3->6->16 channels, 5x5, 28 / 10 wide maps), NCHW, bias + ELU (+ 2x2 max-pool) fused
//
// Reference sites (library calls or Python loops there): /root/reference/src/simple_models.py:9-39 (Net), :257-261,
// :322-335 (dense layers); src/federated_multi.py:108-121 (evaluation); src/federated_cpc.py:149-180 (InfoNCE);
// src/federated_vae_cl.py:101-109 (cost 1).
#include "fedb200.h"

#include <stdexcept>
#include <string>

namespace fedb200 {

static inline void aux_check(const char* name) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: ") + name + ": " + cudaGetErrorString(e));
  count_launch();
}
static int aux_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}
__device__ __forceinline__ float elu_f(float v) { return v > 0.f ? v : (expf(v) - 1.f); }
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------------------------
// C[i, j] (+)= act( sum_k A(i, k) * B(k, j) + bias[j] ),  A(i,k) = a[i*sa_i + k*sa_k],  B(k,j) = b[k*sb_k + j*sb_j]
// BM x BN tile per CTA (64 x 64, or 32 x 32 when the 64-tiles would leave most SMs idle: the dense layers of the model zoo
// are 128 x 16 ... 1280 x 128 outputs), 16-deep k tiles, 256 threads x (BM/16 x BN/16) outputs, true fp32 (FFMA).
// The next k tile is fetched into registers while the current one is multiplied (one barrier per tile): these GEMMs are
// latency bound, so the load of the next tile must overlap the multiply of the current one.
// ------------------------------------------------------------------------------------------------------------------
constexpr int GF_BK = 16;

template <int BM, int BN>
__global__ void __launch_bounds__(256)
gemm_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ bias, float* __restrict__ c,
                int M, int N, int K, long long sa_i, long long sa_k, long long sb_k, long long sb_j, int ldc, int act, int accumulate) {
  constexpr int TM = BM / 16, TN = BN / 16;            // outputs per thread
  constexpr int EA = BM * GF_BK / 256, EB = BN * GF_BK / 256;
  __shared__ float As[2][GF_BK][BM + 4];
  __shared__ float Bs[2][GF_BK][BN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
  float acc[TM][TN];
#pragma unroll
  for (int u = 0; u < TM; ++u)
#pragma unroll
    for (int v = 0; v < TN; ++v) acc[u][v] = 0.f;
  float ra[EA], rb[EB];
  // element e of this thread inside a tile: the contiguous dimension runs along consecutive threads
  auto a_pos = [&](int e, int& ai, int& ak) {
    const int idx = threadIdx.x + e * 256;
    if (sa_k == 1) { ak = idx % GF_BK; ai = idx / GF_BK; } else { ai = idx % BM; ak = idx / BM; }
  };
  auto b_pos = [&](int e, int& bj, int& bk) {
    const int idx = threadIdx.x + e * 256;
    if (sb_j == 1) { bj = idx % BN; bk = idx / BN; } else { bk = idx % GF_BK; bj = idx / GF_BK; }
  };
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < EA; ++e) {
      int ai, ak;
      a_pos(e, ai, ak);
      const int gi = i0 + ai, gk = k0 + ak;
      ra[e] = (gi < M && gk < K) ? __ldg(a + gi * sa_i + gk * sa_k) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < EB; ++e) {
      int bj, bk;
      b_pos(e, bj, bk);
      const int gj = j0 + bj, gk = k0 + bk;
      rb[e] = (gj < N && gk < K) ? __ldg(b + gk * sb_k + gj * sb_j) : 0.f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < EA; ++e) {
      int ai, ak;
      a_pos(e, ai, ak);
      As[buf][ak][ai] = ra[e];
    }
#pragma unroll
    for (int e = 0; e < EB; ++e) {
      int bj, bk;
      b_pos(e, bj, bk);
      Bs[buf][bk][bj] = rb[e];
    }
  };
  const int nk = (K + GF_BK - 1) / GF_BK;
  fetch(0);
  stash(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nk) fetch((kt + 1) * GF_BK);          // in flight while this tile is multiplied
#pragma unroll
    for (int kk = 0; kk < GF_BK; ++kk) {
      float av[TM], bv[TN];
#pragma unroll
      for (int u = 0; u < TM; ++u) av[u] = As[cur][kk][ty * TM + u];
#pragma unroll
      for (int v = 0; v < TN; ++v) bv[v] = Bs[cur][kk][tx * TN + v];
#pragma unroll
      for (int u = 0; u < TM; ++u)
#pragma unroll
        for (int v = 0; v < TN; ++v) acc[u][v] = fmaf(av[u], bv[v], acc[u][v]);
    }
    if (kt + 1 < nk) stash(cur ^ 1);                   // the other buffer was last read before the previous barrier
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < TM; ++u) {
    const int gi = i0 + ty * TM + u;
    if (gi >= M) continue;
#pragma unroll
    for (int v = 0; v < TN; ++v) {
      const int gj = j0 + tx * TN + v;
      if (gj >= N) continue;
      float r = acc[u][v];
      if (bias != nullptr) r += __ldg(bias + gj);
      if (act) r = elu_f(r);
      float* dst = c + size_t(gi) * ldc + gj;
      *dst = accumulate ? (*dst + r) : r;
    }
  }
}

void gemm_f32(const float* a, const float* b, const float* bias, float* c, int M, int N, int K, long long sa_i, long long sa_k,
              long long sb_k, long long sb_j, int ldc, int act, int accumulate, cudaStream_t s) {
  const int ctas64 = ((N + 63) / 64) * ((M + 63) / 64);
  if (ctas64 < aux_sms() / 2) {
    dim3 grid((N + 31) / 32, (M + 31) / 32);
    gemm_f32_kernel<32, 32><<<grid, 256, 0, s>>>(a, b, bias, c, M, N, K, sa_i, sa_k, sb_k, sb_j, ldc, act, accumulate);
  } else {
    dim3 grid((N + 63) / 64, (M + 63) / 64);
    gemm_f32_kernel<64, 64><<<grid, 256, 0, s>>>(a, b, bias, c, M, N, K, sa_i, sa_k, sb_k, sb_j, ldc, act, accumulate);
  }
  aux_check("gemm_f32");
}

// ------------------------------------------------------------------------------------------------------------------
// dz[m, c] = dout[m, c] * (act ? ELU'(z) : 1) with ELU'(z) = out > 0 ? 1 : out + 1;  db[c] += sum_m dz[m, c]
// [M, C] row-major (NHWC activations or dense-layer outputs).  Every thread keeps ONE column (its stride is a multiple
// of C), so the bias sum is a register accumulation + one shared-memory atomic per thread.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
act_bwd_bias_kernel(const float* __restrict__ dout, const float* __restrict__ out, float* __restrict__ dz, float* __restrict__ db,
                    long long total, int C, int act) {
  extern __shared__ float s_db[];
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_db[c] = 0.f;
  __syncthreads();
  const long long nth = (long long)gridDim.x * blockDim.x;
  const long long nth_eff = (nth / C) * C;             // threads beyond it idle: keeps (i % C) constant per thread
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < nth_eff) {
    float acc = 0.f;
    for (long long i = tid; i < total; i += nth_eff) {
      float g = dout[i];
      if (act) {
        const float o = out[i];
        g *= (o > 0.f ? 1.f : o + 1.f);
      }
      if (dz != nullptr) dz[i] = g;
      acc += g;
    }
    if (db != nullptr) atomicAdd(&s_db[int(tid % C)], acc);
  }
  __syncthreads();
  if (db != nullptr)
    for (int c = threadIdx.x; c < C; c += blockDim.x)
      if (s_db[c] != 0.f) atomicAdd(db + c, s_db[c]);
}

void act_bwd_bias(const float* dout, const float* out, float* dz, float* db, long long total, int C, int act, cudaStream_t s) {
  if (C > 8192) throw std::runtime_error("fedb200: act_bwd_bias: too many channels");
  long long want = (total + 256 * 8 - 1) / (256 * 8);
  int grid = int(want < 1 ? 1 : (want > 4LL * aux_sms() ? 4LL * aux_sms() : want));
  while ((long long)grid * 256 < C) ++grid;            // at least one full row of threads
  act_bwd_bias_kernel<<<grid, 256, C * sizeof(float), s>>>(dout, out, dz, db, total, C, act);
  aux_check("act_bwd_bias");
}

// ------------------------------------------------------------------------------------------------------------------
// 2x2 / stride 2 max pooling, NCHW or NHWC memory (nhwc = 1: the layout the wgmma convolutions produce).
// idx: which of the four window positions won (uint8) — the backward needs nothing else.
// ------------------------------------------------------------------------------------------------------------------
struct PoolGeom {
  int N, C, H, W, Ho, Wo, nhwc;
};
__device__ __forceinline__ void pool_decode(const PoolGeom& g, long long i, long long& base, int& sw, int& sh) {
  // i indexes the OUTPUT in its own memory order; returns the offset of the window's top-left input element
  if (g.nhwc) {
    const int c = int(i % g.C);
    long long t = i / g.C;
    const int wo = int(t % g.Wo);
    t /= g.Wo;
    const int ho = int(t % g.Ho);
    const long long n = t / g.Ho;
    sw = g.C;
    sh = g.W * g.C;
    base = ((n * g.H + 2 * ho) * g.W + 2 * wo) * (long long)g.C + c;
  } else {
    const int wo = int(i % g.Wo);
    long long t = i / g.Wo;
    const int ho = int(t % g.Ho);
    const long long pl = t / g.Ho;
    sw = 1;
    sh = g.W;
    base = (pl * g.H + 2 * ho) * g.W + 2 * wo;
  }
}
__global__ void __launch_bounds__(256)
maxpool2x2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, unsigned char* __restrict__ idx, PoolGeom g) {
  const long long total = (long long)g.N * g.C * g.Ho * g.Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long base;
    int sw, sh;
    pool_decode(g, i, base, sw, sh);
    const float* src = x + base;
    float best = src[0];
    unsigned char bi = 0;
    if (src[sw] > best) { best = src[sw]; bi = 1; }
    if (src[sh] > best) { best = src[sh]; bi = 2; }
    if (src[sh + sw] > best) { best = src[sh + sw]; bi = 3; }
    y[i] = best;
    if (idx != nullptr) idx[i] = bi;
  }
}
__global__ void __launch_bounds__(256)
maxpool2x2_bwd_kernel(const float* __restrict__ dy, const unsigned char* __restrict__ idx, float* __restrict__ dx, PoolGeom g) {
  const long long total = (long long)g.N * g.C * g.Ho * g.Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long base;
    int sw, sh;
    pool_decode(g, i, base, sw, sh);
    float* dst = dx + base;
    const float gr = dy[i];
    const unsigned char bi = idx[i];
    dst[0] = bi == 0 ? gr : 0.f;
    dst[sw] = bi == 1 ? gr : 0.f;
    dst[sh] = bi == 2 ? gr : 0.f;
    dst[sh + sw] = bi == 3 ? gr : 0.f;
  }
}
static int ew_grid(long long total) {
  long long want = (total + 255) / 256;
  const long long cap = 16LL * aux_sms();
  return int(want < 1 ? 1 : (want > cap ? cap : want));
}
void maxpool2x2_fwd(const float* x, float* y, unsigned char* idx, int N, int C, int H, int W, int nhwc, cudaStream_t s) {
  PoolGeom g{N, C, H, W, H / 2, W / 2, nhwc};
  maxpool2x2_fwd_kernel<<<ew_grid((long long)N * C * g.Ho * g.Wo), 256, 0, s>>>(x, y, idx, g);
  aux_check("maxpool2x2_fwd");
}
void maxpool2x2_bwd(const float* dy, const unsigned char* idx, float* dx, int N, int C, int H, int W, int nhwc, cudaStream_t s) {
  PoolGeom g{N, C, H, W, H / 2, W / 2, nhwc};
  if ((H & 1) || (W & 1)) cudaMemsetAsync(dx, 0, size_t(N) * C * H * W * sizeof(float), s);   // odd edge rows get no gradient
  maxpool2x2_bwd_kernel<<<ew_grid((long long)N * C * g.Ho * g.Wo), 256, 0, s>>>(dy, idx, dx, g);
  aux_check("maxpool2x2_bwd");
}

// ------------------------------------------------------------------------------------------------------------------
// evaluation: counter[0] += #(argmax_c logits[b, c] == labels[b]), counter[1] += B     (first maximum wins, like torch)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
argmax_count_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, long long* __restrict__ counter, int B, int C) {
  int hit = 0;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    const float* row = logits + size_t(b) * C;
    float best = row[0];
    int bi = 0;
    for (int c = 1; c < C; ++c)
      if (row[c] > best) { best = row[c]; bi = c; }
    hit += (bi == int(labels[b])) ? 1 : 0;
  }
  hit = __reduce_add_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0 && hit != 0) atomicAdd(reinterpret_cast<unsigned long long*>(counter), (unsigned long long)hit);
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(reinterpret_cast<unsigned long long*>(counter + 1), (unsigned long long)B);
}
void argmax_count(const float* logits, const long long* labels, long long* counter, int B, int C, cudaStream_t s) {
  argmax_count_kernel<<<(B + 255) / 256, 256, 0, s>>>(logits, labels, counter, B, C);
  aux_check("argmax_count");
}

// ------------------------------------------------------------------------------------------------------------------
// InfoNCE (federated_cpc.py:149-180).  Z, Zh: [R, P] row-major (R = batch * channels, P = patches).
//   S[i,j] = sum_r Z[r,i] Zh[r,j],  a_i = ||Z[:,i]||, b_j = ||Zh[:,j]||,  G = S / (a b^T),  p = softmax_row(G)
//   loss = - sum_i log(p_ii + 1e-6)
// Forward: ONE kernel — every CTA accumulates the P*P + 2P dot products over a slab of rows (shared-memory tiles, one
// (i, j) pair per thread and pass), partial sums go to a device scratch, the last CTA to finish evaluates the P x P
// epilogue and ALSO the closed-form gradient coefficients
//   dS[i,j] = w_i (p_ij - delta_ij) / (a_i b_j),  va_i = -(sum_j dG_ij G_ij) / a_i^2,  vb_j = -(sum_i dG_ij G_ij) / b_j^2,
// (w_i = p_ii / (p_ii + eps)), so that the backward is one elementwise-class kernel:
//   dZ[r,i] = g (sum_j dS[i,j] Zh[r,j] + va_i Z[r,i]),   dZh[r,j] = g (sum_i dS[i,j] Z[r,i] + vb_j Zh[r,j]).
// ------------------------------------------------------------------------------------------------------------------
constexpr int NCE_MAX_P = 32;
constexpr int NCE_TR = 64;      // rows per shared-memory tile

__global__ void __launch_bounds__(256)
info_nce_fwd_kernel(const float* __restrict__ Z, const float* __restrict__ Zh, int R, int P, float* __restrict__ scratch,
                    float* __restrict__ loss, float* __restrict__ coef) {
  __shared__ float zt[NCE_TR][NCE_MAX_P + 1];
  __shared__ float ht[NCE_TR][NCE_MAX_P + 1];
  __shared__ int s_last;
  const int npair = P * P + 2 * P;                      // S pairs, then a^2 (Z.Z diagonal), then b^2
  float acc[5];                                         // ceil((32*32 + 64) / 256) = 5 pairs per thread at most
#pragma unroll
  for (int q = 0; q < 5; ++q) acc[q] = 0.f;
  const int rows_per_cta = (R + gridDim.x - 1) / gridDim.x;
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(R, r_begin + rows_per_cta);
  for (int r0 = r_begin; r0 < r_end; r0 += NCE_TR) {
    const int nr = min(NCE_TR, r_end - r0);
    for (int e = threadIdx.x; e < nr * P; e += blockDim.x) {
      const int rr = e / P, pp = e - rr * P;
      zt[rr][pp] = Z[size_t(r0 + rr) * P + pp];
      ht[rr][pp] = Zh[size_t(r0 + rr) * P + pp];
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const int pr = threadIdx.x + q * 256;
      if (pr < npair) {
        float s = 0.f;
        if (pr < P * P) {
          const int i = pr / P, j = pr - i * P;
          for (int rr = 0; rr < nr; ++rr) s = fmaf(zt[rr][i], ht[rr][j], s);
        } else if (pr < P * P + P) {
          const int i = pr - P * P;
          for (int rr = 0; rr < nr; ++rr) s = fmaf(zt[rr][i], zt[rr][i], s);
        } else {
          const int j = pr - P * P - P;
          for (int rr = 0; rr < nr; ++rr) s = fmaf(ht[rr][j], ht[rr][j], s);
        }
        acc[q] += s;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    const int pr = threadIdx.x + q * 256;
    if (pr < npair && acc[q] != 0.f) atomicAdd(scratch + pr, acc[q]);
  }
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned* ticket = reinterpret_cast<unsigned*>(scratch + NCE_MAX_P * NCE_MAX_P + 2 * NCE_MAX_P);
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  // ---- epilogue: one row of G per thread --------------------------------------------------------------------------
  __threadfence();
  __shared__ float Gs[NCE_MAX_P][NCE_MAX_P + 1];
  __shared__ float dG[NCE_MAX_P][NCE_MAX_P + 1];
  __shared__ float na[NCE_MAX_P], nb[NCE_MAX_P];
  __shared__ float s_loss[NCE_MAX_P];
  if (threadIdx.x < P) {
    na[threadIdx.x] = sqrtf(__ldcg(scratch + P * P + threadIdx.x));
    nb[threadIdx.x] = sqrtf(__ldcg(scratch + P * P + P + threadIdx.x));
  }
  __syncthreads();
  if (threadIdx.x < P) {
    const int i = threadIdx.x;
    float mx = -3.4e38f;
    for (int j = 0; j < P; ++j) {
      const float g = __ldcg(scratch + i * P + j) / (na[i] * nb[j]);
      Gs[i][j] = g;
      mx = fmaxf(mx, g);
    }
    float den = 0.f;
    for (int j = 0; j < P; ++j) den += expf(Gs[i][j] - mx);
    const float pii = expf(Gs[i][i] - mx) / den;
    s_loss[i] = -logf(pii + 1e-6f);
    const float w = pii / (pii + 1e-6f);
    for (int j = 0; j < P; ++j) {
      const float pij = expf(Gs[i][j] - mx) / den;
      dG[i][j] = w * (pij - (i == j ? 1.f : 0.f));
    }
  }
  __syncthreads();
  if (threadIdx.x < P) {
    const int i = threadIdx.x;
    float sa = 0.f, sb = 0.f;
    for (int j = 0; j < P; ++j) {
      sa += dG[i][j] * Gs[i][j];
      sb += dG[j][i] * Gs[j][i];
      coef[i * P + j] = dG[i][j] / (na[i] * nb[j]);                 // dS
    }
    coef[P * P + i] = -sa / (na[i] * na[i]);                          // va
    coef[P * P + P + i] = -sb / (nb[i] * nb[i]);                      // vb
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f;
    for (int i = 0; i < P; ++i) l += s_loss[i];
    loss[0] = l;
  }
  for (int e = threadIdx.x; e < NCE_MAX_P * NCE_MAX_P + 2 * NCE_MAX_P + 4; e += blockDim.x) scratch[e] = 0.f;   // self-cleaning
}

__global__ void __launch_bounds__(256)
info_nce_bwd_kernel(const float* __restrict__ Z, const float* __restrict__ Zh, const float* __restrict__ coef,
                    const float* __restrict__ gout, float* __restrict__ dZ, float* __restrict__ dZh, int R, int P) {
  __shared__ float dS[NCE_MAX_P][NCE_MAX_P + 1];
  __shared__ float va[NCE_MAX_P], vb[NCE_MAX_P];
  for (int e = threadIdx.x; e < P * P; e += blockDim.x) dS[e / P][e % P] = coef[e];
  if (threadIdx.x < P) { va[threadIdx.x] = coef[P * P + threadIdx.x]; vb[threadIdx.x] = coef[P * P + P + threadIdx.x]; }
  __syncthreads();
  const float g = gout[0];
  const long long total = (long long)R * P;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = int(e / P), c = int(e - (long long)r * P);
    const float* zr = Z + size_t(r) * P;
    const float* hr = Zh + size_t(r) * P;
    float dz = va[c] * zr[c], dh = vb[c] * hr[c];
    for (int j = 0; j < P; ++j) {
      dz = fmaf(dS[c][j], hr[j], dz);
      dh = fmaf(dS[j][c], zr[j], dh);
    }
    dZ[e] = g * dz;
    dZh[e] = g * dh;
  }
}
int info_nce_max_p() { return NCE_MAX_P; }
int info_nce_scratch_floats() { return NCE_MAX_P * NCE_MAX_P + 2 * NCE_MAX_P + 4; }
void info_nce_fwd(const float* Z, const float* Zh, int R, int P, float* scratch, float* loss, float* coef, cudaStream_t s) {
  if (P < 1 || P > NCE_MAX_P) throw std::runtime_error("fedb200: info_nce: 1 <= P <= 32 patches supported by the fused kernel");
  int grid = (R + 4 * NCE_TR - 1) / (4 * NCE_TR);
  grid = grid < 1 ? 1 : (grid > aux_sms() ? aux_sms() : grid);
  info_nce_fwd_kernel<<<grid, 256, 0, s>>>(Z, Zh, R, P, scratch, loss, coef);
  aux_check("info_nce_fwd");
}
void info_nce_bwd(const float* Z, const float* Zh, const float* coef, const float* gout, float* dZ, float* dZh, int R, int P,
                  cudaStream_t s) {
  info_nce_bwd_kernel<<<ew_grid((long long)R * P), 256, 0, s>>>(Z, Zh, coef, gout, dZ, dZh, R, P);
  aux_check("info_nce_bwd");
}

// ------------------------------------------------------------------------------------------------------------------
// VAE-CL cost 1 (federated_vae_cl.py:101-109): rows[k*B + b] = sum_d (x[b,d] - mu[k,b,d])^2 / (2 s[k,b,d]) + log(2 pi s)/2
// mu, s: [Kc*B, D]; x: [B, D] (broadcast over clusters).  One CTA per row; backward is elementwise.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gauss_nll_rows_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ s2,
                          float* __restrict__ rows, int B, int D) {
  __shared__ float sm[8];
  const int row = blockIdx.x;
  const float* xr = x + size_t(row % B) * D;
  const float* mr = mu + size_t(row) * D;
  const float* sr = s2 + size_t(row) * D;
  float acc = 0.f;
  const int Dv = (D & 3) == 0 ? D : 0;                  // 16-byte aligned rows only when D is a multiple of 4
  for (int d = threadIdx.x * 4; d + 3 < Dv; d += blockDim.x * 4) {
    const float4 xv = *reinterpret_cast<const float4*>(xr + d);
    const float4 mv = *reinterpret_cast<const float4*>(mr + d);
    const float4 sv = *reinterpret_cast<const float4*>(sr + d);
    const float e0 = xv.x - mv.x, e1 = xv.y - mv.y, e2 = xv.z - mv.z, e3 = xv.w - mv.w;
    acc += e0 * e0 / (2.f * sv.x) + 0.5f * logf(sv.x * 6.283185307179586f);
    acc += e1 * e1 / (2.f * sv.y) + 0.5f * logf(sv.y * 6.283185307179586f);
    acc += e2 * e2 / (2.f * sv.z) + 0.5f * logf(sv.z * 6.283185307179586f);
    acc += e3 * e3 / (2.f * sv.w) + 0.5f * logf(sv.w * 6.283185307179586f);
  }
  for (int d = (Dv & ~3) + threadIdx.x; d < D; d += blockDim.x) {
    const float e = xr[d] - mr[d];
    acc += e * e / (2.f * sr[d]) + 0.5f * logf(sr[d] * 6.283185307179586f);
  }
  acc = warp_sum_f(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += sm[w];
    rows[row] = t;
  }
}
// dmu = g_row (mu - x) / s;  ds = g_row (1/(2 s) - (x - mu)^2 / (2 s^2))
__global__ void __launch_bounds__(256)
gauss_nll_rows_bwd_kernel(const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ s2,
                          const float* __restrict__ grow, float* __restrict__ dmu, float* __restrict__ ds2, int B, int D,
                          long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / D;
    const int d = int(i - row * D);
    const float g = grow[row];
    const float e = x[size_t(row % B) * D + d] - mu[i];
    const float s = s2[i];
    dmu[i] = -g * e / s;
    ds2[i] = g * (0.5f / s - e * e / (2.f * s * s));
  }
}
void gauss_nll_rows_fwd(const float* x, const float* mu, const float* s2, float* rows, int nrows, int B, int D, cudaStream_t s) {
  gauss_nll_rows_fwd_kernel<<<nrows, 256, 0, s>>>(x, mu, s2, rows, B, D);
  aux_check("gauss_nll_rows_fwd");
}
void gauss_nll_rows_bwd(const float* x, const float* mu, const float* s2, const float* grow, float* dmu, float* ds2, int nrows,
                        int B, int D, cudaStream_t s) {
  const long long total = (long long)nrows * D;
  gauss_nll_rows_bwd_kernel<<<ew_grid(total), 256, 0, s>>>(x, mu, s2, grow, dmu, ds2, B, D, total);
  aux_check("gauss_nll_rows_bwd");
}

// ------------------------------------------------------------------------------------------------------------------
// Direct convolutions for shapes the TMA / wgmma path cannot tile (channel counts not multiples of 4, map widths
// that do not divide 128): NCHW, stride 1, "valid" or zero padding, square k <= 7, weights staged in shared memory.
//   fwd   : y = ELU?(conv(x, w) + b), optionally followed by a fused 2x2 max-pool (the pre-pool map is not stored:
//           the backward recomputes nothing — it gets the winner index and the pooled activation)
//   dgrad : dx[n,ci,h,w] = sum_{co,r,s} dz[n,co,h-r+p,w-s+p] w[co,ci,r,s]
//   wgrad : dw[co,ci,r,s] = sum_{n,ho,wo} dz[n,co,ho,wo] x[n,ci,ho+r-p,wo+s-p]   (+ db), CTA per (co, ci), block reduction
// These layers are tiny (Net: 90 + 61 MFLOP per batch); the point is that no cuDNN call is left on the default model.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
smallconv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                     unsigned char* __restrict__ pidx, int NB, int Ci, int H, int W, int Co, int k, int pad, int act, int pool) {
  extern __shared__ float ws[];                        // [Co][Ci][k][k] + bias[Co]
  const int wn = Co * Ci * k * k;
  for (int e = threadIdx.x; e < wn; e += blockDim.x) ws[e] = w[e];
  for (int e = threadIdx.x; e < Co; e += blockDim.x) ws[wn + e] = bias != nullptr ? bias[e] : 0.f;
  __syncthreads();
  const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
  const int Hp = pool ? Ho / 2 : Ho, Wp = pool ? Wo / 2 : Wo;
  const long long total = (long long)NB * Co * Hp * Wp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wp = int(i % Wp);
    long long t = i / Wp;
    const int hp = int(t % Hp);
    t /= Hp;
    const int co = int(t % Co);
    const int n = int(t / Co);
    const int reps = pool ? 4 : 1;
    float best = -3.4e38f;
    unsigned char bi = 0;
    for (int q = 0; q < reps; ++q) {
      const int ho = pool ? 2 * hp + (q >> 1) : hp, wo = pool ? 2 * wp + (q & 1) : wp;
      float acc = ws[wn + co];
      for (int ci = 0; ci < Ci; ++ci) {
        const float* xp = x + (size_t(n) * Ci + ci) * H * W;
        const float* wp_ = ws + ((co * Ci + ci) * k) * k;
        for (int r = 0; r < k; ++r) {
          const int hh = ho + r - pad;
          if (hh < 0 || hh >= H) continue;
          for (int s = 0; s < k; ++s) {
            const int ww = wo + s - pad;
            if (ww < 0 || ww >= W) continue;
            acc = fmaf(__ldg(xp + hh * W + ww), wp_[r * k + s], acc);
          }
        }
      }
      if (act) acc = elu_f(acc);
      if (acc > best) { best = acc; bi = (unsigned char)q; }
    }
    y[i] = best;
    if (pool && pidx != nullptr) pidx[i] = bi;
  }
}
// dz: gradient w.r.t. the PRE-activation conv output at full resolution [NB, Co, Ho, Wo]
__global__ void __launch_bounds__(256)
smallconv_dgrad_kernel(const float* __restrict__ dz, const float* __restrict__ w, float* __restrict__ dx, int NB, int Ci, int H, int W,
                       int Co, int k, int pad) {
  extern __shared__ float ws[];
  const int wn = Co * Ci * k * k;
  for (int e = threadIdx.x; e < wn; e += blockDim.x) ws[e] = w[e];
  __syncthreads();
  const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
  const long long total = (long long)NB * Ci * H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ww = int(i % W);
    long long t = i / W;
    const int hh = int(t % H);
    t /= H;
    const int ci = int(t % Ci);
    const int n = int(t / Ci);
    float acc = 0.f;
    for (int co = 0; co < Co; ++co) {
      const float* dp = dz + (size_t(n) * Co + co) * Ho * Wo;
      const float* wp_ = ws + ((co * Ci + ci) * k) * k;
      for (int r = 0; r < k; ++r) {
        const int ho = hh - r + pad;
        if (ho < 0 || ho >= Ho) continue;
        for (int s = 0; s < k; ++s) {
          const int wo = ww - s + pad;
          if (wo < 0 || wo >= Wo) continue;
          acc = fmaf(__ldg(dp + ho * Wo + wo), wp_[r * k + s], acc);
        }
      }
    }
    dx[i] = acc;
  }
}
// one CTA per (co, ci): k*k accumulators per thread over a strided share of the (n, ho, wo) range; dw / db accumulated
__global__ void __launch_bounds__(256)
smallconv_wgrad_kernel(const float* __restrict__ dz, const float* __restrict__ x, float* __restrict__ dw, float* __restrict__ db,
                       int NB, int Ci, int H, int W, int Co, int k, int pad) {
  __shared__ float red[8];
  const int co = blockIdx.x / Ci, ci = blockIdx.x - co * Ci;
  const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
  float acc[49];
#pragma unroll
  for (int q = 0; q < 49; ++q) acc[q] = 0.f;
  float bsum = 0.f;
  const int npix = NB * Ho * Wo;
  for (int pix = threadIdx.x; pix < npix; pix += blockDim.x) {
    const int wo = pix % Wo;
    const int t = pix / Wo;
    const int ho = t % Ho;
    const int n = t / Ho;
    const float g = __ldg(dz + ((size_t(n) * Co + co) * Ho + ho) * Wo + wo);
    bsum += g;
    const float* xp = x + (size_t(n) * Ci + ci) * H * W;
#pragma unroll
    for (int r = 0; r < 7; ++r) {
      if (r >= k) break;
      const int hh = ho + r - pad;
      if (hh < 0 || hh >= H) continue;
#pragma unroll
      for (int s = 0; s < 7; ++s) {
        if (s >= k) break;
        const int ww = wo + s - pad;
        if (ww < 0 || ww >= W) continue;
        acc[r * 7 + s] = fmaf(g, __ldg(xp + hh * W + ww), acc[r * 7 + s]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 7; ++r) {
#pragma unroll
    for (int s = 0; s < 7; ++s) {
      if (r >= k || s >= k) continue;                   // uniform across the CTA
      float v = warp_sum_f(acc[r * 7 + s]);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
      __syncthreads();
      if (threadIdx.x == 0) {
        float tsum = 0.f;
        for (int wq = 0; wq < 8; ++wq) tsum += red[wq];
        dw[((size_t(co) * Ci + ci) * k + r) * k + s] += tsum;
      }
      __syncthreads();
    }
  }
  if (db != nullptr && ci == 0) {
    float v = warp_sum_f(bsum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tsum = 0.f;
      for (int wq = 0; wq < 8; ++wq) tsum += red[wq];
      db[co] += tsum;
    }
  }
}
bool smallconv_supported(int Ci, int Co, int k) { return k >= 1 && k <= 7 && (Co * Ci * k * k + Co) * 4 <= 200 * 1024; }
void smallconv_fwd(const float* x, const float* w, const float* bias, float* y, unsigned char* pidx, int NB, int Ci, int H, int W,
                   int Co, int k, int pad, int act, int pool, cudaStream_t s) {
  const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
  const long long total = (long long)NB * Co * (pool ? Ho / 2 : Ho) * (pool ? Wo / 2 : Wo);
  const size_t smem = size_t(Co * Ci * k * k + Co) * sizeof(float);
  static bool cfg = false;
  if (!cfg) {
    cudaFuncSetAttribute(smallconv_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(smallconv_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cfg = true;
  }
  smallconv_fwd_kernel<<<ew_grid(total), 256, smem, s>>>(x, w, bias, y, pidx, NB, Ci, H, W, Co, k, pad, act, pool);
  aux_check("smallconv_fwd");
}
void smallconv_dgrad(const float* dz, const float* w, float* dx, int NB, int Ci, int H, int W, int Co, int k, int pad, cudaStream_t s) {
  const size_t smem = size_t(Co * Ci * k * k) * sizeof(float);
  static bool cfg = false;
  if (!cfg) {
    cudaFuncSetAttribute(smallconv_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cfg = true;
  }
  smallconv_dgrad_kernel<<<ew_grid((long long)NB * Ci * H * W), 256, smem, s>>>(dz, w, dx, NB, Ci, H, W, Co, k, pad);
  aux_check("smallconv_dgrad");
}
void smallconv_wgrad(const float* dz, const float* x, float* dw, float* db, int NB, int Ci, int H, int W, int Co, int k, int pad,
                     cudaStream_t s) {
  smallconv_wgrad_kernel<<<Co * Ci, 256, 0, s>>>(dz, x, dw, db, NB, Ci, H, W, Co, k, pad);
  aux_check("smallconv_wgrad");
}
// dz (pre-activation, full resolution) from the gradient of the pooled / activated output:
//   pool: scatter dy to the winner position; act: multiply by ELU'(z) recomputed from the stored (post-activation) value
__global__ void __launch_bounds__(256)
smallconv_unpool_actbwd_kernel(const float* __restrict__ dy, const float* __restrict__ yout, const unsigned char* __restrict__ pidx,
                               float* __restrict__ dz, long long planes, int Ho, int Wo, int act, int pool) {
  const int Hp = pool ? Ho / 2 : Ho, Wp = pool ? Wo / 2 : Wo;
  const long long total = planes * Hp * Wp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float g = dy[i];
    if (act) {
      const float o = yout[i];
      g *= (o > 0.f ? 1.f : o + 1.f);
    }
    if (!pool) {
      dz[i] = g;
    } else {
      const int wp = int(i % Wp);
      const long long t = i / Wp;
      const int hp = int(t % Hp);
      const long long pl = t / Hp;
      const unsigned char bi = pidx[i];
      float* dst = dz + (pl * Ho + 2 * hp) * Wo + 2 * wp;
      dst[0] = bi == 0 ? g : 0.f;
      dst[1] = bi == 1 ? g : 0.f;
      dst[Wo] = bi == 2 ? g : 0.f;
      dst[Wo + 1] = bi == 3 ? g : 0.f;
    }
  }
}
void smallconv_unpool_actbwd(const float* dy, const float* yout, const unsigned char* pidx, float* dz, long long planes, int Ho, int Wo,
                             int act, int pool, cudaStream_t s) {
  if (pool && ((Ho & 1) || (Wo & 1))) cudaMemsetAsync(dz, 0, size_t(planes) * Ho * Wo * sizeof(float), s);
  const long long total = planes * (pool ? Ho / 2 : Ho) * (pool ? Wo / 2 : Wo);
  smallconv_unpool_actbwd_kernel<<<ew_grid(total), 256, 0, s>>>(dy, yout, pidx, dz, planes, Ho, Wo, act, pool);
  aux_check("smallconv_unpool_actbwd");
}

}  // namespace fedb200

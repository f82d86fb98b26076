// GroupNorm (Wu & He 2018) + residual + ELU on NHWC fp32, forward and backward, for the GroupNorm ResNets.
//
// A sample's activations are one contiguous [HW, C] slab.  Every pass runs on a (split, sample) grid: block (s, n) owns the
// pixel rows [s HW / S, (s + 1) HW / S) of sample n, with the thread layout of the BatchNorm kernels (thread t owns channel
// quad t % (C/4) of rows t / (C/4), t / (C/4) + rpi, ...; 16-byte loads along C).  Partials are kept per (sample, split,
// channel), so any group count G that divides C works, down to one channel per group.
//
// Forward:  gn_stats      per-(n, s, c) mean and M2 of the split (shifted sums, then Chan merges across the block's rows)
//           gn_finalize   per sample: merge the splits per channel, then the channels of each group, in a fixed order ->
//                         mean / rstd [N, G] and the per-(n, c) scale / shift table
//           gn_apply      out = ELU?(y * scale[n, c] + shift[n, c] (+ residual))
// Backward: gn_bwd_reduce per-(n, s, c) sums of du and du * xhat, du = dout * ELU'
//           gn_bwd_merge  A[n, g] = sum_c gamma_c sum du, B[n, g] = sum_c gamma_c sum du xhat; dbeta / dgamma over (n, s)
//           gn_bwd_apply  dy = rstd (gamma_c du - A / M - xhat B / M), M = HW C / G; dres = du
// No floating-point atomics and every sum in a fixed order: the same inputs give the same bits, run after run.
#include "fedb200.h"

#include <stdexcept>
#include <string>

namespace fedb200 {

namespace {

constexpr int GN_THREADS = 256;

void check_launch(const char* name) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: ") + name + ": " + cudaGetErrorString(e));
  count_launch();
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

__device__ __forceinline__ float elu_f(float v) { return v > 0.f ? v : (__expf(v) - 1.f); }

// The block's share of one sample: rows [lo, lo + len) of the [HW, C] slab, thread layout as described above.
struct Slab {
  int q, cq, r0, rpi, lo, len;
  size_t base;      // float4 index of the first row of the split
};
__device__ __forceinline__ Slab slab(int HW, int C, int S) {
  Slab b;
  b.q = C >> 2;
  b.cq = threadIdx.x % b.q;
  b.r0 = threadIdx.x / b.q;
  b.rpi = GN_THREADS / b.q;
  const int s = blockIdx.x, n = blockIdx.y;
  b.lo = int((long long)s * HW / S);
  b.len = int((long long)(s + 1) * HW / S) - b.lo;
  b.base = (size_t(n) * HW + b.lo) * b.q;
  return b;
}
// rows of the split that thread row r0 visits
__device__ __forceinline__ int rows_of(int len, int r0, int rpi) { return r0 < len ? (len - r0 + rpi - 1) / rpi : 0; }

__device__ __forceinline__ float4 ld4(const float* p, size_t i) { return reinterpret_cast<const float4*>(p)[i]; }
__device__ __forceinline__ void st4(float* p, size_t i, float4 v) { reinterpret_cast<float4*>(p)[i] = v; }
__device__ __forceinline__ void to4(float (&a)[4], float4 v) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }

// (n_a, mean_a, m2_a) <- merge with (n_b, mean_b, m2_b)  (Chan, Golub & LeVeque)
__device__ __forceinline__ void chan_merge(float& na, float& ma, float& m2a, float nb, float mb, float m2b) {
  const float n = na + nb;
  if (nb == 0.f) return;
  const float d = mb - ma, f = nb / n;
  ma = fmaf(d, f, ma);
  m2a = m2a + m2b + d * d * na * f;
  na = n;
}

// Per-thread quad partials (p1, p2) of every thread row -> thread rows [0, q) of the block, merged over the rows in order
// (rpi entries).  MERGE: Chan merge of (mean, M2) with the row counts; otherwise plain sums.  Results land in (p1, p2) of the
// threads with r0 == 0.
template <bool MERGE>
__device__ __forceinline__ void block_rows_reduce(float (&p1)[4], float (&p2)[4], const Slab& b, float* sm) {
  float* a = sm + threadIdx.x * 4;
  float* c = sm + GN_THREADS * 4 + threadIdx.x * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) { a[j] = p1[j]; c[j] = p2[j]; }
  __syncthreads();
  if (threadIdx.x < b.q) {
    float cnt = float(rows_of(b.len, 0, b.rpi));
    for (int rr = 1; rr < b.rpi; ++rr) {
      const float* a2 = sm + (rr * b.q + b.cq) * 4;
      const float* c2 = sm + GN_THREADS * 4 + (rr * b.q + b.cq) * 4;
      if (MERGE) {
        const float nb = float(rows_of(b.len, rr, b.rpi));
        float na;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          na = cnt;
          chan_merge(na, p1[j], p2[j], nb, a2[j], c2[j]);
        }
        cnt = na;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) { p1[j] += a2[j]; p2[j] += c2[j]; }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const float* __restrict__ y, float* __restrict__ part, int HW, int C, int S) {
  pdl_prologue();
  __shared__ __align__(16) float sm[2 * GN_THREADS * 4];
  const Slab b = slab(HW, C, S);
  const bool active = b.r0 < b.rpi;
  float p1[4] = {0, 0, 0, 0}, p2[4] = {0, 0, 0, 0};
  const int cnt = active ? rows_of(b.len, b.r0, b.rpi) : 0;
  if (cnt > 0) {
    // shifted sums: every value minus the split's first value of its channel, so an offset far above the spread cancels
    // before it is squared
    float k[4], s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
    to4(k, ld4(y, b.base + b.cq));
    const int step = b.rpi;
    for (int r = b.r0; r < b.len; r += 4 * step) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld4(y, b.base + size_t(r + u * step < b.len ? r + u * step : r) * b.q + b.cq);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + u * step >= b.len) continue;
        float vv[4];
        to4(vv, v[u]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float d = vv[j] - k[j];
          s1[j] += d;
          s2[j] = fmaf(d, d, s2[j]);
        }
      }
    }
    const float inv = 1.f / float(cnt);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float dm = s1[j] * inv;
      p1[j] = k[j] + dm;
      p2[j] = fmaxf(fmaf(-s1[j], dm, s2[j]), 0.f);
    }
  }
  block_rows_reduce<true>(p1, p2, b, sm);
  if (threadIdx.x < b.q) {
    float* dst = part + (size_t(blockIdx.y) * S + blockIdx.x) * 2 * C;
    st4(dst, b.cq, make_float4(p1[0], p1[1], p1[2], p1[3]));
    st4(dst + C, b.cq, make_float4(p2[0], p2[1], p2[2], p2[3]));
  }
}

// one block per sample
__global__ void __launch_bounds__(GN_THREADS)
gn_finalize_kernel(const float* __restrict__ part, const float* __restrict__ gamma, const float* __restrict__ beta,
                   float* __restrict__ mean, float* __restrict__ rstd, float* __restrict__ table, int HW, int C, int G, int S,
                   float eps) {
  pdl_prologue();
  __shared__ float cm[1024], cv[1024];     // per-channel mean / M2 over the sample
  __shared__ float gms[256], grs[256];     // per-group mean / rstd
  const int n = blockIdx.x;
  const float* src = part + size_t(n) * S * 2 * C;
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {
    float na = 0.f, ma = 0.f, m2 = 0.f;
    for (int s = 0; s < S; ++s) {
      const float nb = float(int((long long)(s + 1) * HW / S) - int((long long)s * HW / S));
      if (s == 0) {
        na = nb;
        ma = src[c];
        m2 = src[C + c];
      } else {
        chan_merge(na, ma, m2, nb, src[size_t(s) * 2 * C + c], src[size_t(s) * 2 * C + C + c]);
      }
    }
    cm[c] = ma;
    cv[c] = m2;
  }
  __syncthreads();
  // groups: one warp each; the cpg channels of a group all hold HW values, so the group mean is the mean of the channel
  // means and M2 = sum_c (M2_c + HW (mean_c - mean)^2).  Lane-strided sums + a butterfly: a fixed order.
  const int cpg = C / G, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = warp; g < G; g += GN_THREADS / 32) {
    float s = 0.f;
    for (int i = lane; i < cpg; i += 32) s += cm[g * cpg + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float gm = s / float(cpg);
    float m2 = 0.f;
    for (int i = lane; i < cpg; i += 32) {
      const float d = cm[g * cpg + i] - gm;
      m2 += fmaf(float(HW) * d, d, cv[g * cpg + i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    const float r = rsqrtf(m2 / (float(HW) * float(cpg)) + eps);
    if (lane == 0) {
      mean[size_t(n) * G + g] = gm;
      rstd[size_t(n) * G + g] = r;
      gms[g] = gm;
      grs[g] = r;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {
    const int g = c / cpg;
    const float sc = gamma[c] * grs[g];
    table[size_t(n) * 2 * C + c] = sc;
    table[size_t(n) * 2 * C + C + c] = fmaf(-gms[g], sc, beta[c]);
  }
}

__global__ void __launch_bounds__(GN_THREADS)
gn_apply_kernel(const float* __restrict__ y, const float* __restrict__ table, const float* __restrict__ residual,
                float* __restrict__ out, int HW, int C, int S, int act) {
  pdl_prologue();
  const Slab b = slab(HW, C, S);
  if (b.r0 >= b.rpi) return;
  float sc[4], sh[4];
  to4(sc, ld4(table + size_t(blockIdx.y) * 2 * C, b.cq));
  to4(sh, ld4(table + size_t(blockIdx.y) * 2 * C + C, b.cq));
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  const int step = b.rpi;
  for (int r = b.r0; r < b.len; r += 4 * step) {
    float4 v[4], rs[4];
    size_t i[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) i[u] = b.base + size_t(r + u * step < b.len ? r + u * step : r) * b.q + b.cq;
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld4(y, i[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) rs[u] = residual != nullptr ? ld4(residual, i[u]) : zero;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r + u * step >= b.len) continue;
      float4 o = make_float4(fmaf(v[u].x, sc[0], sh[0]) + rs[u].x, fmaf(v[u].y, sc[1], sh[1]) + rs[u].y,
                             fmaf(v[u].z, sc[2], sh[2]) + rs[u].z, fmaf(v[u].w, sc[3], sh[3]) + rs[u].w);
      if (act) { o.x = elu_f(o.x); o.y = elu_f(o.y); o.z = elu_f(o.z); o.w = elu_f(o.w); }
      st4(out, i[u], o);
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// Per-(n, c) coefficients of one thread's channel quad: mean / rstd of the channel's group, and (MODE 2) the forward's
// scale / shift, recomputed with the forward's arithmetic so that ELU' sees the same pre-activation.
struct GnCoef {
  float mu[4], rs[4], ga[4], sc[4], sh[4];
};
__device__ __forceinline__ GnCoef gn_coef(const float* mean, const float* rstd, const float* gamma, const float* beta, int n,
                                          int cq, int C, int G) {
  GnCoef k;
  const int cpg = C / G;
  to4(k.ga, ld4(gamma, cq));
  float bb[4] = {0, 0, 0, 0};
  if (beta != nullptr) to4(bb, ld4(beta, cq));
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int g = (cq * 4 + j) / cpg;
    k.mu[j] = mean[size_t(n) * G + g];
    k.rs[j] = rstd[size_t(n) * G + g];
    k.sc[j] = k.ga[j] * k.rs[j];
    k.sh[j] = fmaf(-k.mu[j], k.sc[j], bb[j]);
  }
  return k;
}
// du = dout * ELU'(z).  MODE 0: no activation, 1: ELU' from out (z > 0 <=> out > 0, exp(z) = out + 1), 2: z recomputed from y
template <int MODE>
__device__ __forceinline__ void gn_du(float (&d)[4], const float (&o)[4], const float (&v)[4], const GnCoef& k) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (MODE == 1) {
      d[j] *= o[j] > 0.f ? 1.f : (o[j] + 1.f);
    } else if (MODE == 2) {
      const float z = fmaf(v[j], k.sc[j], k.sh[j]);
      d[j] *= z > 0.f ? 1.f : __expf(z);
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_reduce_kernel(const float* __restrict__ dout, const float* __restrict__ out, const float* __restrict__ y,
                     const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                     const float* __restrict__ beta, float* __restrict__ part, int HW, int C, int G, int S) {
  pdl_prologue();
  __shared__ __align__(16) float sm[2 * GN_THREADS * 4];
  const Slab b = slab(HW, C, S);
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  if (b.r0 < b.rpi) {
    const GnCoef k = gn_coef(mean, rstd, gamma, beta, blockIdx.y, b.cq, C, G);
    const int step = b.rpi;
    for (int r = b.r0; r < b.len; r += 4 * step) {
      float4 d[4], o[4], v[4];
      size_t i[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) i[u] = b.base + size_t(r + u * step < b.len ? r + u * step : r) * b.q + b.cq;
#pragma unroll
      for (int u = 0; u < 4; ++u) d[u] = ld4(dout, i[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld4(y, i[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) o[u] = MODE == 1 ? ld4(out, i[u]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + u * step >= b.len) continue;
        float dd[4], oo[4], vv[4];
        to4(dd, d[u]); to4(oo, o[u]); to4(vv, v[u]);
        gn_du<MODE>(dd, oo, vv, k);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s1[j] += dd[j];
          s2[j] = fmaf(dd[j], (vv[j] - k.mu[j]) * k.rs[j], s2[j]);
        }
      }
    }
  }
  block_rows_reduce<false>(s1, s2, b, sm);
  if (threadIdx.x < b.q) {
    float* dst = part + (size_t(blockIdx.y) * S + blockIdx.x) * 2 * C;
    st4(dst, b.cq, make_float4(s1[0], s1[1], s1[2], s1[3]));
    st4(dst + C, b.cq, make_float4(s2[0], s2[1], s2[2], s2[3]));
  }
}

// blocks [0, N): sample n's per-group A, B -> ab[n, g], ab[N G + n G + g].  Blocks [N, N + C/32): 32 channels each, dbeta /
// dgamma summed over the N S partial rows (8 row slices in order, then the slices in order); skipped when neither is wanted.
constexpr int GN_SLICES = GN_THREADS / 32;
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_merge_kernel(const float* __restrict__ part, const float* __restrict__ gamma, float* __restrict__ ab,
                    float* __restrict__ dgamma, float* __restrict__ dbeta, int N, int C, int G, int S) {
  pdl_prologue();
  __shared__ float t1[1024], t2[1024];
  if (int(blockIdx.x) < N) {
    const int n = blockIdx.x;
    const float* src = part + size_t(n) * S * 2 * C;
    for (int c = threadIdx.x; c < C; c += GN_THREADS) {
      float a = 0.f, b = 0.f;
      for (int s = 0; s < S; ++s) {
        a += src[size_t(s) * 2 * C + c];
        b += src[size_t(s) * 2 * C + C + c];
      }
      t1[c] = gamma[c] * a;
      t2[c] = gamma[c] * b;
    }
    __syncthreads();
    const int cpg = C / G, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int g = warp; g < G; g += GN_THREADS / 32) {
      float a = 0.f, b = 0.f;
      for (int i = lane; i < cpg; i += 32) {
        a += t1[g * cpg + i];
        b += t2[g * cpg + i];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
      }
      if (lane == 0) {
        ab[size_t(n) * G + g] = a;
        ab[size_t(N) * G + size_t(n) * G + g] = b;
      }
    }
    return;
  }
  const int c = (blockIdx.x - N) * 32 + (threadIdx.x & 31), slice = threadIdx.x >> 5;
  const int R = N * S, r_lo = int((long long)slice * R / GN_SLICES), r_hi = int((long long)(slice + 1) * R / GN_SLICES);
  float a = 0.f, b = 0.f;
  if (c < C)
    for (int r = r_lo; r < r_hi; ++r) {
      a += part[size_t(r) * 2 * C + c];
      b += part[size_t(r) * 2 * C + C + c];
    }
  t1[threadIdx.x] = a;
  t2[threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.x < 32 && c < C) {
    a = t1[threadIdx.x];
    b = t2[threadIdx.x];
    for (int sl = 1; sl < GN_SLICES; ++sl) {
      a += t1[sl * 32 + threadIdx.x];
      b += t2[sl * 32 + threadIdx.x];
    }
    if (dbeta != nullptr) dbeta[c] = a;
    if (dgamma != nullptr) dgamma[c] = b;
  }
}

template <int MODE>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_apply_kernel(const float* __restrict__ dout, const float* __restrict__ out, const float* __restrict__ y,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                    const float* __restrict__ beta, const float* __restrict__ ab, float* __restrict__ dy,
                    float* __restrict__ dres, int N, int HW, int C, int G, int S) {
  pdl_prologue();
  const Slab b = slab(HW, C, S);
  if (b.r0 >= b.rpi) return;
  const int n = blockIdx.y, cpg = C / G;
  const GnCoef k = gn_coef(mean, rstd, gamma, beta, n, b.cq, C, G);
  // dy = ca du + cx xhat + cc, xhat = (y - mean) rstd
  float ca[4], cx[4], cc[4];
  const float invM = 1.f / (float(HW) * float(cpg));
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int g = (b.cq * 4 + j) / cpg;
    const float A = ab[size_t(n) * G + g], B = ab[size_t(N) * G + size_t(n) * G + g];
    ca[j] = k.rs[j] * k.ga[j];
    cx[j] = -k.rs[j] * B * invM;
    cc[j] = -k.rs[j] * A * invM;
  }
  const int step = b.rpi;
  for (int r = b.r0; r < b.len; r += 4 * step) {
    float4 d[4], o[4], v[4];
    size_t i[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) i[u] = b.base + size_t(r + u * step < b.len ? r + u * step : r) * b.q + b.cq;
#pragma unroll
    for (int u = 0; u < 4; ++u) d[u] = ld4(dout, i[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld4(y, i[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) o[u] = MODE == 1 ? ld4(out, i[u]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r + u * step >= b.len) continue;
      float dd[4], oo[4], vv[4], g4[4];
      to4(dd, d[u]); to4(oo, o[u]); to4(vv, v[u]);
      gn_du<MODE>(dd, oo, vv, k);
#pragma unroll
      for (int j = 0; j < 4; ++j) g4[j] = fmaf(ca[j], dd[j], fmaf(cx[j], (vv[j] - k.mu[j]) * k.rs[j], cc[j]));
      st4(dy, i[u], make_float4(g4[0], g4[1], g4[2], g4[3]));
      if (dres != nullptr) st4(dres, i[u], make_float4(dd[0], dd[1], dd[2], dd[3]));
    }
  }
}

void check_shape(const char* name, int N, int HW, int C, int G) {
  if (N < 1 || HW < 1 || (C & 3) || C < 4 || C > 1024 || G < 1 || G > 256 || C % G)
    throw std::runtime_error(std::string("fedb200: ") + name + " needs N, HW >= 1, C % 4 == 0, 4 <= C <= 1024 and G | C, "
                             "G <= 256");
}

int bwd_mode(const float* out, const float* beta, int act) {
  if (!act) return 0;
  if (out != nullptr) return 1;
  if (beta == nullptr) throw std::runtime_error("fedb200: gn_elu_bwd needs either the layer output or beta");
  return 2;
}

}  // namespace

int gn_splits(int N, int HW, int C) {
  // enough (split, sample) blocks for ~4 per SM, and at least four rows per thread in every split
  const int rpi = GN_THREADS / (C >> 2);
  int most = HW / (4 * rpi);
  if (most < 1) most = 1;
  int s = (4 * sm_count() + N - 1) / N;
  if (s > most) s = most;
  return s < 1 ? 1 : s;
}

void gn_elu_fwd(const float* y, const float* gamma, const float* beta, const float* residual, float* out, float* mean,
                float* rstd, float* part, float* table, int N, int HW, int C, int G, float eps, int act, cudaStream_t s) {
  check_shape("gn_elu_fwd", N, HW, C, G);
  const int S = gn_splits(N, HW, C);
  launch_pdl(gn_stats_kernel, dim3(S, N), dim3(GN_THREADS), 0, s, y, part, HW, C, S);
  check_launch("gn_stats");
  launch_pdl(gn_finalize_kernel, dim3(N), dim3(GN_THREADS), 0, s, part, gamma, beta, mean, rstd, table, HW, C, G, S, eps);
  check_launch("gn_finalize");
  launch_pdl(gn_apply_kernel, dim3(S, N), dim3(GN_THREADS), 0, s, y, table, residual, out, HW, C, S, act);
  check_launch("gn_apply");
}

void gn_elu_bwd(const float* dout, const float* out, const float* y, const float* mean, const float* rstd, const float* gamma,
                const float* beta, float* part, float* ab, float* dy, float* dres, float* dgamma, float* dbeta, int N, int HW,
                int C, int G, int act, cudaStream_t s) {
  check_shape("gn_elu_bwd", N, HW, C, G);
  const int S = gn_splits(N, HW, C);
  const int mode = bwd_mode(out, beta, act);
  const dim3 grid(S, N);
  switch (mode) {
    case 0: launch_pdl(gn_bwd_reduce_kernel<0>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, part, HW, C, G, S); break;
    case 1: launch_pdl(gn_bwd_reduce_kernel<1>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, part, HW, C, G, S); break;
    default: launch_pdl(gn_bwd_reduce_kernel<2>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, part, HW, C, G, S); break;
  }
  check_launch("gn_bwd_reduce");
  const int cblocks = (dgamma != nullptr || dbeta != nullptr) ? (C + 31) / 32 : 0;
  launch_pdl(gn_bwd_merge_kernel, dim3(N + cblocks), dim3(GN_THREADS), 0, s, part, gamma, ab, dgamma, dbeta, N, C, G, S);
  check_launch("gn_bwd_merge");
  switch (mode) {
    case 0: launch_pdl(gn_bwd_apply_kernel<0>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, ab, dy, dres, N, HW, C, G, S); break;
    case 1: launch_pdl(gn_bwd_apply_kernel<1>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, ab, dy, dres, N, HW, C, G, S); break;
    default: launch_pdl(gn_bwd_apply_kernel<2>, grid, dim3(GN_THREADS), 0, s, dout, out, y, mean, rstd, gamma, beta, ab, dy, dres, N, HW, C, G, S); break;
  }
  check_launch("gn_bwd_apply");
}

}  // namespace fedb200

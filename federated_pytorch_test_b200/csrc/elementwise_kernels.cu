// Memory-bound fused elementwise kernels of the ResNet path (SURVEY G2-G4, G22): all NHWC fp32,
// 128-bit accesses along the channel axis, per-channel parameters staged in shared memory.
//  * normalize_u8_nhwc : uint8 NHWC pixels -> (x/255-mean)/std as NHWC (optionally padded to 4 channels) or NCHW
//  * col_stats        : per-channel sum / sum of squares (only for layers whose conv did not emit them)
//  * bn_elu_fwd        : BatchNorm(batch stats from the conv epilogue) + residual + ELU in ONE pass; block 0 also
//                        updates the running statistics and stores mean/invstd for the backward pass
//  * bn_elu_bwd_reduce / bn_elu_bwd_apply : the two passes of the fused ELU'+BN backward
//  * avgpool_nhwc (+bwd), weight_krsc_flip (dgrad weights: swap Cin/Cout, rotate taps by 180 degrees)
#include "fedb200.h"

#include <cstdlib>

#include <cooperative_groups.h>
#include <stdexcept>
#include <string>

namespace cg = cooperative_groups;

namespace fedb200 {

static inline void check_launch(const char* name) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: ") + name + ": " + cudaGetErrorString(e));
  count_launch();
}
static int sm_count() {
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
// d ELU(u)/du expressed through the output o = ELU(u):  u > 0 <=> o > 0;  u <= 0 => exp(u) = o + 1
__device__ __forceinline__ float elu_grad_from_out(float o) { return o > 0.f ? 1.f : (o + 1.f); }

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
normalize_u8_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int npix, int c_out, float m0, float m1,
                    float m2, float s0, float s1, float s2, int to_nchw, int HW) {
  const float sc[3] = {1.f / (255.f * s0), 1.f / (255.f * s1), 1.f / (255.f * s2)};
  const float sh[3] = {-m0 / s0, -m1 / s1, -m2 / s2};
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += gridDim.x * blockDim.x) {
    const uint8_t* px = in + size_t(p) * 3;
    const float v0 = fmaf(float(px[0]), sc[0], sh[0]);
    const float v1 = fmaf(float(px[1]), sc[1], sh[1]);
    const float v2 = fmaf(float(px[2]), sc[2], sh[2]);
    if (to_nchw) {
      const int n = p / HW, r = p - n * HW;
      float* o = out + size_t(n) * 3 * HW + r;
      o[0] = v0;
      o[HW] = v1;
      o[2 * HW] = v2;
    } else if (c_out == 4) {
      reinterpret_cast<float4*>(out)[p] = make_float4(v0, v1, v2, 0.f);
    } else {
      float* o = out + size_t(p) * 3;
      o[0] = v0;
      o[1] = v1;
      o[2] = v2;
    }
  }
}
void normalize_u8_nhwc(const uint8_t* in, float* out, int npix, int c_out, const float* mean3, const float* std3,
                       int to_nchw, int H, int W, cudaStream_t s) {
  int grid = (npix + 255) / 256;
  if (grid > sm_count() * 16) grid = sm_count() * 16;
  normalize_u8_kernel<<<grid, 256, 0, s>>>(in, out, npix, c_out, mean3[0], mean3[1], mean3[2], std3[0], std3[1],
                                           std3[2], to_nchw, H * W);
  check_launch("normalize_u8");
}

// ------------------------------------------------------------------------------------------------
// Thread layout for [M, C] tensors with C % 4 == 0 (q = C/4 channel quads): thread t owns quad (t % q) for the rows
// (t / q) + k * rows_per_iter.  Consecutive threads touch consecutive 16-B words of a row, a thread's per-channel
// parameters live in REGISTERS for the whole kernel (no per-element modulo, no shared-memory parameter reads), and
// every loop keeps four independent 16-B loads per tensor in flight.
//
// Reductions end in atomicAdds on a [2C] vector that spans only a few 128-B lines, i.e. a few L2 slices: with ~600
// blocks the ~10^5 same-line atomics, not the streaming, would set the kernel time.  The reduction kernels therefore run at
// most two 512-thread blocks per SM.
// ------------------------------------------------------------------------------------------------
constexpr int EW_THREADS = 256;
constexpr int RED_THREADS = 512;

struct RowLayout {
  int q, cq, r0, rpi;
};
__device__ __forceinline__ RowLayout row_layout(int C, int threads) {
  RowLayout L;
  L.q = C >> 2;
  if ((L.q & (L.q - 1)) == 0) {
    const int sh = 31 - __clz(L.q);
    L.cq = threadIdx.x & (L.q - 1);
    L.r0 = threadIdx.x >> sh;
    L.rpi = threads >> sh;
  } else {
    L.cq = threadIdx.x % L.q;
    L.r0 = threadIdx.x / L.q;
    L.rpi = threads / L.q;
  }
  return L;
}
__device__ __forceinline__ float4 ld4(const float* p, size_t row, int q, int cq) {
  return reinterpret_cast<const float4*>(p)[row * q + cq];
}
__device__ __forceinline__ void st4(float* p, size_t row, int q, int cq, float4 v) {
  reinterpret_cast<float4*>(p)[row * q + cq] = v;
}
// block-wide reduction of per-thread channel-quad partials (s1, s2) over the rows of the block, then one atomicAdd
// per channel and block
__device__ __forceinline__ void block_quad_reduce(const float (&s1)[4], const float (&s2)[4], float* sm, const RowLayout& L,
                                                  float* out1, float* out2) {
  const int T = blockDim.x;
  float* a = sm + threadIdx.x * 4;
  float* b = sm + T * 4 + threadIdx.x * 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) { a[j] = s1[j]; b[j] = s2[j]; }
  __syncthreads();
  // threads [0, 2q): the first q sum s1 of their quad over the block's rows, the next q sum s2
  if (threadIdx.x < 2 * L.q) {
    const int which = threadIdx.x >= L.q;
    const int quad = threadIdx.x - which * L.q;
    const float* base = sm + which * T * 4 + quad * 4;
    float t[4] = {0, 0, 0, 0};
    for (int rr = 0; rr < L.rpi; ++rr) {
      const float4 v = *reinterpret_cast<const float4*>(base + rr * L.q * 4);
      t[0] += v.x; t[1] += v.y; t[2] += v.z; t[3] += v.w;
    }
    // one 16-B vector reduction per channel quad (resolved at L2, no return value)
    float* dst = (which ? out2 : out1) + quad * 4;
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(t[0]), "f"(t[1]), "f"(t[2]), "f"(t[3]) : "memory");
  }
}
static int reduce_rows_per_thread() {
  static int rows = -1;
  if (rows < 0) {
    const char* v = std::getenv("FEDB200_RED_ROWS");
    rows = (v != nullptr && std::atoi(v) > 0) ? std::atoi(v) : 4;
  }
  return rows;
}
static int reduce_grid(int M, int rpi) {
  // One block of four rows in flight per thread, at most two CTAs per SM.  The first version asked for >= 16 rows per thread (few
  // blocks => few same-line atomics), which left the small tensors on 32-64 CTAs, far too few to stream them at DRAM speed.
  // FEDB200_RED_ROWS=16: old grid.
  const int rows = reduce_rows_per_thread();
  int grid = (M + rpi * rows - 1) / (rpi * rows);
  if (grid > sm_count() * 2) grid = sm_count() * 2;
  return grid < 1 ? 1 : grid;
}
static int stream_grid(int M, int rpi) {
  int grid = (M + rpi * 4 - 1) / (rpi * 4);
  if (grid > sm_count() * 8) grid = sm_count() * 8;
  return grid < 1 ? 1 : grid;
}

__global__ void __launch_bounds__(RED_THREADS)
col_stats_kernel(const float* __restrict__ y, float* __restrict__ stats, int M, int C) {
  pdl_prologue();
  extern __shared__ float sm[];                   // [2][RED_THREADS][4]
  const RowLayout L = row_layout(C, RED_THREADS);
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  if (L.r0 < L.rpi) {
    const int step = gridDim.x * L.rpi;
    // always four rows in flight; rows past the end re-read row r and are masked out
    for (int r = blockIdx.x * L.rpi + L.r0; r < M; r += 4 * step) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld4(y, size_t(r + u * step < M ? r + u * step : r), L.q, L.cq);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + u * step >= M) v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        s1[0] += v[u].x; s1[1] += v[u].y; s1[2] += v[u].z; s1[3] += v[u].w;
        s2[0] = fmaf(v[u].x, v[u].x, s2[0]); s2[1] = fmaf(v[u].y, v[u].y, s2[1]);
        s2[2] = fmaf(v[u].z, v[u].z, s2[2]); s2[3] = fmaf(v[u].w, v[u].w, s2[3]);
      }
    }
  }
  block_quad_reduce(s1, s2, sm, L, stats, stats + C);
}
void col_stats(const float* y, float* stats, int M, int C, cudaStream_t s) {
  if ((C & 3) || C > 2 * RED_THREADS) throw std::runtime_error("fedb200: col_stats needs C % 4 == 0 and C <= 1024");
  const int rpi = RED_THREADS / (C >> 2);
  launch_pdl(col_stats_kernel, dim3(reduce_grid(M, rpi)), dim3(RED_THREADS), 2 * RED_THREADS * 4 * sizeof(float), s, y, stats, M, C);
  check_launch("col_stats");
}

__global__ void __launch_bounds__(EW_THREADS)
bn_elu_fwd_kernel(const float* __restrict__ y, float* __restrict__ stats, const float* __restrict__ gamma,
                  const float* __restrict__ beta, const float* __restrict__ residual, float* __restrict__ out,
                  float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ save_mean,
                  float* __restrict__ save_invstd, int M, int C, float eps, float momentum, int act, int self_clean) {
  pdl_prologue();
  __shared__ int last_block;
  const RowLayout L = row_layout(C, EW_THREADS);
  const bool active = L.r0 < L.rpi;
  float sc[4] = {0, 0, 0, 0}, sh[4] = {0, 0, 0, 0};
  if (active) {
    const float invM = 1.f / float(M);
    const float4 s1 = reinterpret_cast<const float4*>(stats)[L.cq];
    const float4 s2 = reinterpret_cast<const float4*>(stats + C)[L.cq];
    const float4 g = reinterpret_cast<const float4*>(gamma)[L.cq];
    const float4 b = reinterpret_cast<const float4*>(beta)[L.cq];
    const float a1[4] = {s1.x, s1.y, s1.z, s1.w}, a2[4] = {s2.x, s2.y, s2.z, s2.w};
    const float gg[4] = {g.x, g.y, g.z, g.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float mean = a1[j] * invM;
      float var = fmaf(-mean, mean, a2[j] * invM);
      var = var > 0.f ? var : 0.f;
      const float invstd = rsqrtf(var + eps);
      sc[j] = gg[j] * invstd;
      sh[j] = fmaf(-mean, sc[j], bb[j]);
      if (blockIdx.x == 0 && L.r0 == 0) {
        const int c = L.cq * 4 + j;
        save_mean[c] = mean;
        save_invstd[c] = invstd;
        if (running_mean != nullptr) {
          const float unbiased = M > 1 ? var * float(M) / float(M - 1) : var;
          running_mean[c] = fmaf(momentum, mean - running_mean[c], running_mean[c]);
          running_var[c] = fmaf(momentum, unbiased - running_var[c], running_var[c]);
        }
      }
    }
  }
  if (self_clean) {
    // Every thread of this block has consumed the statistics.  The last block to say so zeroes the accumulators (and
    // the counter behind them) for the next convolution that uses this buffer: no memset launch per layer.
    __syncthreads();
    unsigned int* counter = reinterpret_cast<unsigned int*>(stats + 2 * C);
    if (threadIdx.x == 0) {
      __threadfence();
      last_block = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last_block) {
      for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) stats[c] = 0.f;
      if (threadIdx.x == 0) *counter = 0u;
    }
  }
  if (!active) return;
  const int step = gridDim.x * L.rpi;
  auto apply = [&](float4 v, float4 r) {
    float4 o = make_float4(fmaf(v.x, sc[0], sh[0]) + r.x, fmaf(v.y, sc[1], sh[1]) + r.y, fmaf(v.z, sc[2], sh[2]) + r.z,
                           fmaf(v.w, sc[3], sh[3]) + r.w);
    if (act) { o.x = elu_f(o.x); o.y = elu_f(o.y); o.z = elu_f(o.z); o.w = elu_f(o.w); }
    return o;
  };
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = blockIdx.x * L.rpi + L.r0; r < M; r += 4 * step) {
    float4 v[4], rs[4];
    size_t row[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) row[u] = size_t(r + u * step < M ? r + u * step : r);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld4(y, row[u], L.q, L.cq);
#pragma unroll
    for (int u = 0; u < 4; ++u) rs[u] = residual != nullptr ? ld4(residual, row[u], L.q, L.cq) : zero;
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (r + u * step < M) st4(out, row[u], L.q, L.cq, apply(v[u], rs[u]));
  }
}
void bn_elu_fwd(const float* y, float* stats, const float* gamma, const float* beta, const float* residual,
                float* out, float* running_mean, float* running_var, float* save_mean, float* save_invstd, int M, int C,
                float eps, float momentum, int act, int self_clean, cudaStream_t s) {
  if ((C & 3) || C > 4 * EW_THREADS) throw std::runtime_error("fedb200: bn_elu_fwd needs C % 4 == 0 and C <= 1024");
  const int rpi = EW_THREADS / (C >> 2);
  launch_pdl(bn_elu_fwd_kernel, dim3(stream_grid(M, rpi)), dim3(EW_THREADS), 0, s, y, stats, gamma, beta, residual, out, running_mean,
                                                                running_var, save_mean, save_invstd, M, C, eps, momentum,
                                                                act, self_clean);
  check_launch("bn_elu_fwd");
}

// du = dout * ELU'(z).  With the layer output at hand ELU' comes from it (z > 0 <=> out > 0, exp(z) = out + 1); when
// the layer had no residual input, z = y * scale + shift is recomputed instead and `out` is never read (one tensor
// pass less in each of the two backward kernels).
struct BnBwdCoef {
  float mu[4], is[4], sc[4], sh[4];
};
__device__ __forceinline__ BnBwdCoef bn_bwd_coef(const float* mean, const float* invstd, const float* gamma, const float* beta,
                                                 int cq) {
  BnBwdCoef k;
  const float4 m = reinterpret_cast<const float4*>(mean)[cq], i = reinterpret_cast<const float4*>(invstd)[cq];
  const float4 g = reinterpret_cast<const float4*>(gamma)[cq];
  const float4 b = beta != nullptr ? reinterpret_cast<const float4*>(beta)[cq] : make_float4(0.f, 0.f, 0.f, 0.f);
  k.mu[0] = m.x; k.mu[1] = m.y; k.mu[2] = m.z; k.mu[3] = m.w;
  k.is[0] = i.x; k.is[1] = i.y; k.is[2] = i.z; k.is[3] = i.w;
  const float gg[4] = {g.x, g.y, g.z, g.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    k.sc[j] = gg[j] * k.is[j];
    k.sh[j] = fmaf(-k.mu[j], k.sc[j], bb[j]);
  }
  return k;
}
template <int MODE>   // 0: no activation, 1: ELU' from out, 2: ELU' recomputed from y
__device__ __forceinline__ float4 bn_du(float4 d, float4 o, float4 v, const BnBwdCoef& k) {
  if (MODE == 1) {
    d.x *= elu_grad_from_out(o.x); d.y *= elu_grad_from_out(o.y); d.z *= elu_grad_from_out(o.z); d.w *= elu_grad_from_out(o.w);
  } else if (MODE == 2) {
    const float z0 = fmaf(v.x, k.sc[0], k.sh[0]), z1 = fmaf(v.y, k.sc[1], k.sh[1]);
    const float z2 = fmaf(v.z, k.sc[2], k.sh[2]), z3 = fmaf(v.w, k.sc[3], k.sh[3]);
    d.x *= z0 > 0.f ? 1.f : __expf(z0); d.y *= z1 > 0.f ? 1.f : __expf(z1);
    d.z *= z2 > 0.f ? 1.f : __expf(z2); d.w *= z3 > 0.f ? 1.f : __expf(z3);
  }
  return d;
}

// backward pass 1: sums[c] = sum_rows du, sums[C+c] = sum_rows du * xhat
template <int MODE>
__global__ void __launch_bounds__(RED_THREADS)
bn_elu_bwd_reduce_kernel(const float* __restrict__ dout, const float* __restrict__ out, const float* __restrict__ y,
                         const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float* __restrict__ sums, int M, int C) {
  pdl_prologue();
  extern __shared__ float sm[];
  const RowLayout L = row_layout(C, RED_THREADS);
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  if (L.r0 < L.rpi) {
    const BnBwdCoef k = bn_bwd_coef(mean, invstd, gamma, beta, L.cq);
    const int step = gridDim.x * L.rpi;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    auto acc = [&](float4 d, float4 v) {
      s1[0] += d.x; s1[1] += d.y; s1[2] += d.z; s1[3] += d.w;
      s2[0] = fmaf(d.x, (v.x - k.mu[0]) * k.is[0], s2[0]); s2[1] = fmaf(d.y, (v.y - k.mu[1]) * k.is[1], s2[1]);
      s2[2] = fmaf(d.z, (v.z - k.mu[2]) * k.is[2], s2[2]); s2[3] = fmaf(d.w, (v.w - k.mu[3]) * k.is[3], s2[3]);
    };
    for (int r = blockIdx.x * L.rpi + L.r0; r < M; r += 4 * step) {
      float4 d[4], o[4], v[4];
      size_t row[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) row[u] = size_t(r + u * step < M ? r + u * step : r);
#pragma unroll
      for (int u = 0; u < 4; ++u) d[u] = ld4(dout, row[u], L.q, L.cq);
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = ld4(y, row[u], L.q, L.cq);
#pragma unroll
      for (int u = 0; u < 4; ++u) o[u] = MODE == 1 ? ld4(out, row[u], L.q, L.cq) : zero;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + u * step >= M) d[u] = zero;                 // masked row: contributes nothing
        acc(bn_du<MODE>(d[u], o[u], v[u], k), v[u]);
      }
    }
  }
  block_quad_reduce(s1, s2, sm, L, sums, sums + C);
}
static int bwd_mode(const float* out, const float* beta, int act) {
  if (!act) return 0;
  if (out != nullptr) return 1;
  if (beta == nullptr) throw std::runtime_error("fedb200: bn_elu_bwd needs either the layer output or beta");
  return 2;
}
void bn_elu_bwd_reduce(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                       const float* gamma, const float* beta, float* sums, int M, int C, int act, int sums_clean, cudaStream_t s) {
  if ((C & 3) || C > 2 * RED_THREADS) throw std::runtime_error("fedb200: bn_elu_bwd needs C % 4 == 0 and C <= 1024");
  if (!sums_clean) cudaMemsetAsync(sums, 0, 2 * C * sizeof(float), s);     // a self-cleaning per-layer buffer arrives zeroed
  const int rpi = RED_THREADS / (C >> 2);
  const int grid = reduce_grid(M, rpi);
  const size_t smem = 2 * RED_THREADS * 4 * sizeof(float);
  switch (bwd_mode(out, beta, act)) {
    case 0: launch_pdl(bn_elu_bwd_reduce_kernel<0>, dim3(grid), dim3(RED_THREADS), smem, s, dout, out, y, mean, invstd, gamma, beta, sums, M, C); break;
    case 1: launch_pdl(bn_elu_bwd_reduce_kernel<1>, dim3(grid), dim3(RED_THREADS), smem, s, dout, out, y, mean, invstd, gamma, beta, sums, M, C); break;
    default: launch_pdl(bn_elu_bwd_reduce_kernel<2>, dim3(grid), dim3(RED_THREADS), smem, s, dout, out, y, mean, invstd, gamma, beta, sums, M, C); break;
  }
  check_launch("bn_elu_bwd_reduce");
}

// backward pass 2: dy = gamma*invstd*(du - sum_du/M - xhat*sum_du_xhat/M); dres = du; dgamma/dbeta from sums.
// Rows are visited from the END of the tensor: pass 1 has just streamed dout/y/out front to back, so their tails are
// what the L2 (50 MB on an H100) still holds.
template <int MODE>
__global__ void __launch_bounds__(EW_THREADS)
bn_elu_bwd_apply_kernel(const float* __restrict__ dout, const float* __restrict__ out, const float* __restrict__ y,
                        const float* __restrict__ mean, const float* __restrict__ invstd,
                        const float* __restrict__ gamma, const float* __restrict__ beta, float* sums,
                        float* __restrict__ dy, float* __restrict__ dres, float* __restrict__ dgamma,
                        float* __restrict__ dbeta, int M, int C, int self_clean) {
  pdl_prologue();
  __shared__ int s_last;
  const RowLayout L = row_layout(C, EW_THREADS);
  const bool active = L.r0 < L.rpi;
  BnBwdCoef k;
  float ca[4], cb[4], cc[4];                      // dy = ca*du + cb*y + cc  (affine in du, y)
  if (active) {
    k = bn_bwd_coef(mean, invstd, gamma, beta, L.cq);
    const float invM = 1.f / float(M);
    const float4 a = reinterpret_cast<const float4*>(sums)[L.cq], b = reinterpret_cast<const float4*>(sums + C)[L.cq];
    const float4 g = reinterpret_cast<const float4*>(gamma)[L.cq];
    const float sdu[4] = {a.x, a.y, a.z, a.w}, sdx[4] = {b.x, b.y, b.z, b.w}, gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float kk = gg[j] * k.is[j];
      ca[j] = kk;
      cb[j] = -kk * k.is[j] * sdx[j] * invM;
      cc[j] = -kk * sdu[j] * invM + kk * k.is[j] * sdx[j] * invM * k.mu[j];
      if (blockIdx.x == 0 && L.r0 == 0) {
        if (dgamma != nullptr) dgamma[L.cq * 4 + j] += sdx[j];
        if (dbeta != nullptr) dbeta[L.cq * 4 + j] += sdu[j];
      }
    }
  }
  if (self_clean) {
    // `sums` = [sum du | sum du*xhat | counter] is a per-layer buffer that stays allocated: the last CTA to have read it
    // re-zeroes it for the next backward pass (no memset node per BatchNorm layer in the captured step).
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned int t = atomicAdd(reinterpret_cast<unsigned int*>(sums + 2 * C), 1u);
      s_last = (t == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
      for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sums[c] = 0.f;
      if (threadIdx.x == 0) *reinterpret_cast<unsigned int*>(sums + 2 * C) = 0u;
    }
  }
  if (!active) return;
  const int step = gridDim.x * L.rpi;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  auto emit = [&](size_t row, float4 d, float4 v) {
    st4(dy, row, L.q, L.cq, make_float4(fmaf(ca[0], d.x, fmaf(cb[0], v.x, cc[0])), fmaf(ca[1], d.y, fmaf(cb[1], v.y, cc[1])),
                                        fmaf(ca[2], d.z, fmaf(cb[2], v.z, cc[2])), fmaf(ca[3], d.w, fmaf(cb[3], v.w, cc[3]))));
    if (dres != nullptr) st4(dres, row, L.q, L.cq, d);
  };
  for (int r = blockIdx.x * L.rpi + L.r0; r < M; r += 4 * step) {
    float4 d[4], o[4], v[4];
    size_t row[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) row[u] = size_t(M - 1 - (r + u * step < M ? r + u * step : r));
#pragma unroll
    for (int u = 0; u < 4; ++u) d[u] = ld4(dout, row[u], L.q, L.cq);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld4(y, row[u], L.q, L.cq);
#pragma unroll
    for (int u = 0; u < 4; ++u) o[u] = MODE == 1 ? ld4(out, row[u], L.q, L.cq) : zero;
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (r + u * step < M) emit(row[u], bn_du<MODE>(d[u], o[u], v[u], k), v[u]);
  }
}
void bn_elu_bwd_apply(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, float* sums, float* dy, float* dres, float* dgamma,
                      float* dbeta, int M, int C, int act, int self_clean, cudaStream_t s) {
  if ((C & 3) || C > 4 * EW_THREADS) throw std::runtime_error("fedb200: bn_elu_bwd needs C % 4 == 0 and C <= 1024");
  const int rpi = EW_THREADS / (C >> 2);
  const int grid = stream_grid(M, rpi);
  switch (bwd_mode(out, beta, act)) {
    case 0: launch_pdl(bn_elu_bwd_apply_kernel<0>, dim3(grid), dim3(EW_THREADS), 0, s, dout, out, y, mean, invstd, gamma, beta, sums, dy, dres, dgamma, dbeta, M, C, self_clean); break;
    case 1: launch_pdl(bn_elu_bwd_apply_kernel<1>, dim3(grid), dim3(EW_THREADS), 0, s, dout, out, y, mean, invstd, gamma, beta, sums, dy, dres, dgamma, dbeta, M, C, self_clean); break;
    default: launch_pdl(bn_elu_bwd_apply_kernel<2>, dim3(grid), dim3(EW_THREADS), 0, s, dout, out, y, mean, invstd, gamma, beta, sums, dy, dres, dgamma, dbeta, M, C, self_clean); break;
  }
  check_launch("bn_elu_bwd_apply");
}

// ------------------------------------------------------------------------------------------------
// EXPERIMENTAL (opt-in, FEDB200_BN_BWD_FUSED=1): both passes of the
// BN(+ELU) backward in ONE cooperative kernel for the small layers (layer3 / layer4: 8 / 4 MB per tensor).  The two-pass
// version costs a memset + 2 launches and reads every tensor twice; here each
// thread keeps its <= MAXR rows of du and y in registers across a grid barrier, so the tensors are read once.
// Requires gridDim.x * rows_per_iter * MAXR >= M with all blocks co-resident (cooperative launch).
// ------------------------------------------------------------------------------------------------
template <int MODE, int MAXR>
__global__ void __launch_bounds__(RED_THREADS)
bn_elu_bwd_fused_kernel(const float* __restrict__ dout, const float* __restrict__ out, const float* __restrict__ y,
                        const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
                        const float* __restrict__ beta, float* __restrict__ sums, float* __restrict__ dy,
                        float* __restrict__ dres, float* __restrict__ dgamma, float* __restrict__ dbeta, int M, int C) {
  extern __shared__ float sm[];
  cg::grid_group grid = cg::this_grid();
  const RowLayout L = row_layout(C, RED_THREADS);
  const bool active = L.r0 < L.rpi;
  const int step = gridDim.x * L.rpi;
  const int r_first = blockIdx.x * L.rpi + L.r0;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 du[MAXR], v[MAXR];
  float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  BnBwdCoef k = {};
  if (active) {
    k = bn_bwd_coef(mean, invstd, gamma, beta, L.cq);
#pragma unroll
    for (int u = 0; u < MAXR; ++u) {
      const int r = r_first + u * step;
      const bool ok = r < M;
      const size_t row = size_t(ok ? r : r_first < M ? r_first : 0);
      const float4 d = ld4(dout, row, L.q, L.cq);
      v[u] = ld4(y, row, L.q, L.cq);
      const float4 o = MODE == 1 ? ld4(out, row, L.q, L.cq) : zero;
      du[u] = ok ? bn_du<MODE>(d, o, v[u], k) : zero;
      s1[0] += du[u].x; s1[1] += du[u].y; s1[2] += du[u].z; s1[3] += du[u].w;
      s2[0] = fmaf(du[u].x, (v[u].x - k.mu[0]) * k.is[0], s2[0]); s2[1] = fmaf(du[u].y, (v[u].y - k.mu[1]) * k.is[1], s2[1]);
      s2[2] = fmaf(du[u].z, (v[u].z - k.mu[2]) * k.is[2], s2[2]); s2[3] = fmaf(du[u].w, (v[u].w - k.mu[3]) * k.is[3], s2[3]);
    }
  }
  block_quad_reduce(s1, s2, sm, L, sums, sums + C);
  __threadfence();
  grid.sync();
  if (!active) return;
  float ca[4], cb[4], cc[4];
  {
    const float invM = 1.f / float(M);
    const float4 a = __ldcg(reinterpret_cast<const float4*>(sums) + L.cq);
    const float4 b = __ldcg(reinterpret_cast<const float4*>(sums + C) + L.cq);
    const float4 g = reinterpret_cast<const float4*>(gamma)[L.cq];
    const float sdu[4] = {a.x, a.y, a.z, a.w}, sdx[4] = {b.x, b.y, b.z, b.w}, gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float kk = gg[j] * k.is[j];
      ca[j] = kk;
      cb[j] = -kk * k.is[j] * sdx[j] * invM;
      cc[j] = -kk * sdu[j] * invM + kk * k.is[j] * sdx[j] * invM * k.mu[j];
      if (blockIdx.x == 0 && L.r0 == 0) {
        if (dgamma != nullptr) dgamma[L.cq * 4 + j] += sdx[j];
        if (dbeta != nullptr) dbeta[L.cq * 4 + j] += sdu[j];
      }
    }
  }
#pragma unroll
  for (int u = 0; u < MAXR; ++u) {
    const int r = r_first + u * step;
    if (r < M) {
      st4(dy, size_t(r), L.q, L.cq,
          make_float4(fmaf(ca[0], du[u].x, fmaf(cb[0], v[u].x, cc[0])), fmaf(ca[1], du[u].y, fmaf(cb[1], v[u].y, cc[1])),
                      fmaf(ca[2], du[u].z, fmaf(cb[2], v[u].z, cc[2])), fmaf(ca[3], du[u].w, fmaf(cb[3], v[u].w, cc[3]))));
      if (dres != nullptr) st4(dres, size_t(r), L.q, L.cq, du[u]);
    }
  }
}
// returns false (nothing launched) when the tensor does not fit the register-resident scheme
bool bn_elu_bwd_fused(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, float* sums, float* dy, float* dres, float* dgamma,
                      float* dbeta, int M, int C, int act, cudaStream_t s) {
  constexpr int MAXR = 8;
  if ((C & 3) || C > 2 * RED_THREADS) return false;
  const int rpi = RED_THREADS / (C >> 2);
  if (rpi < 1) return false;
  int grid = sm_count();
  const int need = (M + rpi - 1) / rpi;                 // row groups
  if (grid > need) grid = need;
  if ((need + grid - 1) / grid > MAXR) return false;
  cudaMemsetAsync(sums, 0, 2 * C * sizeof(float), s);
  const size_t smem = 2 * RED_THREADS * 4 * sizeof(float);
  void* args[] = {(void*)&dout, (void*)&out, (void*)&y, (void*)&mean, (void*)&invstd, (void*)&gamma, (void*)&beta,
                  (void*)&sums, (void*)&dy, (void*)&dres, (void*)&dgamma, (void*)&dbeta, (void*)&M, (void*)&C};
  const void* fn = nullptr;
  switch (bwd_mode(out, beta, act)) {
    case 0: fn = (const void*)bn_elu_bwd_fused_kernel<0, MAXR>; break;
    case 1: fn = (const void*)bn_elu_bwd_fused_kernel<1, MAXR>; break;
    default: fn = (const void*)bn_elu_bwd_fused_kernel<2, MAXR>; break;
  }
  cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(RED_THREADS), args, smem, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: bn_elu_bwd_fused: ") + cudaGetErrorString(e));
  count_launch();
  return true;
}

__global__ void __launch_bounds__(256)
avgpool_kernel(const float* __restrict__ x, float* __restrict__ out, int NB, int HW, int C) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over NB*C
  if (i >= NB * C) return;
  const int n = i / C, c = i - n * C;
  const float* p = x + size_t(n) * HW * C + c;
  float s = 0.f;
  for (int k = 0; k < HW; ++k) s += p[size_t(k) * C];
  out[i] = s / float(HW);
}
void avgpool_nhwc(const float* x, float* out, int NB, int HW, int C, cudaStream_t s) {
  launch_pdl(avgpool_kernel, dim3((NB * C + 255) / 256), dim3(256), 0, s, x, out, NB, HW, C);
  check_launch("avgpool_nhwc");
}
// ------------------------------------------------------------------------------------------------
// Fused classifier head (FEDB200_HEAD_FUSED=0 switches it off):
// avg_pool(window) -> flatten -> Linear in ONE true-fp32 kernel per direction (SURVEY G4 + G5, simple_models.py:213-216).
// The library path is an avgpool kernel + a SIMT sgemm for a 128x10x512 problem; here one block per sample pools
// its [HW, C] map into shared memory and eight warps produce the O <= 32 logits with FMA chains + shuffle reductions.
// ------------------------------------------------------------------------------------------------
constexpr int HEAD_THREADS = 256;
__global__ void __launch_bounds__(HEAD_THREADS)
head_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ pooled, float* __restrict__ logits, int HW, int C, int O) {
  extern __shared__ float sp[];                    // pooled[C]
  const int n = blockIdx.x;
  const float inv = 1.f / float(HW);
  const float* xn = x + size_t(n) * HW * C;
  for (int c = threadIdx.x; c < C; c += HEAD_THREADS) {
    float s = 0.f;
    for (int k = 0; k < HW; ++k) s += xn[size_t(k) * C + c];
    s *= inv;
    sp[c] = s;
    pooled[size_t(n) * C + c] = s;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = warp; o < O; o += HEAD_THREADS / 32) {
    const float* wo = w + size_t(o) * C;
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) acc = fmaf(sp[c], wo[c], acc);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) logits[size_t(n) * O + o] = acc + (bias != nullptr ? bias[o] : 0.f);
  }
}
// dx[n, k, c] = (1/HW) * sum_o dlogits[n, o] * w[o, c]
__global__ void __launch_bounds__(HEAD_THREADS)
head_bwd_kernel(const float* __restrict__ dlogits, const float* __restrict__ w, float* __restrict__ dx, int HW, int C,
                int O) {
  __shared__ float dl[32];
  const int n = blockIdx.x;
  if (threadIdx.x < O) dl[threadIdx.x] = dlogits[size_t(n) * O + threadIdx.x];
  __syncthreads();
  const float inv = 1.f / float(HW);
  float* dxn = dx + size_t(n) * HW * C;
  for (int c = threadIdx.x; c < C; c += HEAD_THREADS) {
    float g = 0.f;
    for (int o = 0; o < O; ++o) g = fmaf(dl[o], w[size_t(o) * C + c], g);
    g *= inv;
    for (int k = 0; k < HW; ++k) dxn[size_t(k) * C + c] = g;
  }
}
void head_fwd(const float* x, const float* w, const float* bias, float* pooled, float* logits, int NB, int HW, int C, int O,
              cudaStream_t s) {
  if (O > 32) throw std::runtime_error("fedb200: head_fwd supports at most 32 outputs");
  head_fwd_kernel<<<NB, HEAD_THREADS, C * sizeof(float), s>>>(x, w, bias, pooled, logits, HW, C, O);
  check_launch("head_fwd");
}
void head_bwd(const float* dlogits, const float* w, float* dx, int NB, int HW, int C, int O, cudaStream_t s) {
  if (O > 32) throw std::runtime_error("fedb200: head_bwd supports at most 32 outputs");
  head_bwd_kernel<<<NB, HEAD_THREADS, 0, s>>>(dlogits, w, dx, HW, C, O);
  check_launch("head_bwd");
}

__global__ void __launch_bounds__(256)
avgpool_bwd_kernel(const float* __restrict__ dout, float* __restrict__ dx, int NB, int HW, int C) {
  pdl_prologue();
  const size_t total = size_t(NB) * HW * C;
  const float inv = 1.f / float(HW);
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += size_t(gridDim.x) * blockDim.x) {
    const int c = int(i % C);
    const int n = int(i / (size_t(HW) * C));
    dx[i] = dout[size_t(n) * C + c] * inv;
  }
}
void avgpool_nhwc_bwd(const float* dout, float* dx, int NB, int HW, int C, cudaStream_t s) {
  const size_t total = size_t(NB) * HW * C;
  int grid = int((total + 1023) / 1024);
  if (grid > sm_count() * 8) grid = sm_count() * 8;
  launch_pdl(avgpool_bwd_kernel, dim3(grid), dim3(256), 0, s, dout, dx, NB, HW, C);
  check_launch("avgpool_nhwc_bwd");
}

// w: [C_out][kh][kw][C_in]  ->  out: [C_in][kh][kw][C_out] with taps rotated by 180 degrees
// (the stride-1 data gradient is a convolution of dY with these weights)
__global__ void __launch_bounds__(256)
weight_flip_kernel(const float* __restrict__ w, float* __restrict__ out, int C_out, int C_in, int kh, int kw) {
  pdl_prologue();
  const int taps = kh * kw;
  const size_t total = size_t(C_out) * taps * C_in;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += size_t(gridDim.x) * blockDim.x) {
    const int co = int(i % C_out);
    const int t = int((i / C_out) % taps);
    const int ci = int(i / (size_t(C_out) * taps));
    out[i] = w[(size_t(co) * taps + (taps - 1 - t)) * C_in + ci];
  }
}
void weight_krsc_flip(const float* w, float* out, int C_out, int C_in, int kh, int kw, cudaStream_t s) {
  const size_t total = size_t(C_out) * kh * kw * C_in;
  int grid = int((total + 255) / 256);
  if (grid > sm_count() * 8) grid = sm_count() * 8;
  launch_pdl(weight_flip_kernel, dim3(grid), dim3(256), 0, s, w, out, C_out, C_in, kh, kw);
  check_launch("weight_krsc_flip");
}

// ConvTranspose2d(k = 4, stride 2, padding 1) weight [Ci, Co, 4, 4] (any strides) -> KRSC filter [4 * Co, 3, 3, Ci] of the equivalent
// 3x3 / pad 1 convolution with phase-major output channels (ops/conv_math.py::pack_convT_s2_weight: output phase ph takes filter
// rows 3, 1 at window positions 0, 1 and phase 1 rows 2, 0 at positions 1, 2; the other position is zero).  One launch instead
// of a 36-way torch.stack per transposed convolution and step.
__device__ __forceinline__ int convT_tap(int phase, int t) {
  return phase == 0 ? (t == 0 ? 3 : (t == 1 ? 1 : -1)) : (t == 0 ? -1 : (t == 1 ? 2 : 0));
}
__global__ void __launch_bounds__(256)
convT_pack_kernel(const float* __restrict__ w, float* __restrict__ out, int Ci, int Co, long long s_ci, long long s_co, long long s_r,
                  long long s_s) {
  pdl_prologue();
  const size_t total = size_t(4) * Co * 9 * Ci;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += size_t(gridDim.x) * blockDim.x) {
    const int ci = int(i % Ci);
    size_t t = i / Ci;
    const int ts = int(t % 3);
    t /= 3;
    const int tr = int(t % 3);
    t /= 3;
    const int co = int(t % Co);
    const int phase = int(t / Co);
    const int r = convT_tap(phase >> 1, tr), sx = convT_tap(phase & 1, ts);
    out[i] = (r >= 0 && sx >= 0) ? w[ci * s_ci + co * s_co + r * s_r + sx * s_s] : 0.f;
  }
}
void convT_pack(const float* w, float* out, int Ci, int Co, long long s_ci, long long s_co, long long s_r, long long s_s, cudaStream_t s) {
  const size_t total = size_t(4) * Co * 9 * Ci;
  int grid = int((total + 255) / 256);
  if (grid > sm_count() * 8) grid = sm_count() * 8;
  launch_pdl(convT_pack_kernel, dim3(grid), dim3(256), 0, s, w, out, Ci, Co, s_ci, s_co, s_r, s_s);
  check_launch("convT_pack");
}

}  // namespace fedb200

// Level-1 kernels over flat parameter blocks (SURVEY G14-G16, G20).
//  * adam_prox_kernel    : Adam update with the FedProx / augmented-Lagrangian / elastic-net gradient folded in
//  * l1_l2, make_pair, welford, penalty_value, penalty_grad, multi_dot : one pass + in-kernel reductions,
//    results stay on the device (callers read several scalars with ONE D2H copy)
//  * lbfgs_two_loop_kernel: the whole two-loop recursion (2k+2 dependent passes) as ONE cooperative persistent
//    kernel with a software grid barrier — no host round trips between the dependent dot products.
// Memory-bound: every kernel streams each vector once with 128-bit accesses; reductions are
// warp-shuffle -> shared -> one atomicAdd per block.
#include "fedb200.h"

#include <cstdlib>

#include <cooperative_groups.h>
#include <atomic>
#include <stdexcept>
#include <string>

namespace cg = cooperative_groups;

namespace fedb200 {

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches += n; }
long long launch_count() { return g_launches.load(); }
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = std::getenv("FEDB200_PDL");
    v = (e != nullptr && std::atoi(e) != 0) ? 1 : 0;   // opt-in: inside a captured step the launch gaps are already hidden
  }
  return v == 1;
}

static inline void check_launch(const char* name) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: ") + name + ": " + cudaGetErrorString(e));
  count_launch();
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}
static inline int grid_for(int n, int per_thread = 4, int threads = 256, int waves = 8) {
  long long blocks = (static_cast<long long>(n) + threads * per_thread - 1) / (threads * per_thread);
  long long cap = static_cast<long long>(num_sms()) * waves;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks < cap ? blocks : cap);
}

__device__ __forceinline__ float warp_red(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Block-wide sum of NV values per thread; result valid in thread 0.
template <int NV>
__device__ __forceinline__ void block_reduce(float (&v)[NV], float* sm /* [NV*32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_red(v[i]);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) sm[i * 32 + warp] = v[i];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float x = lane < nw ? sm[i * 32 + lane] : 0.f;
      v[i] = warp_red(x);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float sgnf(float x) { return (x > 0.f) - (x < 0.f); }

// ------------------------------------------------------------------------------------------------
__global__ void bump_step_kernel(int* step) { *step += 1; }

void bump_step(int* step_dev, cudaStream_t s) {
  bump_step_kernel<<<1, 1, 0, s>>>(step_dev);
  check_launch("bump_step");
}

__global__ void __launch_bounds__(256)
adam_prox_kernel(float* __restrict__ x, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 const int* __restrict__ step_dev, int n, float lr, float b1, float b2, float eps,
                 const float* __restrict__ z, const float* __restrict__ y, float rho_host, float l1, float l2,
                 const float* __restrict__ rho_dev) {
  // adaptive ADMM keeps the penalty in device memory (written by bb_update_kernel): a captured graph never goes stale
  const float rho = rho_dev != nullptr ? __ldg(rho_dev) : rho_host;
  const float t = static_cast<float>(*step_dev);
  const float bc1 = 1.f - powf(b1, t);
  const float bc2 = 1.f - powf(b2, t);
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  const int n4 = n >> 2;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 xv = reinterpret_cast<float4*>(x)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), yv = zv;
    if (z != nullptr) zv = reinterpret_cast<const float4*>(z)[i];
    if (y != nullptr) yv = reinterpret_cast<const float4*>(y)[i];
    float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w}, ms[4] = {mv.x, mv.y, mv.z, mv.w},
          vs[4] = {vv.x, vv.y, vv.z, vv.w}, zs[4] = {zv.x, zv.y, zv.z, zv.w}, ys[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float gt = gs[j] + ys[j] + l1 * sgnf(xs[j]) + 2.f * l2 * xs[j];
      if (z != nullptr) gt += rho * (xs[j] - zs[j]);
      ms[j] = b1 * ms[j] + (1.f - b1) * gt;
      vs[j] = b2 * vs[j] + (1.f - b2) * gt * gt;
      const float denom = sqrtf(vs[j]) * inv_sqrt_bc2 + eps;
      xs[j] -= step_size * ms[j] / denom;
    }
    reinterpret_cast<float4*>(x)[i] = make_float4(xs[0], xs[1], xs[2], xs[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(ms[0], ms[1], ms[2], ms[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(vs[0], vs[1], vs[2], vs[3]);
  }
  // scalar tail (n not a multiple of 4)
  for (int i = (n4 << 2) + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float xi = x[i];
    float gt = g[i] + (y ? y[i] : 0.f) + l1 * sgnf(xi) + 2.f * l2 * xi;
    if (z != nullptr) gt += rho * (xi - z[i]);
    const float mi = b1 * m[i] + (1.f - b1) * gt;
    const float vi = b2 * v[i] + (1.f - b2) * gt * gt;
    m[i] = mi;
    v[i] = vi;
    x[i] = xi - step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + eps);
  }
}

void adam_prox(float* x, const float* g, float* m, float* v, const int* step_dev, int n, float lr, float b1, float b2,
               float eps, const float* z, const float* y, float rho, float l1, float l2, cudaStream_t s,
               const float* rho_dev) {
  adam_prox_kernel<<<grid_for(n), 256, 0, s>>>(x, g, m, v, step_dev, n, lr, b1, b2, eps, z, y, rho, l1, l2, rho_dev);
  check_launch("adam_prox");
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) l1_l2_kernel(const float* __restrict__ g, int n, float* __restrict__ out2) {
  __shared__ float sm[64];
  float acc[2] = {0.f, 0.f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float x = g[i];
    acc[0] += fabsf(x);
    acc[1] = fmaf(x, x, acc[1]);
  }
  block_reduce<2>(acc, sm);
  if (threadIdx.x == 0) {
    atomicAdd(out2, acc[0]);
    atomicAdd(out2 + 1, acc[1]);
  }
}
void l1_l2(const float* g, int n, float* out2, cudaStream_t s) {
  cudaMemsetAsync(out2, 0, 2 * sizeof(float), s);
  l1_l2_kernel<<<grid_for(n, 8), 256, 0, s>>>(g, n, out2);
  check_launch("l1_l2");
}

__global__ void __launch_bounds__(256)
make_pair_kernel(const float* __restrict__ g, const float* __restrict__ gp, const float* __restrict__ d, float t,
                 float trust, float* __restrict__ y, float* __restrict__ sv, int n, float* __restrict__ out3) {
  __shared__ float sm[96];
  float acc[3] = {0.f, 0.f, 0.f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float si = t * d[i];
    const float yi = g[i] - gp[i] + trust * si;
    y[i] = yi;
    sv[i] = si;
    acc[0] = fmaf(yi, si, acc[0]);
    acc[1] = fmaf(si, si, acc[1]);
    acc[2] = fmaf(yi, yi, acc[2]);
  }
  block_reduce<3>(acc, sm);
  if (threadIdx.x == 0) {
    atomicAdd(out3, acc[0]);
    atomicAdd(out3 + 1, acc[1]);
    atomicAdd(out3 + 2, acc[2]);
  }
}
void make_pair(const float* g, const float* gprev, const float* d, float t, float trust, float* y, float* sv, int n,
               float* out3, cudaStream_t s) {
  cudaMemsetAsync(out3, 0, 3 * sizeof(float), s);
  make_pair_kernel<<<grid_for(n, 4), 256, 0, s>>>(g, gprev, d, t, trust, y, sv, n, out3);
  check_launch("make_pair");
}

__global__ void __launch_bounds__(256)
welford_kernel(const float* __restrict__ g, float* __restrict__ mean, float* __restrict__ m2, int n, float inv_n,
               float* __restrict__ out1) {
  __shared__ float sm[32];
  float acc[1] = {0.f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float gi = g[i];
    const float delta = gi - mean[i];
    const float mu = mean[i] + delta * inv_n;
    const float q = m2[i] + (gi - mu) * delta;
    mean[i] = mu;
    m2[i] = q;
    acc[0] += q;
  }
  block_reduce<1>(acc, sm);
  if (threadIdx.x == 0) atomicAdd(out1, acc[0]);
}
void welford(const float* g, float* mean, float* m2, int n, float inv_n, float* out1, cudaStream_t s) {
  cudaMemsetAsync(out1, 0, sizeof(float), s);
  welford_kernel<<<grid_for(n, 4), 256, 0, s>>>(g, mean, m2, n, inv_n, out1);
  check_launch("welford");
}

__global__ void __launch_bounds__(256)
penalty_value_kernel(const float* __restrict__ x, const float* __restrict__ z, const float* __restrict__ y, float rho,
                     float l1, float l2, int n, float* __restrict__ out1) {
  __shared__ float sm[32];
  float acc[1] = {0.f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float xi = x[i];
    float v = l1 * fabsf(xi) + l2 * xi * xi;
    if (z != nullptr) {
      const float dx = xi - z[i];
      v += 0.5f * rho * dx * dx;
      if (y != nullptr) v = fmaf(y[i], dx, v);
    }
    acc[0] += v;
  }
  block_reduce<1>(acc, sm);
  if (threadIdx.x == 0) atomicAdd(out1, acc[0]);
}
void penalty_value(const float* x, const float* z, const float* y, float rho, float l1, float l2, int n, float* out1,
                   cudaStream_t s) {
  cudaMemsetAsync(out1, 0, sizeof(float), s);
  penalty_value_kernel<<<grid_for(n, 4), 256, 0, s>>>(x, z, y, rho, l1, l2, n, out1);
  check_launch("penalty_value");
}

__global__ void __launch_bounds__(256)
penalty_grad_kernel(float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ z,
                    const float* __restrict__ y, float rho, float l1, float l2, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float xi = x[i];
    float gt = g[i] + l1 * sgnf(xi) + 2.f * l2 * xi;
    if (z != nullptr) gt += rho * (xi - z[i]);
    if (y != nullptr) gt += y[i];
    g[i] = gt;
  }
}
void penalty_grad(float* g, const float* x, const float* z, const float* y, float rho, float l1, float l2, int n,
                  cudaStream_t s) {
  penalty_grad_kernel<<<grid_for(n, 4), 256, 0, s>>>(g, x, z, y, rho, l1, l2, n);
  check_launch("penalty_grad");
}

// up to 8 dot products of equal-length vectors in one pass (BB adaptive rho: 6 per worker)
struct DotPtrs {
  const float* a[8];
  const float* b[8];
};
__global__ void __launch_bounds__(256) multi_dot_kernel(DotPtrs p, int npairs, int n, float* __restrict__ out) {
  __shared__ float sm[8 * 32];
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (k < npairs) acc[k] = fmaf(p.a[k][i], p.b[k][i], acc[k]);
  }
  block_reduce<8>(acc, sm);
  if (threadIdx.x == 0)
    for (int k = 0; k < npairs; ++k) atomicAdd(out + k, acc[k]);
}
void multi_dot(const float* const* a, const float* const* b, int npairs, int n, float* out, cudaStream_t s) {
  if (npairs > 8) throw std::runtime_error("fedb200: multi_dot supports at most 8 pairs");
  DotPtrs p{};
  for (int k = 0; k < npairs; ++k) {
    p.a[k] = a[k];
    p.b[k] = b[k];
  }
  cudaMemsetAsync(out, 0, npairs * sizeof(float), s);
  multi_dot_kernel<<<grid_for(n, 4), 256, 0, s>>>(p, npairs, n, out);
  check_launch("multi_dot");
}

// ------------------------------------------------------------------------------------------------
// L-BFGS two-loop recursion, one cooperative kernel.
//   q = -g;  for i = k-1..0: al_i = ro_i (s_i.q); q -= al_i y_i
//   r = H q; for i = 0..k-1: be_i = ro_i (y_i.r); r += (al_i - be_i) s_i         (lbfgsnew.py:645-659)
// Each dependent dot product is accumulated during the pass that produces its input vector; passes are
// separated by a grid barrier.  work layout (floats): ro[k] | al[k] | dots[2k+2]; all zero on entry.
// ------------------------------------------------------------------------------------------------
constexpr int TL_MAX_HIST = 32;

size_t lbfgs_two_loop_work_floats(int k) { return size_t(5 * k + 4); }  // ro[k] | al[k] | dots[3k+1]

__device__ __forceinline__ void block_dot_commit(float v, float* sm, float* dst) {
  float a[1] = {v};
  block_reduce<1>(a, sm);
  if (threadIdx.x == 0) atomicAdd(dst, a[0]);
}

__global__ void __launch_bounds__(512)
lbfgs_two_loop_kernel(const float* __restrict__ Y, const float* __restrict__ S, const int* __restrict__ order, int k,
                      int n, int ld, const float* __restrict__ g, float hdiag, float* __restrict__ d,
                      float* __restrict__ work) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float sm[32];
  __shared__ int rows[TL_MAX_HIST];
  if (threadIdx.x < k) rows[threadIdx.x] = order[threadIdx.x];
  __syncthreads();
  float* ro = work;
  float* al = work + k;
  float* dots = work + 2 * k;           // dots[0..k): y_i.s_i ; dots[k + j]: running dependent dots
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;

  // pass 0: q = -g, curvature dots y_i.s_i, and s_{k-1}.q
  {
    float acc[TL_MAX_HIST];
#pragma unroll
    for (int i = 0; i < TL_MAX_HIST; ++i) acc[i] = 0.f;
    float first = 0.f;
    const float* s_last = S + size_t(rows[k - 1]) * ld;
    for (int j = tid; j < n; j += nth) {
      const float q = -g[j];
      d[j] = q;
      first = fmaf(s_last[j], q, first);
      for (int i = 0; i < k; ++i) acc[i] = fmaf(Y[size_t(rows[i]) * ld + j], S[size_t(rows[i]) * ld + j], acc[i]);
    }
    for (int i = 0; i < k; ++i) block_dot_commit(acc[i], sm, dots + i);
    block_dot_commit(first, sm, dots + k);
  }
  grid.sync();
  int slot = k;  // dots[slot] holds s_i.q for the current i
  for (int i = k - 1; i >= 0; --i) {
    const float roi = 1.f / __ldcg(dots + i);
    const float ali = __ldcg(dots + slot) * roi;
    if (tid == 0) {
      ro[i] = roi;
      al[i] = ali;
    }
    const float* yi = Y + size_t(rows[i]) * ld;
    const float* nxt = i > 0 ? S + size_t(rows[i - 1]) * ld : Y + size_t(rows[0]) * ld;  // next dependent dot
    const float scale = i > 0 ? 1.f : hdiag;   // last pass of the first loop also applies r = H q
    float acc = 0.f;
    for (int j = tid; j < n; j += nth) {
      const float q = (d[j] - ali * yi[j]) * scale;
      d[j] = q;
      acc = fmaf(nxt[j], q, acc);
    }
    block_dot_commit(acc, sm, dots + slot + 1);
    ++slot;
    grid.sync();
  }
  // second loop: dots[slot] = y_0.r
  for (int i = 0; i < k; ++i) {
    const float roi = 1.f / __ldcg(dots + i);
    const float bei = __ldcg(dots + slot) * roi;
    const float ali = __ldcg(dots + k + (k - 1 - i)) * roi;   // al_i recomputed from its stored dot (same value as above)
    const float coef = ali - bei;
    const float* si = S + size_t(rows[i]) * ld;
    const float* nxt = i + 1 < k ? Y + size_t(rows[i + 1]) * ld : nullptr;
    float acc = 0.f;
    for (int j = tid; j < n; j += nth) {
      const float r = fmaf(coef, si[j], d[j]);
      d[j] = r;
      if (nxt != nullptr) acc = fmaf(nxt[j], r, acc);
    }
    if (nxt != nullptr) block_dot_commit(acc, sm, dots + slot + 1);
    ++slot;
    grid.sync();
  }
}

void lbfgs_two_loop(const float* Y, const float* S, const int* order, int k, int n, int ld, const float* g, float hdiag,
                    float* d, float* work, cudaStream_t s) {
  if (k < 1 || k > TL_MAX_HIST) throw std::runtime_error("fedb200: lbfgs_two_loop history must be in [1,32]");
  cudaMemsetAsync(work, 0, lbfgs_two_loop_work_floats(k) * sizeof(float), s);
  int threads = 512;
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lbfgs_two_loop_kernel, threads, 0);
  if (per_sm < 1) per_sm = 1;
  int want = (n + threads - 1) / threads;
  int grid = num_sms() * (per_sm > 2 ? 2 : per_sm);
  if (want < grid) grid = want < 1 ? 1 : want;
  void* args[] = {(void*)&Y, (void*)&S, (void*)&order, (void*)&k, (void*)&n, (void*)&ld, (void*)&g, (void*)&hdiag,
                  (void*)&d, (void*)&work};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)lbfgs_two_loop_kernel, dim3(grid), dim3(threads), args, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: lbfgs_two_loop: ") + cudaGetErrorString(e));
  count_launch();
}

}  // namespace fedb200

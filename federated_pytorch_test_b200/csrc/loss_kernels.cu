// Fused loss kernels (SURVEY G9, G10): forward value + everything the backward needs in one pass.
//  * cross_entropy_fwd/bwd : one warp per sample; log-sum-exp, mean NLL (atomicAdd) and the softmax probabilities
//  * soft_ce_fwd/bwd       : the same for label-smoothed / mixed targets built in registers, mean in a fixed order
//  * vae_loss_fwd/bwd      : sum (recon-x)^2 - 1/2 sum(1 + logvar - mu^2 - exp(logvar)) as ONE reduction
#include "fedb200.h"

#include <stdexcept>
#include <string>

namespace fedb200 {

static inline void check_launch(const char* name) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: ") + name + ": " + cudaGetErrorString(e));
  count_launch();
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__global__ void __launch_bounds__(256)
ce_fwd_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, float* __restrict__ loss,
              float* __restrict__ probs, int B, int C) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const float* row = logits + size_t(warp) * C;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
  mx = wmax(mx);
  float se = 0.f;
  for (int c = lane; c < C; c += 32) se += __expf(row[c] - mx);
  se = wsum(se);
  const float lse = mx + __logf(se);
  const float inv = 1.f / se;
  for (int c = lane; c < C; c += 32) probs[size_t(warp) * C + c] = __expf(row[c] - mx) * inv;
  if (lane == 0) atomicAdd(loss, (lse - row[labels[warp]]) / float(B));
}
void cross_entropy_fwd(const float* logits, const long long* labels, float* loss, float* probs, int B, int C,
                       cudaStream_t s) {
  cudaMemsetAsync(loss, 0, sizeof(float), s);
  ce_fwd_kernel<<<(B * 32 + 255) / 256, 256, 0, s>>>(logits, labels, loss, probs, B, C);
  check_launch("cross_entropy_fwd");
}
__global__ void __launch_bounds__(256)
ce_bwd_kernel(const float* __restrict__ probs, const long long* __restrict__ labels, const float* __restrict__ gout,
              float* __restrict__ dlogits, int B, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float g = gout[0] / float(B);
  dlogits[i] = (probs[i] - (labels[b] == c ? 1.f : 0.f)) * g;
}
void cross_entropy_bwd(const float* probs, const long long* labels, const float* gout, float* dlogits, int B, int C,
                       cudaStream_t s) {
  ce_bwd_kernel<<<(B * C + 255) / 256, 256, 0, s>>>(probs, labels, gout, dlogits, B, C);
  check_launch("cross_entropy_bwd");
}

// Soft-target cross-entropy of label smoothing and mixup / CutMix: sample i's target is
// q_i = lam s(y_i) + (1 - lam) s(y_{B-1-i}) with s(y) = (1 - eps) onehot(y) + eps / C, formed in registers (lam read from
// device memory, 1 when lam == nullptr).  ONE CTA: warp w takes samples w, w + nw, ... and adds their losses in that order;
// thread 0 adds the warps' sums in warp order.  No atomics, so the loss has the same bits on every call.
__device__ __forceinline__ float soft_target(int c, long long yi, long long yj, float lam, float eps, int C) {
  const float hit = (c == yi ? lam : 0.f) + (c == yj ? 1.f - lam : 0.f);
  return (1.f - eps) * hit + eps / float(C);
}
constexpr int SOFT_CE_THREADS = 512;
__global__ void __launch_bounds__(SOFT_CE_THREADS)
soft_ce_fwd_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, const float* __restrict__ lam_p,
                   float eps, float* __restrict__ loss, float* __restrict__ probs, int B, int C) {
  __shared__ float part[SOFT_CE_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float lam = lam_p != nullptr ? lam_p[0] : 1.f;
  float acc = 0.f;
  for (int i = warp; i < B; i += nw) {
    const float* row = logits + size_t(i) * C;
    const long long yi = labels[i], yj = labels[B - 1 - i];
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
    mx = wmax(mx);
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += expf(row[c] - mx);
    se = wsum(se);
    const float lse = mx + logf(se);
    const float inv = 1.f / se;
    float l = 0.f;
    for (int c = lane; c < C; c += 32) {
      probs[size_t(i) * C + c] = expf(row[c] - mx) * inv;
      l = fmaf(soft_target(c, yi, yj, lam, eps, C), lse - row[c], l);      // -q_c log p_c, every term >= 0
    }
    acc += wsum(l);
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += part[w];
    loss[0] = t / float(B);
  }
}
void soft_ce_fwd(const float* logits, const long long* labels, const float* lam, float eps, float* loss, float* probs, int B,
                 int C, cudaStream_t s) {
  soft_ce_fwd_kernel<<<1, SOFT_CE_THREADS, 0, s>>>(logits, labels, lam, eps, loss, probs, B, C);
  check_launch("soft_ce_fwd");
}
__global__ void __launch_bounds__(256)
soft_ce_bwd_kernel(const float* __restrict__ probs, const long long* __restrict__ labels, const float* __restrict__ lam_p,
                   float eps, const float* __restrict__ gout, float* __restrict__ dlogits, int B, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float lam = lam_p != nullptr ? lam_p[0] : 1.f;
  const float g = gout[0] / float(B);
  dlogits[i] = (probs[i] - soft_target(c, labels[b], labels[B - 1 - b], lam, eps, C)) * g;
}
void soft_ce_bwd(const float* probs, const long long* labels, const float* lam, float eps, const float* gout, float* dlogits,
                 int B, int C, cudaStream_t s) {
  soft_ce_bwd_kernel<<<(B * C + 255) / 256, 256, 0, s>>>(probs, labels, lam, eps, gout, dlogits, B, C);
  check_launch("soft_ce_bwd");
}

__global__ void __launch_bounds__(256)
vae_fwd_kernel(const float* __restrict__ recon, const float* __restrict__ x, int n, const float* __restrict__ mu,
               const float* __restrict__ logvar, int nl, float* __restrict__ out) {
  __shared__ float sm[8];
  float acc = 0.f;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float d = recon[i] - x[i];
    acc = fmaf(d, d, acc);
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
    const float m = mu[i], lv = logvar[i];
    acc -= 0.5f * (1.f + lv - m * m - __expf(lv));
  }
  acc = wsum(acc);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.f;
    v = wsum(v);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}
void vae_loss_fwd(const float* recon, const float* x, int n, const float* mu, const float* logvar, int nl, float* out,
                  cudaStream_t s) {
  cudaMemsetAsync(out, 0, sizeof(float), s);
  int grid = (n + 1023) / 1024;
  if (grid > 132 * 4) grid = 132 * 4;
  if (grid < 1) grid = 1;
  vae_fwd_kernel<<<grid, 256, 0, s>>>(recon, x, n, mu, logvar, nl, out);
  check_launch("vae_loss_fwd");
}
__global__ void __launch_bounds__(256)
vae_bwd_kernel(const float* __restrict__ recon, const float* __restrict__ x, int n, const float* __restrict__ mu,
               const float* __restrict__ logvar, int nl, const float* __restrict__ gout, float* __restrict__ drecon,
               float* __restrict__ dmu, float* __restrict__ dlogvar) {
  const float g = gout[0];
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) drecon[i] = 2.f * (recon[i] - x[i]) * g;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
    dmu[i] = mu[i] * g;
    dlogvar[i] = -0.5f * (1.f - __expf(logvar[i])) * g;
  }
}
void vae_loss_bwd(const float* recon, const float* x, int n, const float* mu, const float* logvar, int nl,
                  const float* gout, float* drecon, float* dmu, float* dlogvar, cudaStream_t s) {
  int grid = (n + 1023) / 1024;
  if (grid > 132 * 4) grid = 132 * 4;
  if (grid < 1) grid = 1;
  vae_bwd_kernel<<<grid, 256, 0, s>>>(recon, x, n, mu, logvar, nl, gout, drecon, dmu, dlogvar);
  check_launch("vae_loss_bwd");
}

}  // namespace fedb200

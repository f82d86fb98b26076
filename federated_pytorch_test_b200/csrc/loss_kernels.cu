// Fused loss kernels (SURVEY G9, G10): forward value + everything the backward needs in one pass.
//  * cross_entropy_fwd/bwd : one warp per sample; log-sum-exp, mean NLL (atomicAdd) and the softmax probabilities
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

// Convolution WEIGHT gradient on Hopper tensor cores (SURVEY G1 wgrad, G6/G7 backward) — any k x k, stride, dilation,
// padding.
//
//   dW[co, r, s, ci] = sum over output pixels (n, ho, wo) of  dy[n, ho, wo, co] * x[n, ho*st + r*dl - pd, wo*st + s*dl - pd, ci]
//
// As a GEMM: rows j = (tap, ci) (M, 128 per CTA, 64 per warpgroup), columns co (N = BN), reduction over the PIXEL index
// (K, 32 per k-block).  Both operands are stored pixel-major with the channel contiguous (NHWC), i.e. MN-major, and
// wgmma reads tf32 operands only K-major.  So the CTA gathers each k-block with channel-contiguous (coalesced) loads —
// the shifted input window of a tap, zero outside the image, is just a different address — and writes it transposed into
// unswizzled K-major tiles of 8 x 16-byte core matrices.  The gather is register double-buffered: the loads of k-block
// i + 1 are in flight while the MMAs of k-block i run.
//
// Work decomposition: CTA = (j tile) x (co tile) x (split of the pixel range).  Partial sums are added into dW with
// red.global.add.f32; the caller provides dW zeroed, or the parameter's gradient buffer itself (accumulation is what
// autograd wants).
//
// BM = 64 (the host picks it when taps * C_x <= 64, e.g. the 3 x 3 stem on its 4-channel input): one 64-row tile whose rows
// are (tap, ci) over ALL C_x stored channels, so each thread gathers whole 16-byte channel quads (C_x % 4 == 0) of 2 pixels
// instead of 16 single floats; rows of padding channels (ci >= C_w) are computed and dropped by the epilogue.  The two
// warpgroups split each k-block's 4 MMA k-steps, and warpgroup 1 hands its partial sums to warpgroup 0 through shared memory.
#pragma once
#include "sm90.cuh"

namespace fedb200 {

constexpr int WG_THREADS = 256;                 // two warpgroups
constexpr int WG_BM = 128;                      // (tap, ci) rows per CTA
constexpr int WG_BK = 32;                       // pixels per k-block
constexpr int WG_A_BYTES = WG_BM * WG_BK * 4;   // 16 KB
constexpr int WG_BM_SMALL = 64;                 // rows of the small-J tile (BM = 64)

struct WgradParams {
  int H, W, Cx, Cw, Co, kw, stride, pad, dil, H_out, W_out;
  int J;                // taps * Cw: GEMM rows
  int P;                // output pixels NB * H_out * W_out
  int kb_per_split;     // k-blocks (of WG_BK pixels) per CTA
  int j_tiles, co_tiles;
  float* dw;            // [Co, taps, Cw]
};

// byte offset of element (row, k) of a [rows x 32] K-major tile of core matrices: LBO = 128 B (along K), SBO = 1024 B
__device__ __forceinline__ uint32_t wg_core_offset(int row, int k) {
  return uint32_t((row >> 3) * 1024 + (k >> 2) * 128 + (row & 7) * 16 + (k & 3) * 4);
}
__device__ __forceinline__ float to_tf32(float v) {   // round to nearest (as the TMA unit does for the forward kernels)
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

// BM = 64: see the header.  Same operand layout and rounding as the 128-row tile.
template <int BN>
__device__ __forceinline__ void wgrad_small_j(const float* __restrict__ x, const float* __restrict__ dy, const WgradParams& p) {
  constexpr int A_BYTES = WG_BM_SMALL * WG_BK * 4;     // 8 KB
  constexpr int B_BYTES = BN * WG_BK * 4;
  constexpr int BUF_BYTES = A_BYTES + B_BYTES;
  constexpr int QUADS = WG_BM_SMALL / 4;               // 16 channel quads (rows 4 q .. 4 q + 3)
  constexpr int A_GROUPS = WG_THREADS / QUADS;         // 16 pixel groups
  constexpr int A_PER = WG_BK / A_GROUPS;              // 2 float4 per thread and k-block
  constexpr int B_GROUPS = WG_THREADS / BN;
  constexpr int B_PER = WG_BK / B_GROUPS;
  constexpr int NACC = BN / 2;
  static_assert(2 * BUF_BYTES >= WG_THREADS / 2 * NACC * 4, "the cross-warpgroup sum reuses the operand buffers");
  extern __shared__ __align__(1024) uint8_t smem[];

  const int tid = threadIdx.x;
  const int g = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  int unit = blockIdx.x;                               // j_tiles == 1
  const int ct = unit % p.co_tiles;
  const int split = unit / p.co_tiles;
  const int co0 = ct * BN;
  const int kb_begin = split * p.kb_per_split;
  const int kb_total = (p.P + WG_BK - 1) / WG_BK;
  const int nkb = min(p.kb_per_split, kb_total - kb_begin);
  const int HWo = p.H_out * p.W_out;
  const int taps = p.J / p.Cw;
  const int Jx = taps * p.Cx;                          // gathered rows: every stored channel

  // lane bits 0-1 -> pixel, bits 2-5 -> quad: a warp's scatter stores hit 8 distinct (row % 8, k % 4) banks
  const int a_q = (tid >> 2) & (QUADS - 1), a_pg = (tid & 3) | ((tid >> 6) << 2);
  const int j4 = 4 * a_q;
  const bool j_ok = j4 < Jx;
  const int tap = j_ok ? j4 / p.Cx : 0;
  const int ci = j_ok ? j4 - tap * p.Cx : 0;
  const int dh = (tap / p.kw) * p.dil - p.pad, dwo = (tap % p.kw) * p.dil - p.pad;
  const int b_row = tid % BN, b_pg = tid / BN;
  const int co = co0 + b_row;
  const bool co_ok = co < p.Co;

  float4 ra[A_PER];
  float rb[B_PER];
  auto gather = [&](int kb) {
    const int pbase = (kb_begin + kb) * WG_BK;
#pragma unroll
    for (int q = 0; q < A_PER; ++q) {
      const int pix = pbase + a_pg + A_GROUPS * q;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j_ok && pix < p.P) {
        const int n = pix / HWo, rem = pix - n * HWo;
        const int ho = rem / p.W_out, wo = rem - ho * p.W_out;
        const int h = ho * p.stride + dh, w = wo * p.stride + dwo;
        if (h >= 0 && h < p.H && w >= 0 && w < p.W)
          v = __ldg(reinterpret_cast<const float4*>(x + ((size_t(n) * p.H + h) * p.W + w) * p.Cx + ci));
      }
      ra[q] = v;
    }
#pragma unroll
    for (int q = 0; q < B_PER; ++q) {
      const int pix = pbase + b_pg + B_GROUPS * q;
      rb[q] = (co_ok && pix < p.P) ? __ldg(dy + size_t(pix) * p.Co + co) : 0.f;
    }
  };
  auto scatter = [&](int buf) {
    uint8_t* a = smem + buf * BUF_BYTES;
    uint8_t* b = a + A_BYTES;
#pragma unroll
    for (int q = 0; q < A_PER; ++q) {
      const int k = a_pg + A_GROUPS * q;
      const float v[4] = {ra[q].x, ra[q].y, ra[q].z, ra[q].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) *reinterpret_cast<float*>(a + wg_core_offset(j4 + c, k)) = to_tf32(v[c]);
    }
#pragma unroll
    for (int q = 0; q < B_PER; ++q) *reinterpret_cast<float*>(b + wg_core_offset(b_row, b_pg + B_GROUPS * q)) = to_tf32(rb[q]);
    fence_proxy_async();
  };

  pdl_launch_dependents();
  pdl_wait();
  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  const uint32_t base = smem_u32(smem);
  if (nkb > 0) {
    gather(0);
    scatter(0);
    __syncthreads();
  }
  for (int kb = 0; kb < nkb; ++kb) {
    const int buf = kb & 1;
    if (kb + 1 < nkb) gather(kb + 1);
    const uint32_t a_addr = base + uint32_t(buf * BUF_BYTES);
    const uint32_t b_addr = a_addr + uint32_t(A_BYTES);
    wgmma_fence();
    wgmma_fence_acc(acc);
#pragma unroll
    for (int kk = 0; kk < WG_BK / 16; ++kk) {          // warpgroup g: k-steps 2 g, 2 g + 1
      const uint32_t k = uint32_t(2 * g + kk);
      wgmma_tf32<BN>(acc, make_kmajor_interleave_desc(a_addr + 256u * k, 128, 1024),
                     make_kmajor_interleave_desc(b_addr + 256u * k, 128, 1024), 1u);
    }
    wgmma_commit();
    if (kb + 1 < nkb) scatter(buf ^ 1);
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    __syncthreads();
  }

  // warpgroup 1 -> shared memory (the operand buffers are free after the loop's last barrier) -> warpgroup 0 adds
  float* red = reinterpret_cast<float*>(smem);
  const int t128 = tid & 127;
  if (g == 1) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) red[i * 128 + t128] = acc[i];
  }
  __syncthreads();
  if (g == 1 || nkb <= 0) return;
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] += red[i * 128 + t128];
  const int r_a = 16 * warp + (lane >> 2);
#pragma unroll
  for (int i = 0; i < NACC / 4; ++i) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int jj = r_a + 8 * (e >> 1);
      const int cc = co0 + 8 * i + 2 * (lane & 3) + (e & 1);
      const int t_ = jj / p.Cx, c_ = jj - t_ * p.Cx;
      if (jj < Jx && c_ < p.Cw && cc < p.Co) atomicAdd(p.dw + size_t(cc) * p.J + t_ * p.Cw + c_, acc[4 * i + e]);
    }
  }
}

template <int BN, int BM = WG_BM>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_wgmma_kernel(const float* __restrict__ x, const float* __restrict__ dy, const WgradParams p) {
  static_assert(BM == WG_BM || BM == WG_BM_SMALL, "128- or 64-row tiles");
  if constexpr (BM == WG_BM_SMALL) {
    wgrad_small_j<BN>(x, dy, p);
    return;
  }
  constexpr int B_BYTES = BN * WG_BK * 4;
  constexpr int BUF_BYTES = WG_A_BYTES + B_BYTES;
  constexpr int A_PER = WG_BM * WG_BK / WG_THREADS;    // 16 A elements per thread and k-block
  constexpr int B_GROUPS = WG_THREADS / BN;            // pixel groups of the B gather
  constexpr int B_PER = WG_BK / B_GROUPS;              // B elements per thread and k-block
  constexpr int NACC = BN / 2;
  extern __shared__ __align__(1024) uint8_t smem[];    // [2 buffers][A | B]

  const int tid = threadIdx.x;
  const int g = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  int unit = blockIdx.x;
  const int jt = unit % p.j_tiles;
  unit /= p.j_tiles;
  const int ct = unit % p.co_tiles;
  const int split = unit / p.co_tiles;
  const int j0 = jt * WG_BM, co0 = ct * BN;
  const int kb_begin = split * p.kb_per_split;
  const int kb_total = (p.P + WG_BK - 1) / WG_BK;
  const int nkb = min(p.kb_per_split, kb_total - kb_begin);
  const int HWo = p.H_out * p.W_out;

  // A gather: this thread's row j is fixed, its pixels are a_pg, a_pg + 2, ...
  const int a_row = tid & (WG_BM - 1), a_pg = tid >> 7;
  const int j = j0 + a_row;
  const bool j_ok = j < p.J;
  const int tap = j_ok ? j / p.Cw : 0;
  const int ci = j_ok ? j - tap * p.Cw : 0;
  const int dh = (tap / p.kw) * p.dil - p.pad, dwo = (tap % p.kw) * p.dil - p.pad;
  // B gather: this thread's column co is fixed, its pixels are b_pg, b_pg + B_GROUPS, ...
  const int b_row = tid % BN, b_pg = tid / BN;
  const int co = co0 + b_row;
  const bool co_ok = co < p.Co;

  float ra[A_PER], rb[B_PER];
  auto gather = [&](int kb) {
    const int pbase = (kb_begin + kb) * WG_BK;
#pragma unroll
    for (int q = 0; q < A_PER; ++q) {
      const int pix = pbase + a_pg + 2 * q;
      float v = 0.f;
      if (j_ok && pix < p.P) {
        const int n = pix / HWo, rem = pix - n * HWo;
        const int ho = rem / p.W_out, wo = rem - ho * p.W_out;
        const int h = ho * p.stride + dh, w = wo * p.stride + dwo;
        if (h >= 0 && h < p.H && w >= 0 && w < p.W) v = __ldg(x + ((size_t(n) * p.H + h) * p.W + w) * p.Cx + ci);
      }
      ra[q] = v;
    }
#pragma unroll
    for (int q = 0; q < B_PER; ++q) {
      const int pix = pbase + b_pg + B_GROUPS * q;
      rb[q] = (co_ok && pix < p.P) ? __ldg(dy + size_t(pix) * p.Co + co) : 0.f;
    }
  };
  auto scatter = [&](int buf) {
    uint8_t* a = smem + buf * BUF_BYTES;
    uint8_t* b = a + WG_A_BYTES;
#pragma unroll
    for (int q = 0; q < A_PER; ++q) *reinterpret_cast<float*>(a + wg_core_offset(a_row, a_pg + 2 * q)) = to_tf32(ra[q]);
#pragma unroll
    for (int q = 0; q < B_PER; ++q) *reinterpret_cast<float*>(b + wg_core_offset(b_row, b_pg + B_GROUPS * q)) = to_tf32(rb[q]);
    fence_proxy_async();      // generic-proxy writes -> visible to the tensor core's (async proxy) reads
  };

  pdl_launch_dependents();
  pdl_wait();
  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  const uint32_t base = smem_u32(smem);
  if (nkb > 0) {
    gather(0);
    scatter(0);
    __syncthreads();
  }
  for (int kb = 0; kb < nkb; ++kb) {
    const int buf = kb & 1;
    if (kb + 1 < nkb) gather(kb + 1);
    const uint32_t a_addr = base + uint32_t(buf * BUF_BYTES) + uint32_t(g) * 8192u;   // rows 64 g .. 64 g + 63
    const uint32_t b_addr = base + uint32_t(buf * BUF_BYTES + WG_A_BYTES);
    wgmma_fence();
    wgmma_fence_acc(acc);
#pragma unroll
    for (int k = 0; k < WG_BK / 8; ++k)
      wgmma_tf32<BN>(acc, make_kmajor_interleave_desc(a_addr + 256u * k, 128, 1024),
                     make_kmajor_interleave_desc(b_addr + 256u * k, 128, 1024), 1u);
    wgmma_commit();
    if (kb + 1 < nkb) scatter(buf ^ 1);   // the other buffer's MMAs were waited for in the previous iteration
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    __syncthreads();
  }

  // fragment: row 16 warp + lane / 4 (+ 8) of this warpgroup's 64 rows, column 8 i + 2 (lane & 3) (+ 1)
  const int r_a = j0 + 64 * g + 16 * warp + (lane >> 2);
#pragma unroll
  for (int i = 0; i < NACC / 4; ++i) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int jj = r_a + 8 * (e >> 1);
      const int cc = co0 + 8 * i + 2 * (lane & 3) + (e & 1);
      if (jj < p.J && cc < p.Co && nkb > 0) atomicAdd(p.dw + size_t(cc) * p.J + jj, acc[4 * i + e]);
    }
  }
}

}  // namespace fedb200

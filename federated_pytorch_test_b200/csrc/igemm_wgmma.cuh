// Implicit GEMM on Hopper tensor cores: ONE persistent, warp-specialised kernel for
//   (a) plain GEMM          C[M,N]   = A[M,K] * B[N,K]^T                 (Linear layers)
//   (b) NHWC convolution    Y[m,co]  = sum_{r,s,ci} X[n,h*st+r*d-p,w*st+s*d-p,ci] * W[co,r,s,ci]
// A and B tiles are brought in by TMA as swizzled K-major tiles (32 fp32 = 128 B per row, rounded to tf32 by the TMA
// unit); for (b) the A tile of filter tap (r,s) is a 4-D TMA box over the NHWC activation [C,W,H,N] shifted by the tap
// offset, with out-of-bounds rows/columns zero-filled by the TMA unit — the im2col matrix is never materialised.
//
// One CTA per SM walks a static list of output tiles (tile = blockIdx.x + i * gridDim.x over [K split][M tile][N tile]);
// the shared-memory ring keeps rolling across tiles, so the producer fetches the next tile's operands while the
// consumers run the epilogue of the current one.
//
// Roles (384 threads = three warpgroups):
//   warpgroup 0     one thread issues the TMA loads (full / empty mbarrier ring);
//   warpgroups 1, 2 each owns 64 of the 128 tile rows: wgmma.m64nBLOCK_Nk8 (tf32 in, fp32 accumulate in registers),
//                   then the fused epilogue:
//   * bias + ELU (dense layers, VAE / CPC convolutions), or
//   * per-channel sum / sum-of-squares of the tile (BatchNorm batch statistics, reduced across the CTA in shared
//     memory, one atomicAdd per channel per tile), or
//   * eval-mode BatchNorm from the running statistics + residual + ELU (inference: conv + BN + add + ELU in one launch);
//   * output through a 128B-swizzled staging tile and bulk tensor stores (reduce-adds for split-K), or
//     direct stores when the row pitch is not 16-byte aligned.
#pragma once
#include "sm90.cuh"
#include "fedb200.h"

namespace fedb200 {

constexpr int IG_BLOCK_M = 128;
constexpr int IG_BLOCK_K = 32;  // fp32 elements per k-block = 128 B = one swizzle row
constexpr int IG_MMA_K = 8;     // tf32: 32 B per MMA k-step
constexpr int IG_THREADS = 384;

struct IgemmParams {
  int M, N;              // output rows (pixels) and columns (channels)
  int num_k_blocks;      // taps * cblocks
  int cblocks;           // ceil(Cin / 32); k-block kb -> tap = kb / cblocks, cb = kb % cblocks
  int taps_w;            // filter width (tap -> r = tap / taps_w, s = tap % taps_w); 1 for GEMM
  int b_cols_per_tap;    // columns of the weight matrix per tap (= Cin as stored)
  int is_conv;           // 0: A is a 2-D map [K, M]; 1: A is a 4-D map [C, W, H, N]
  int HW_out, W_out;     // conv: output pixels per image, output width
  int stride, pad, dil;  // conv geometry
  float* out;            // [M, ldo]
  int ldo;
  const float* bias;     // [N] or nullptr
  int act;               // 1 = ELU
  float* stats;          // [2*N]: sum, sumsq per column (atomicAdd) or nullptr
  int kb_per_split;      // split-K: K slice z handles k-blocks [z*kb_per_split, ...) and reduce-adds into a zeroed output
  int k_splits;          // 1 = plain stores (+ fused stats); > 1 = reduction through L2, stats done by the caller
  int m_tiles, n_tiles, total_tiles;   // tile t -> (t % n_tiles, (t / n_tiles) % m_tiles, K split)
  int shuffle_ci;        // > 0: the N columns are (ph, pw, ci) phase-packed channels of a stride-2 data gradient /
                         // transposed conv; each 32 x 32 chunk is stored to out[n, 2 ho + ph, 2 wo + pw, ci0 .. ci0 + 31] through a
                         // 5-D tensor map (no separate pixel-shuffle pass).  shuffle_ci = channels of the shuffled output.
  int tma_store;         // write the output with bulk tensor stores / reduce-adds (needs ldo % 4 == 0)
  int cw;                // convolutions with few input channels: channels per filter tap inside a 32-wide k-block.
                         // 0 / 32 = one tap per k-block (C_in padded to 32 by the TMA zero fill: 4x wasted MMAs at C_in = 8);
                         // 8 / 16 = "tap packing": a k-block holds 32 / cw taps, each its own cw-channel sub-tile (rows of cw * 4 bytes,
                         // TMA SWIZZLE_32B / 64B, wgmma descriptors of the matching layout).  num_k_blocks = ceil(taps / (32 / cw)).
  int taps_total;        // kh * kw (tap packing: taps beyond it load out-of-bounds zeros)
  int ms_kh;             // > 0: "multi-dilation" convolution — the filter rows are ms_branches groups of ms_kh rows,
                         // group b reads the input with dilation ms_dil[b] and padding ms_pad[b] (one byte each, packed); the weight
                         // matrix is block diagonal (branch b owns its own output channels).  The five dilated stem convolutions
                         // of the CPC encoder run as ONE launch writing the concatenated tensor (SURVEY G6).  pad = 0, dil = 1 then.
  unsigned long long ms_dil, ms_pad;
  // eval-mode BatchNorm (k_splits == 1, stats == nullptr): column c -> v * s_c + t_c with s_c = gamma_c / sqrt(var_c + eps),
  // t_c = beta_c - mean_c * s_c (per tile in shared memory), then + residual, then act.  bn_gamma == nullptr: off (the host
  // launches the EVAL_BN instantiation of the kernel exactly when it is set).
  const float* bn_gamma;
  const float* bn_beta;
  const float* bn_mean;
  const float* bn_var;
  float bn_eps;
  const float* residual; // [M, ldr] (NHWC, like the output) or nullptr; ldr even, 8-byte aligned
  int ldr;
  // window reuse (igemm_wgmma_pix_kernel<CO, STAGES, WIN_KH > 0>): a k-block is one (filter column s, 32-channel block) unit
  // whose stage is [win_rows x W_out pixels x 128 B | WIN_KH weight boxes of C_out rows x 128 B]; num_k_blocks = kw * cblocks.
  int win_rows;          // image rows per window: tile rows + WIN_KH - 1
  int win_a_bytes;       // win_rows * W_out * 128
  int win_stage_bytes;   // win_a_bytes + WIN_KH * C_out * 128 (a multiple of 1024)
};

template <int BLOCK_N, int STAGES>
struct IgemmSmem {
  static constexpr int A_BYTES = IG_BLOCK_M * IG_BLOCK_K * 4;   // 16 KB
  static constexpr int B_BYTES = BLOCK_N * IG_BLOCK_K * 4;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;         // one k-block: [A | B]
  static constexpr int STAGING_BYTES = 2 * 64 * 32 * 4;         // per consumer warpgroup: two 32 x 32 output boxes
  // column partials (sum, sumsq) of the tile per consumer warp, or eval-BN (scale, shift) of the tile in the first 2 * BLOCK_N
  static constexpr int STATS_BYTES = 8 * 2 * BLOCK_N * 4;
  static constexpr int BAR_BYTES = 2 * STAGES * 8;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + STAGING_BYTES + STATS_BYTES + BAR_BYTES + 1024;  // + align slack
};

struct TileCoord {
  int m0, n0, kb_begin, kb_count;
};
__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int t, int block_m, int block_n) {
  const int n_idx = t % p.n_tiles;
  const int rest = t / p.n_tiles;
  const int m_idx = rest % p.m_tiles;
  const int z = rest / p.m_tiles;
  TileCoord c;
  c.m0 = m_idx * block_m;
  c.n0 = n_idx * block_n;
  c.kb_begin = z * p.kb_per_split;
  c.kb_count = min(p.kb_per_split, p.num_k_blocks - c.kb_begin);
  return c;
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t n) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// TMA producer (one thread): walks this CTA's tiles and streams their k-blocks through the STAGES-deep ring, each stage
// [A: TILE_M operand rows (pixels or GEMM rows) x 32 | B: BLOCK_N weight rows x 32], full / empty mbarrier protocol.
template <int TILE_M, int BLOCK_N, int STAGES, int A_BYTES, int STAGE_BYTES>
__device__ __forceinline__ void igemm_produce(const IgemmParams& p, uint8_t* tiles, uint64_t* full_bar, uint64_t* empty_bar,
                                              const CUtensorMap* tmap_a, const CUtensorMap* tmap_b) {
  int s = 0;
  uint32_t ph = 0;
  const int cwp = (p.cw == 8 || p.cw == 16) ? p.cw : 0;        // tap packing
  const int tpk = cwp ? IG_BLOCK_K / cwp : 1;
  const int img_oob = p.is_conv ? p.M / p.HW_out + 1 : 0;        // first image index past the tensor: the TMA unit zero-fills
  const int col_oob = p.taps_total * p.b_cols_per_tap + IG_BLOCK_K;   // first weight column past the filter (+ a box)
  // tap -> offset inside the (padded) input window
  auto tap_offset = [&](int rr_, int sx_, int& cw_, int& ch_) {
    cw_ = sx_ * p.dil - p.pad;
    ch_ = rr_ * p.dil;
    if (p.ms_kh > 0) {                                          // multi-dilation: rows are (branch, row) pairs
      const int br = rr_ / p.ms_kh, rr = rr_ - br * p.ms_kh;
      const int d = int((p.ms_dil >> (8 * br)) & 0xffull), pd = int((p.ms_pad >> (8 * br)) & 0xffull);
      cw_ = sx_ * d - pd;
      ch_ = rr * d - pd;
    }
  };
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileCoord c = decode_tile(p, t, TILE_M, BLOCK_N);
    int img = 0, h0 = 0;
    if (p.is_conv) {                    // past the end: image index >= NB, the TMA unit zero-fills
      img = c.m0 / p.HW_out;
      h0 = ((c.m0 - img * p.HW_out) / p.W_out) * p.stride - p.pad;
    }
    int tap = c.kb_begin / p.cblocks;
    int cb = c.kb_begin - tap * p.cblocks;
    int r = tap / p.taps_w, sx = tap - r * p.taps_w;
    for (int kb = c.kb_begin; kb < c.kb_begin + c.kb_count; ++kb) {
      mbar_wait(&empty_bar[s], ph ^ 1);
      uint8_t* a_dst = tiles + s * STAGE_BYTES;
      uint8_t* b_dst = a_dst + A_BYTES;
      mbar_arrive_expect_tx(&full_bar[s], uint32_t(STAGE_BYTES));
      if (cwp) {
        // tpk taps per k-block, each a [TILE_M rows x cwp channels] sub-tile of A and a [BLOCK_N x cwp] sub-tile of B
        const int sub_a = TILE_M * cwp * 4, sub_b = BLOCK_N * cwp * 4;
        for (int jt = 0; jt < tpk; ++jt) {
          const int tp = kb * tpk + jt;
          const bool real = tp < p.taps_total;
          int cw = 0, ch = 0;
          if (real) tap_offset(tp / p.taps_w, tp % p.taps_w, cw, ch);
          // a tap past the filter: image index out of range -> zeros
          tma_load_4d(a_dst + jt * sub_a, tmap_a, &full_bar[s], 0, cw, h0 + ch, real ? img : img_oob);
          tma_load_2d(b_dst + jt * sub_b, tmap_b, &full_bar[s], real ? tp * p.b_cols_per_tap : col_oob, c.n0);
        }
      } else {
        int cw, ch;
        tap_offset(r, sx, cw, ch);
        if (p.is_conv)
          tma_load_4d(a_dst, tmap_a, &full_bar[s], cb * IG_BLOCK_K, cw, h0 + ch, img);
        else
          tma_load_2d(a_dst, tmap_a, &full_bar[s], kb * IG_BLOCK_K, c.m0);
        tma_load_2d(b_dst, tmap_b, &full_bar[s], (r * p.taps_w + sx) * p.b_cols_per_tap + cb * IG_BLOCK_K, c.n0);
        if (++cb == p.cblocks) {
          cb = 0;
          if (++sx == p.taps_w) { sx = 0; ++r; }
        }
      }
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  }
}

// EVAL_BN: the eval-mode BatchNorm (+ residual) epilogue (IgemmParams::bn_*) is compiled in; a separate instantiation, so the
// training and GEMM launches keep the plain epilogue's code and register budget.
template <int BLOCK_N, int STAGES, bool EVAL_BN>
__global__ void __launch_bounds__(IG_THREADS, 1)
igemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_c, const IgemmParams p) {
  using S = IgemmSmem<BLOCK_N, STAGES>;
  static_assert(BLOCK_N == 32 || BLOCK_N == 64 || BLOCK_N == 128, "BLOCK_N must be 32, 64 or 128");
  static_assert(S::TOTAL <= 227 * 1024, "shared memory budget");
  static_assert(S::STAGE_BYTES % 1024 == 0, "stages must keep the 1024-byte swizzle alignment");
  constexpr int NACC = BLOCK_N / 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  float* staging = reinterpret_cast<float*>(smem + STAGES * S::STAGE_BYTES);
  float* colsum = reinterpret_cast<float*>(smem + STAGES * S::STAGE_BYTES + S::STAGING_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(colsum + 8 * 2 * BLOCK_N);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (p.tma_store) tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);            // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0)
      igemm_produce<IG_BLOCK_M, BLOCK_N, STAGES, S::A_BYTES, S::STAGE_BYTES>(p, tiles, full_bar, empty_bar, &tmap_a, &tmap_b);
    return;
  }

  // ===================== consumers: warpgroup g owns tile rows [64 g, 64 g + 64) =====================
  const int g = wg - 1;
  const int warp = tid >> 5, lane = tid & 31;
  // operand rows of 128 bytes (one tap x 32 channels per k-block) or, with tap packing, cw * 4 bytes per sub-tile
  const uint32_t cwq = (p.cw == 8 || p.cw == 16) ? uint32_t(p.cw) : uint32_t(IG_BLOCK_K);
  const uint32_t mma_per_sub = cwq / IG_MMA_K;                             // MMAs (K = 8) per sub-tile: 1, 2 or 4
  const uint64_t adesc0 = make_kmajor_desc(smem_u32(tiles) + uint32_t(g) * 64u * cwq * 4u, cwq * 4u);
  const uint64_t bdesc0 = make_kmajor_desc(smem_u32(tiles) + uint32_t(S::A_BYTES), cwq * 4u);
  uint32_t a_off[IG_BLOCK_K / IG_MMA_K], b_off[IG_BLOCK_K / IG_MMA_K];    // descriptor offsets (16-B units) of the 4 k-steps
#pragma unroll
  for (int k = 0; k < IG_BLOCK_K / IG_MMA_K; ++k) {
    const uint32_t sub = uint32_t(k) / mma_per_sub, in = uint32_t(k) - sub * mma_per_sub;
    a_off[k] = (sub * uint32_t(IG_BLOCK_M) * cwq * 4u + in * 32u) >> 4;
    b_off[k] = (sub * uint32_t(BLOCK_N) * cwq * 4u + in * 32u) >> 4;
  }
  float* stg = staging + g * 2048;            // [2 boxes][32 rows][32 floats], 1024-B aligned, chunk index XOR (row & 7)
  const uint32_t wg_bar = 1 + uint32_t(g);    // named barrier of this warpgroup; 3 = both consumer warpgroups
  const int row_in = 16 * warp + (lane >> 2); // tile-local row (within the warpgroup) of d[4i], d[4i+1]; d[4i+2..3]: + 8
  const int col_in = 2 * (lane & 3);          // column of d[4i] within its 8-column block

  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  int s = 0;
  uint32_t ph = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileCoord c = decode_tile(p, t, IG_BLOCK_M, BLOCK_N);
    if constexpr (EVAL_BN) {
      // eval-mode BatchNorm: the tile's per-column scale / shift, once per tile, in the (otherwise unused) statistics area
      named_bar_sync(3, 256);                    // the previous tile's epilogue has read them
      for (int cc = threadIdx.x - 128; cc < BLOCK_N; cc += 256) {
        const int col = c.n0 + cc;
        float sc = 0.f, sh = 0.f;
        if (col < p.N) {
          sc = __ldg(p.bn_gamma + col) * rsqrtf(__ldg(p.bn_var + col) + p.bn_eps);
          sh = fmaf(-__ldg(p.bn_mean + col), sc, __ldg(p.bn_beta + col));
        }
        colsum[cc] = sc;
        colsum[BLOCK_N + cc] = sh;
      }
      named_bar_sync(3, 256);
    }
    // ---- main loop: one k-block per stage, the previous stage is released once its MMAs have retired
    int prev = -1;
    for (int i = 0; i < c.kb_count; ++i) {
      mbar_wait(&full_bar[s], ph);
      const uint64_t so = uint64_t(uint32_t(s) * uint32_t(S::STAGE_BYTES >> 4));
      wgmma_fence();
      wgmma_fence_acc(acc);
#pragma unroll
      for (int k = 0; k < IG_BLOCK_K / IG_MMA_K; ++k)
        wgmma_tf32<BLOCK_N>(acc, adesc0 + so + a_off[k], bdesc0 + so + b_off[k], (i > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_fence_acc(acc);
      wgmma_wait<1>();
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue
    const int row_a = c.m0 + 64 * g + row_in, row_b = row_a + 8;
    const bool ok_a = row_a < p.M, ok_b = row_b < p.M;
#pragma unroll
    for (int i = 0; i < NACC / 4; ++i) {
      // residual pair (col, col + 1) of rows a and b: one 8-byte load each (N is even on this path)
      float2 ra = make_float2(0.f, 0.f), rb = ra;
      if constexpr (EVAL_BN) {
        if (p.residual != nullptr && c.n0 + 8 * i + col_in < p.N) {
          const float* r0 = p.residual + c.n0 + 8 * i + col_in;
          if (ok_a) ra = __ldg(reinterpret_cast<const float2*>(r0 + size_t(row_a) * p.ldr));
          if (ok_b) rb = __ldg(reinterpret_cast<const float2*>(r0 + size_t(row_b) * p.ldr));
        }
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = c.n0 + 8 * i + col_in + e;
        float va = acc[4 * i + e], vb = acc[4 * i + 2 + e];
        if (p.bias != nullptr && col < p.N) {
          const float b = __ldg(p.bias + col);
          va += b;
          vb += b;
        }
        if constexpr (EVAL_BN) {
          const float sc = colsum[8 * i + col_in + e], sh = colsum[BLOCK_N + 8 * i + col_in + e];
          va = fmaf(va, sc, sh) + (e ? ra.y : ra.x);
          vb = fmaf(vb, sc, sh) + (e ? rb.y : rb.x);
        }
        if (p.act) { va = elu1(va); vb = elu1(vb); }
        acc[4 * i + e] = ok_a ? va : 0.f;         // rows past M are clipped by the store and must not reach the statistics
        acc[4 * i + 2 + e] = ok_b ? vb : 0.f;
      }
    }
    if (p.stats != nullptr) {
      // this warp's 16 rows, summed per column, to its own slot: plain stores (a float atomicAdd to shared memory is a
      // compare-and-swap loop, and eight warps contend for every column)
      float* wsum = colsum + (4 * g + warp) * 2 * BLOCK_N;
#pragma unroll
      for (int i = 0; i < NACC / 4; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float va = acc[4 * i + e], vb = acc[4 * i + 2 + e];
          float s1 = va + vb, s2 = fmaf(va, va, vb * vb);
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {           // lanes with the same (lane & 3) hold the same column
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            s2 += __shfl_xor_sync(0xffffffffu, s2, o);
          }
          if (lane < 4) {
            wsum[8 * i + col_in + e] = s1;
            wsum[BLOCK_N + 8 * i + col_in + e] = s2;
          }
        }
      }
    }
    if (p.tma_store) {
      // registers -> 128B-swizzled staging boxes (32 rows x 32 floats) -> one bulk tensor store (or reduce-add) per box
#pragma unroll
      for (int c0 = 0; c0 < BLOCK_N; c0 += 32) {
        if (tid == 0) tma_store_wait_read();     // the previous chunk's stores have drained the staging boxes
        named_bar_sync(wg_bar, 128);
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          const int i = c0 / 8 + ii;
          const int cc = 8 * ii + col_in;        // column within the chunk (even)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = row_in + 8 * h;        // 0..63
            const int rr = r & 31;
            float* dst = stg + (r >> 5) * 1024 + rr * 32 + (((uint32_t(cc) >> 2) ^ uint32_t(rr & 7)) << 2) + (cc & 3);
            *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
          }
        }
        fence_proxy_async();
        named_bar_sync(wg_bar, 128);
        if (tid == 0) {
          const int pc = c.n0 + c0;
          for (int b = 0; b < 2; ++b) {
            const int row0 = c.m0 + 64 * g + 32 * b;
            if (row0 >= p.M || pc >= p.N) continue;
            const float* src = stg + b * 1024;
            if (p.shuffle_ci > 0) {
              const int phase = pc / p.shuffle_ci;   // packed channel (ph, pw, ci) of this chunk
              if (p.k_splits > 1) tma_reduce_add_5d(&tmap_c, src, pc - phase * p.shuffle_ci, phase & 1, 0, phase >> 1, row0 / p.W_out);
              else tma_store_5d(&tmap_c, src, pc - phase * p.shuffle_ci, phase & 1, 0, phase >> 1, row0 / p.W_out);
            } else if (p.k_splits > 1) {
              tma_reduce_add_2d(&tmap_c, src, pc, row0);
            } else {
              tma_store_2d(&tmap_c, src, pc, row0);
            }
          }
          tma_store_commit();
        }
      }
    } else {
      // outputs whose row pitch is not a multiple of 16 B (e.g. 10-class logits): direct stores from the fragments
#pragma unroll
      for (int i = 0; i < NACC / 4; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = h ? row_b : row_a;
          if (!(h ? ok_b : ok_a)) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = c.n0 + 8 * i + col_in + e;
            if (col >= p.N) continue;
            float* dst = p.out + size_t(row) * p.ldo + col;
            if (p.k_splits > 1) atomicAdd(dst, acc[4 * i + 2 * h + e]);
            else *dst = acc[4 * i + 2 * h + e];
          }
        }
      }
    }
    if (p.stats != nullptr) {
      named_bar_sync(3, 256);                    // every warp has stored its partials
      for (int j = threadIdx.x - 128; j < 2 * BLOCK_N; j += 256) {   // j < BLOCK_N: sums, else sums of squares
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += colsum[w * 2 * BLOCK_N + j];
        const int cc = j < BLOCK_N ? j : j - BLOCK_N;
        if (c.n0 + cc < p.N) atomicAdd(p.stats + (j < BLOCK_N ? 0 : p.N) + c.n0 + cc, v);
      }
      named_bar_sync(3, 256);                    // read before the next tile's partials overwrite them
    }
  }
  if (p.tma_store && tid == 0) tma_store_wait_read();   // shared memory must outlive the last bulk store's read
}

// ================================================================================================================
// Pixel-major convolution for C_out = 64 / 128: output channels on the wgmma M side, 256 output pixels on the N side.
// wgmma.m64n256k8 reads its 64-row weight operand and the 256-pixel activation operand from shared memory at
// 1/64 + 1/16 B per multiply-accumulate (against 4/N + 1/16 for the 128-pixel x N-channel tile above), and a stage of
// 64 or 128 weight rows + 256 pixels costs the TMA fill less shared-memory bandwidth per MAC as well.
// Same producer, ring protocol, tap packing and tile walk as igemm_wgmma_kernel; the stage is [pixels (A) | weights (B)].
//   C_out = 64  (ping-pong): each consumer warpgroup owns every other tile (64 ch x 256 px); one warpgroup's main loop
//               runs while the other one's epilogue does (the ring hands the stages out in tile order).
//   C_out = 128 (cooperative): warpgroup g computes channels [64 g, 64 g + 64) of every tile.
// Epilogue: plain store, plus the BatchNorm sum / sum of squares (IgemmParams::stats) when they are asked for.
// The [channel][pixel] fragment is transposed through 128B-swizzled 32 x 32 staging boxes into NHWC bulk tensor stores.
// Requires k_splits == 1, no bias / activation / eval-mode BatchNorm, and a 16-byte aligned output with ldo == C_out.
// ================================================================================================================
//
// Window reuse (WIN_KH = kh > 0; stride 1, dilation 1, C_in a multiple of 32, a tile = whole rows of one image, W_out * 128 B a
// multiple of the 1024-byte swizzle atom): filter rows r and r + 1 read the same pixels one image row apart, so a k-block is one
// (filter column s, 32-channel block) unit.  Its stage holds ONE box of tile rows + kh - 1 image rows at column shift s - pad
// (rows above / below the image zero-filled by the TMA unit) and the kh weight boxes of taps (0, s) .. (kh - 1, s); filter
// row r reads the window from image row r on, i.e. the wgmma B descriptor starts r * W_out * 128 B (whole swizzle atoms) later.
// Layer 1 of ResNet18 (64 channels, 32 x 32) moves 384 KB from L2 per tile instead of 720 KB.  The host runs it for C_out = 64
// (3 stages fit; at 128 channels 2 stages of 84 KB measured slower than the per-tap loop).
// ================================================================================================================
constexpr int PX_BLOCK_M = 256;     // output pixels per tile

template <int CO, int STAGES>
struct PixSmem {
  static constexpr int A_BYTES = PX_BLOCK_M * IG_BLOCK_K * 4;   // 32 KB of pixels
  static constexpr int B_BYTES = CO * IG_BLOCK_K * 4;           // 8 / 16 KB of weights
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGING_BYTES = 2 * 2 * 2 * 32 * 32 * 4; // per consumer warpgroup: two buffers of two 32 x 32 boxes
  static constexpr int BAR_BYTES = 2 * STAGES * 8;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + STAGING_BYTES + BAR_BYTES + 1024;  // + align slack
  // window reuse: the stage size depends on the shape (IgemmParams::win_stage_bytes)
  static constexpr int window_total(int stage_bytes) { return STAGES * stage_bytes + STAGING_BYTES + BAR_BYTES + 1024; }
};

// Window-reuse producer (one thread): per tile, per unit (s, cb): one 4-D box {32, W_out, win_rows, 1} of the input at
// (cb * 32, s - pad, h0 - pad, img) and KH 2-D weight boxes [C_out x 32] of taps (r, s), r = 0 .. KH - 1.
template <int CO, int STAGES, int KH>
__device__ __forceinline__ void igemm_produce_window(const IgemmParams& p, uint8_t* tiles, uint64_t* full_bar, uint64_t* empty_bar,
                                                     const CUtensorMap* tmap_a, const CUtensorMap* tmap_b) {
  constexpr uint32_t W_BOX = CO * IG_BLOCK_K * 4;
  const uint32_t stage_bytes = uint32_t(p.win_stage_bytes);
  int s = 0;
  uint32_t ph = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileCoord c = decode_tile(p, t, PX_BLOCK_M, CO);
    const int img = c.m0 / p.HW_out;
    const int h0 = (c.m0 - img * p.HW_out) / p.W_out - p.pad;
    for (int sx = 0; sx < p.taps_w; ++sx) {
      for (int cb = 0; cb < p.cblocks; ++cb) {
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* a_dst = tiles + s * stage_bytes;
        uint8_t* b_dst = a_dst + p.win_a_bytes;
        mbar_arrive_expect_tx(&full_bar[s], stage_bytes);
        tma_load_4d(a_dst, tmap_a, &full_bar[s], cb * IG_BLOCK_K, sx - p.pad, h0, img);
#pragma unroll
        for (int r = 0; r < KH; ++r)
          tma_load_2d(b_dst + r * W_BOX, tmap_b, &full_bar[s], (r * p.taps_w + sx) * p.b_cols_per_tap + cb * IG_BLOCK_K, 0);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  }
}

// WIN_KH = 0: the per-tap main loop; WIN_KH = kh > 0: window reuse for filters of kh rows (a compile-time count, so the
// kh x 4 MMAs of a unit are one unrolled run that ptxas issues back to back).
template <int CO, int STAGES, int WIN_KH>
__global__ void __launch_bounds__(IG_THREADS, 1)
igemm_wgmma_pix_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_c, const IgemmParams p) {
  using S = PixSmem<CO, STAGES>;
  constexpr bool WINDOW = WIN_KH > 0;
  static_assert(CO == 64 || CO == 128, "pixel-major tiles serve 64 or 128 output channels");
  static_assert(WINDOW || S::TOTAL <= 227 * 1024, "shared memory budget");   // window reuse: checked by the host
  static_assert(S::STAGE_BYTES % 1024 == 0, "stages must keep the 1024-byte swizzle alignment");
  constexpr bool PINGPONG = CO == 64;
  // bytes per ring stage; window reuse: [window | kh weight boxes]
  const uint32_t stage_bytes = WINDOW ? uint32_t(p.win_stage_bytes) : uint32_t(S::STAGE_BYTES);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* tiles = smem;
  float* staging = reinterpret_cast<float*>(smem + STAGES * stage_bytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * stage_bytes + S::STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_c);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PINGPONG ? 1 : 2);   // the tile's warpgroup / both warpgroups release a stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      if constexpr (WINDOW) igemm_produce_window<CO, STAGES, WIN_KH>(p, tiles, full_bar, empty_bar, &tmap_a, &tmap_b);
      else igemm_produce<PX_BLOCK_M, CO, STAGES, S::A_BYTES, S::STAGE_BYTES>(p, tiles, full_bar, empty_bar, &tmap_a, &tmap_b);
    }
    return;
  }
  setmaxnreg_inc<232>();

  const int g = wg - 1;
  const int warp = tid >> 5, lane = tid & 31;
  const int ch_wg = PINGPONG ? 0 : 64 * g;                       // first output channel of this warpgroup
  const uint32_t cwq = (p.cw == 8 || p.cw == 16) ? uint32_t(p.cw) : uint32_t(IG_BLOCK_K);
  const uint32_t mma_per_sub = cwq / IG_MMA_K;
  // wgmma A = the weight rows of this warpgroup's channels, wgmma B = the 256 pixel rows
  const uint32_t a_bytes = WINDOW ? uint32_t(p.win_a_bytes) : uint32_t(S::A_BYTES);
  const uint64_t adesc0 = make_kmajor_desc(smem_u32(tiles) + a_bytes + uint32_t(ch_wg) * cwq * 4u, cwq * 4u);
  const uint64_t bdesc0 = make_kmajor_desc(smem_u32(tiles), cwq * 4u);
  uint32_t a_off[IG_BLOCK_K / IG_MMA_K], b_off[IG_BLOCK_K / IG_MMA_K];
#pragma unroll
  for (int k = 0; k < IG_BLOCK_K / IG_MMA_K; ++k) {
    const uint32_t sub = uint32_t(k) / mma_per_sub, in = uint32_t(k) - sub * mma_per_sub;
    a_off[k] = (sub * uint32_t(CO) * cwq * 4u + in * 32u) >> 4;
    b_off[k] = (sub * uint32_t(PX_BLOCK_M) * cwq * 4u + in * 32u) >> 4;
  }
  float* stg = staging + g * 4096;            // [2 buffers][2 boxes][32 pixels][32 channels], chunk index XOR (pixel & 7)
  const uint32_t wg_bar = 1 + uint32_t(g);
  const int ch_lo = 16 * warp + (lane >> 2);  // channel (within the warpgroup's 64) of d[4i], d[4i+1]; d[4i+2..3]: + 8
  const int px_in = 2 * (lane & 3);           // pixel of d[4i] within its 8-pixel block

  float acc[128];
  const int step = PINGPONG ? 2 : 1;
  for (int j = PINGPONG ? g : 0, t = blockIdx.x + j * gridDim.x; t < p.total_tiles; j += step, t += step * gridDim.x) {
    const TileCoord c = decode_tile(p, t, PX_BLOCK_M, CO);
    // ring position of this tile's first k-block (window reuse: unit): every tile has num_k_blocks of them (no split-K)
    const uint32_t pos = uint32_t(j) * uint32_t(c.kb_count);
    int s = int(pos % STAGES);
    uint32_t ph = (pos / STAGES) & 1u;
    // Ping-pong: the main loops take turns (named barrier 3 + g: "warpgroup g may start").  A full-barrier parity wait
    // only tells the last two fills of a stage apart, so a warpgroup may wait on its k-blocks only once every k-block
    // before them has been waited on, i.e. once the other warpgroup's main loop has passed its last wait.  This holds
    // for any number of stages: the producer refills a stage only after the one consumer of its previous fill released it.
    if (PINGPONG && j > 0) named_bar_sync(3 + uint32_t(g), 256);
    int prev = -1;
    for (int i = 0; i < c.kb_count; ++i) {
      mbar_wait(&full_bar[s], ph);
      const uint64_t so = uint64_t(uint32_t(s) * (stage_bytes >> 4));
      wgmma_fence();
      wgmma_fence_acc(acc);
      if constexpr (WINDOW) {
        // filter row r: weight box r, and the window from image row r on (W_out * 128 B per row, in 16-byte units)
        const uint32_t px_row = uint32_t(p.W_out) * 8u;
#pragma unroll
        for (int r = 0; r < WIN_KH; ++r) {
          const uint64_t ao = so + uint32_t(r) * uint32_t(CO * 8), bo = so + uint32_t(r) * px_row;
#pragma unroll
          for (int k = 0; k < IG_BLOCK_K / IG_MMA_K; ++k)
            wgmma_tf32_n256(acc, adesc0 + ao + a_off[k], bdesc0 + bo + b_off[k], (i > 0 || r > 0 || k > 0) ? 1u : 0u);
        }
      } else {
#pragma unroll
        for (int k = 0; k < IG_BLOCK_K / IG_MMA_K; ++k)
          wgmma_tf32_n256(acc, adesc0 + so + a_off[k], bdesc0 + so + b_off[k], (i > 0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_fence_acc(acc);
      wgmma_wait<1>();
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
    // hand the turn to the other warpgroup if it has a next tile (every arrival meets exactly one wait)
    if (PINGPONG && t + gridDim.x < p.total_tiles) named_bar_arrive(4 - uint32_t(g), 256);
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);

    // ---- epilogue.  Pixels past M (last tile of an odd batch) must not reach the statistics; the store clips them.
    if (c.m0 + PX_BLOCK_M > p.M) {
#pragma unroll
      for (int i = 0; i < 32; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (c.m0 + 8 * i + px_in + e >= p.M) { acc[4 * i + e] = 0.f; acc[4 * i + 2 + e] = 0.f; }
    }
    if (p.stats != nullptr) {
      // a row of the fragment is one channel: sum inside the thread, then over the 4 lanes of the quad
      float s1a = 0.f, s2a = 0.f, s1b = 0.f, s2b = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float va = acc[4 * i + e], vb = acc[4 * i + 2 + e];
          s1a += va; s2a = fmaf(va, va, s2a);
          s1b += vb; s2b = fmaf(vb, vb, s2b);
        }
      }
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        s1a += __shfl_xor_sync(0xffffffffu, s1a, o);
        s2a += __shfl_xor_sync(0xffffffffu, s2a, o);
        s1b += __shfl_xor_sync(0xffffffffu, s1b, o);
        s2b += __shfl_xor_sync(0xffffffffu, s2b, o);
      }
      if ((lane & 3) == 0) {
        const int ca = ch_wg + ch_lo;
        atomicAdd(p.stats + ca, s1a);
        atomicAdd(p.stats + p.N + ca, s2a);
        atomicAdd(p.stats + ca + 8, s1b);
        atomicAdd(p.stats + p.N + ca + 8, s2b);
      }
    }
    // 8 chunks of 32 pixels x 64 channels, double-buffered: a buffer is rewritten once the stores of two chunks ago have read it
#pragma unroll
    for (int q = 0; q < PX_BLOCK_M / 32; ++q) {
      float* buf = stg + (q & 1) * 2048;
      if (tid == 0) tma_store_wait_read_n<1>();
      named_bar_sync(wg_bar, 128);
#pragma unroll
      for (int ii = 0; ii < 4; ++ii) {
        const int i = 4 * q + ii;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ch = ch_lo + 8 * h;                   // 0..63
          const int cc = ch & 31;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int px = 8 * ii + px_in + e;            // 0..31: the staging row
            buf[(ch >> 5) * 1024 + px * 32 + (((uint32_t(cc) >> 2) ^ uint32_t(px & 7)) << 2) + (cc & 3)] = acc[4 * i + 2 * h + e];
          }
        }
      }
      fence_proxy_async();
      named_bar_sync(wg_bar, 128);
      if (tid == 0) {
        const int row0 = c.m0 + 32 * q;
        if (row0 < p.M) {
#pragma unroll
          for (int b = 0; b < 2; ++b) tma_store_2d(&tmap_c, buf + b * 1024, ch_wg + 32 * b, row0);
        }
        tma_store_commit();
      }
    }
  }
  if (tid == 0) tma_store_wait_read();   // shared memory must outlive the last bulk store's read
}

}  // namespace fedb200

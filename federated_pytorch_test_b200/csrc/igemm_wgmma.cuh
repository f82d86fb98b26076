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
//     memory, one atomicAdd per channel per tile);
//   * output through a 128B-swizzled staging tile and bulk tensor stores (reduce-adds for split-K / accumulation), or
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
  int accumulate;        // out += result (bulk reduce-add / atomics) instead of out = result; no memset
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
  int shuffle_ci;        // > 0: the N columns are (ph, pw, ci) phase-packed channels of a stride-2 data gradient /
                         // transposed conv; each 32 x 32 chunk is stored to out[n, 2 ho + ph, 2 wo + pw, ci0 .. ci0 + 31] through a
                         // 5-D tensor map (no separate pixel-shuffle pass).  shuffle_ci = channels of the shuffled output.
};

template <int BLOCK_N, int STAGES>
struct IgemmSmem {
  static constexpr int A_BYTES = IG_BLOCK_M * IG_BLOCK_K * 4;   // 16 KB
  static constexpr int B_BYTES = BLOCK_N * IG_BLOCK_K * 4;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;         // one k-block: [A | B]
  static constexpr int STAGING_BYTES = 2 * 64 * 32 * 4;         // per consumer warpgroup: two 32 x 32 output boxes
  static constexpr int STATS_BYTES = 2 * BLOCK_N * 4;           // column partials (sum, sumsq) of the current tile
  static constexpr int BAR_BYTES = 2 * STAGES * 8;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + STAGING_BYTES + STATS_BYTES + BAR_BYTES + 1024;  // + align slack
};

struct TileCoord {
  int m0, n0, kb_begin, kb_count;
};
__device__ __forceinline__ TileCoord decode_tile(const IgemmParams& p, int t, int block_n) {
  const int n_idx = t % p.n_tiles;
  const int rest = t / p.n_tiles;
  const int m_idx = rest % p.m_tiles;
  const int z = rest / p.m_tiles;
  TileCoord c;
  c.m0 = m_idx * IG_BLOCK_M;
  c.n0 = n_idx * block_n;
  c.kb_begin = z * p.kb_per_split;
  c.kb_count = min(p.kb_per_split, p.num_k_blocks - c.kb_begin);
  return c;
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

template <int BLOCK_N, int STAGES>
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
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(colsum + 2 * BLOCK_N);
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
  for (int i = threadIdx.x; i < 2 * BLOCK_N; i += IG_THREADS) colsum[i] = 0.f;
  __syncthreads();
  pdl_wait();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
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
        const TileCoord c = decode_tile(p, t, BLOCK_N);
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
          uint8_t* a_dst = tiles + s * S::STAGE_BYTES;
          uint8_t* b_dst = a_dst + S::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], uint32_t(S::STAGE_BYTES));
          if (cwp) {
            // tpk taps per k-block, each a [128 rows x cwp channels] sub-tile of A and a [BLOCK_N x cwp] sub-tile of B
            const int sub_a = IG_BLOCK_M * cwp * 4, sub_b = BLOCK_N * cwp * 4;
            for (int jt = 0; jt < tpk; ++jt) {
              const int tp = kb * tpk + jt;
              const bool real = tp < p.taps_total;
              int cw = 0, ch = 0;
              if (real) tap_offset(tp / p.taps_w, tp % p.taps_w, cw, ch);
              // a tap past the filter: image index out of range -> zeros
              tma_load_4d(a_dst + jt * sub_a, &tmap_a, &full_bar[s], 0, cw, h0 + ch, real ? img : img_oob);
              tma_load_2d(b_dst + jt * sub_b, &tmap_b, &full_bar[s], real ? tp * p.b_cols_per_tap : col_oob, c.n0);
            }
          } else {
            int cw, ch;
            tap_offset(r, sx, cw, ch);
            if (p.is_conv)
              tma_load_4d(a_dst, &tmap_a, &full_bar[s], cb * IG_BLOCK_K, cw, h0 + ch, img);
            else
              tma_load_2d(a_dst, &tmap_a, &full_bar[s], kb * IG_BLOCK_K, c.m0);
            tma_load_2d(b_dst, &tmap_b, &full_bar[s], (r * p.taps_w + sx) * p.b_cols_per_tap + cb * IG_BLOCK_K, c.n0);
            if (++cb == p.cblocks) {
              cb = 0;
              if (++sx == p.taps_w) { sx = 0; ++r; }
            }
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
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
    const TileCoord c = decode_tile(p, t, BLOCK_N);
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
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = c.n0 + 8 * i + col_in + e;
        float va = acc[4 * i + e], vb = acc[4 * i + 2 + e];
        if (p.bias != nullptr && col < p.N) {
          const float b = __ldg(p.bias + col);
          va += b;
          vb += b;
        }
        if (p.act) { va = elu1(va); vb = elu1(vb); }
        acc[4 * i + e] = ok_a ? va : 0.f;         // rows past M are clipped by the store and must not reach the statistics
        acc[4 * i + 2 + e] = ok_b ? vb : 0.f;
      }
    }
    if (p.stats != nullptr) {
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
            atomicAdd(&colsum[8 * i + col_in + e], s1);
            atomicAdd(&colsum[BLOCK_N + 8 * i + col_in + e], s2);
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
            } else if (p.k_splits > 1 || p.accumulate) {
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
            if (p.k_splits > 1 || p.accumulate) atomicAdd(dst, acc[4 * i + 2 * h + e]);
            else *dst = acc[4 * i + 2 * h + e];
          }
        }
      }
    }
    if (p.stats != nullptr) {
      named_bar_sync(3, 256);                    // both warpgroups have added their partials
      for (int cc = threadIdx.x - 128; cc < BLOCK_N; cc += 256) {
        if (c.n0 + cc < p.N) {
          atomicAdd(p.stats + c.n0 + cc, colsum[cc]);
          atomicAdd(p.stats + p.N + c.n0 + cc, colsum[BLOCK_N + cc]);
        }
        colsum[cc] = 0.f;
        colsum[BLOCK_N + cc] = 0.f;
      }
      named_bar_sync(3, 256);                    // zeroed before the next tile adds to it
    }
  }
  if (p.tma_store && tid == 0) tma_store_wait_read();   // shared memory must outlive the last bulk store's read
}

}  // namespace fedb200

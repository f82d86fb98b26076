// Fused block collectives over NVLink peer memory — FedAvg / FedProx / consensus-ADMM aggregation as ONE kernel
// (SURVEY G17-G20, §5.8).  No NCCL on this path, no host involvement inside a round (CUDA-graph capturable: the epoch,
// the penalty rho and every accumulator live in device memory; nothing is memset or cloned per call).
//
// Every replica's parameter block is a slice of a flat arena that is mapped into every process (symmetric memory:
// CUDA VMM/IPC peer mappings, bound to an NVSwitch multicast object when the fabric supports it).  The kernel gets the
// slice pointers of ALL K replicas (its own and its peers') and runs
//
//   A. per-CTA flag barrier with the same-numbered CTA of every peer: the inputs of every rank are final
//   1. reduce.  ONE-SHOT (small blocks): every rank reduces the whole vector out of peer memory — one
//      `multimem.ld_reduce.add.v4.f32` on the multicast address (the sum is formed inside the switch) or K
//      `ld.relaxed.sys.v4` loads — scales it, stores the new consensus vector z locally and accumulates ||z_old - z||^2.
//      TWO-SHOT (blocks >= 256 KB, one replica per rank): rank r reduces only slice r and BROADCASTS the result with
//      `multimem.st` (or P2P stores) straight into every rank's weights (FedAvg) or consensus vector (FedProx/ADMM):
//      per-GPU NVLink traffic n*4*(K-1)/K bytes in + out instead of n*4*(K-1) bytes in.
//   B. per-CTA flag barrier: every peer has finished reading my x / y and its broadcast has landed here
//   2. local epilogue in place: FedAvg writes z back into every local replica (one-shot) or copies the broadcast
//      weights into z (two-shot); FedProx accumulates ||rho (x - z)||^2; ADMM performs the dual ascent
//      y += rho (x - z) and accumulates the same norm
//   C. the last CTA to finish exchanges the round's statistics through the control pads (FedProx/ADMM: dual part,
//      primal part, #non-finite; DP, compressed and SecAgg rounds: their own statistics) and writes the result record.
//
// CTA b works on the SAME index set on every rank and in both passes, so barriers A and B only involve CTA b of each
// rank (threads 0..world-1 signal / poll one peer each): there is no grid-wide barrier in the kernel.
//
// mode: 0 = FedAvg (z = sum x / K, write-back), 1 = FedProx (no write-back), 2 = ADMM (z = sum(y + rho x)/(K rho)).
// A second instantiation (FEDOPT) runs FedAvg with a server optimizer (FedAvgM / FedAdagrad / FedAdam / FedYogi) between
// the reduction and the write-back.  DP instantiations add DP-FedAvg's Gaussian noise to the mean, after dp_clip_kernel
// (end of file) has clipped the workers' updates.  Compressed instantiations (QBITS) reduce stochastically rounded 8- / 4-bit
// codes of the workers' updates, which every rank encodes for its own replicas before barrier A.  Sampled instantiations
// (SAMP) average only the round's participants, weighted by their sample counts, reading them over P2P.  Secure-aggregation
// instantiations (QBITS = SA_QBITS) sum pairwise ChaCha20-masked fixed-point codes, whose masks cancel in the sum.
// Reference sites: /root/reference/src/federated_multi.py:203-217, fedprox_multi.py:211-232, consensus_multi.py:242-299.
#include "fedb200.h"

#include <cooperative_groups.h>
#include <stdexcept>
#include <string>
#include <type_traits>

namespace cg = cooperative_groups;

namespace fedb200 {

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_sys_v4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float ld_sys_f32(const float* p) {
  float v;
  asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_sys_v4(float* p, float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_sys_f32(float* p, float v) {
  asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// in-switch reduction over all devices bound to the multicast object
__device__ __forceinline__ float4 multimem_ld_reduce_v4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ float multimem_ld_reduce_f32(const float* mc) {
  float v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f32 %0, [%1];" : "=f"(v) : "l"(mc) : "memory");
  return v;
}
// one store, replicated by the switch into the same offset of every device bound to the multicast object
__device__ __forceinline__ void multimem_st_v4(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ float warp_add(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float block_add(float v, float* sm) {
  v = warp_add(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.f;
    r = warp_add(r);
  }
  __syncthreads();
  return r;  // valid in thread 0
}

// Poll a flag until it reaches `epoch`.  A timeout does not trap (that would kill the CUDA context, ADVICE r1): it is
// reported through the status word and the kernel runs to its end so that the host can raise a proper error.
__device__ __forceinline__ bool wait_flag(const uint32_t* flag, uint32_t epoch, long long limit) {
  const long long t0 = clock64();
  int spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(flag) - epoch) < 0) {
    if ((++spins & 63) == 0 && clock64() - t0 > limit) return false;
  }
  return true;
}

// Barrier between CTA `blockIdx.x` of this rank and the same CTA of every peer.  `row` = PAD_FLAG_A / PAD_FLAG_B.
// Callers have executed __threadfence_system() after any store the peers must observe.
__device__ __forceinline__ void cta_peer_barrier(uint32_t* const* ctrl, int world, int rank, int row, uint32_t epoch,
                                                 long long limit, float* status, int* s_abort) {
  if (world <= 1) return;
  __syncthreads();
  if (threadIdx.x < world && *s_abort == 0) {
    const int peer = threadIdx.x;
    st_release_sys(ctrl[peer] + row + blockIdx.x * COMM_MAX_WORLD + rank, epoch);
    if (!wait_flag(ctrl[rank] + row + blockIdx.x * COMM_MAX_WORLD + peer, epoch, limit)) {
      *status = 100.f + float(peer);      // names the missing rank (SURVEY §5.3)
      atomicExch(s_abort, 1);
    }
  }
  __syncthreads();
}

// One-off exchange with every peer on flag row `row` (PAD_FLAG_C / PAD_FLAG_D), run by threads 0..world-1 after each has
// written its payload into peer threadIdx.x's pad: publish the payload, signal that peer, and wait for its signal.
__device__ __forceinline__ void peer_post_wait(uint32_t* const* ctrl, int rank, int row, uint32_t epoch, long long limit,
                                               float* status, int* s_abort) {
  const int peer = threadIdx.x;
  __threadfence_system();
  st_release_sys(ctrl[peer] + row + rank, epoch);
  if (*s_abort == 0 && !wait_flag(ctrl[rank] + row + peer, epoch, limit)) {
    *status = 100.f + float(peer);
    atomicExch(s_abort, 1);
  }
}

// the dual residual ||zo - zn||^2 and the non-finite count of the new values zn, accumulated over one float4
__device__ __forceinline__ void dual_nan_v4(float4 zo, float4 zn, float& dual, float& bad) {
  const float dx = zo.x - zn.x, dy = zo.y - zn.y, dz = zo.z - zn.z, dw = zo.w - zn.w;
  dual = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, dual))));
  if (!(isfinite(zn.x) && isfinite(zn.y) && isfinite(zn.z) && isfinite(zn.w))) bad += 1.f;
}

// two-shot broadcast of a float4 into the same offset of every rank: multimem.st when a multicast address is bound, else
// P2P stores
__device__ __forceinline__ void bcast_v4(float* mc, float* const* w, int world, size_t off, float4 v) {
  if (mc != nullptr) multimem_st_v4(mc + off, v);
  else for (int p = 0; p < world; ++p) st_sys_v4(w[p] + off, v);
}

// sum over all K workers of x_k (+ y_k / rho-scaled for ADMM) at float4 index `off`: one in-switch reduction or K peer loads
__device__ __forceinline__ float4 gather_v4(const CommArgs& a, size_t off, float rho, bool use_mc) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (use_mc) {
    acc = multimem_ld_reduce_v4(a.mc_x + off);
    if (a.mode == 2) {
      const float4 ys = multimem_ld_reduce_v4(a.mc_y + off);
      acc.x = fmaf(rho, acc.x, ys.x); acc.y = fmaf(rho, acc.y, ys.y);
      acc.z = fmaf(rho, acc.z, ys.z); acc.w = fmaf(rho, acc.w, ys.w);
    }
  } else {
#pragma unroll 4
    for (int k = 0; k < a.K; ++k) {
      const float4 xv = ld_sys_v4(a.x[k] + off);
      if (a.mode == 2) {
        const float4 yv = ld_sys_v4(a.y[k] + off);
        acc.x += fmaf(rho, xv.x, yv.x); acc.y += fmaf(rho, xv.y, yv.y);
        acc.z += fmaf(rho, xv.z, yv.z); acc.w += fmaf(rho, xv.w, yv.w);
      } else {
        acc.x += xv.x; acc.y += xv.y; acc.z += xv.z; acc.w += xv.w;
      }
    }
  }
  return acc;
}

// Server optimizer step on one element (Reddi et al. 2021, Algorithm 2, no bias correction; FedAvgM: Hsu et al. 2019).
// d = mean - z is the round's pseudo-gradient; m and v are updated in place; returns the new server model.
__device__ __forceinline__ float fedopt_step(const CommArgs& a, float z, float mean, float& m, float& v) {
  const float d = mean - z;
  if (a.opt == FEDOPT_AVGM) {                       // z + lr m, evaluated as mean + (lr m - d): exactly FedAvg's mean when
    m = fmaf(a.beta1, m, d);                        // beta = 0 and lr = 1
    return mean + fmaf(a.lr, m, -d);
  }
  m = fmaf(a.beta1, m, (1.f - a.beta1) * d);
  const float d2 = d * d;
  if (a.opt == FEDOPT_ADAGRAD) {
    v += d2;
  } else if (a.opt == FEDOPT_ADAM) {
    v = fmaf(a.beta2, v, (1.f - a.beta2) * d2);
  } else {                                          // yogi: v - (1 - beta2) d^2 sign(v - d^2)
    const float s = v > d2 ? 1.f : (v < d2 ? -1.f : 0.f);
    v = fmaf(-(1.f - a.beta2) * d2, s, v);
  }
  return fmaf(a.lr, m / (sqrtf(v) + a.tau), z);
}
__device__ __forceinline__ float4 fedopt_step_v4(const CommArgs& a, float4 z, float4 mean, float4& m, float4& v) {
  return make_float4(fedopt_step(a, z.x, mean.x, m.x, v.x), fedopt_step(a, z.y, mean.y, m.y, v.y),
                     fedopt_step(a, z.z, mean.z, m.z, v.z), fedopt_step(a, z.w, mean.w, m.w, v.w));
}

// ---- robust aggregation: coordinate-wise median / trimmed mean (Yin et al. 2018) --------------------------------------
// Batcher's odd-even merge sort network on P = 4 / 8 / 16 values, as a compile-time comparator list (5 / 19 / 63
// compare-exchanges).  The loops below unroll completely, so every index is a constant and the values stay in registers.
template <int P>
struct OddEvenMergeNet {
  int n = 0;
  int lo[P * P] = {};
  int hi[P * P] = {};
  constexpr OddEvenMergeNet() {
    for (int p = 1; p < P; p <<= 1)
      for (int k = p; k >= 1; k >>= 1)
        for (int j = k % p; j + k < P; j += 2 * k)
          for (int i = 0; i < k && i + j + k < P; ++i)
            if ((i + j) / (2 * p) == (i + j + k) / (2 * p)) {
              lo[n] = i + j;
              hi[n] = i + j + k;
              ++n;
            }
  }
};

// NaN orders as +inf, +-inf keep their sign: NaN / Inf in at most trim_b workers (median: fewer than half) cannot reach
// the aggregate.
__device__ __forceinline__ float robust_canon(float x) { return isnan(x) ? __int_as_float(0x7f800000) : x; }

// Sorts v[0..P) (the K inputs, padded with +inf) and returns the rule's aggregate.  median: the middle value for odd K,
// (lo + hi) * 0.5 of the two middle values for even K (np.median).  trimmed mean: the sum of the sorted values
// trim_b .. K - trim_b - 1 in ascending order, divided (correctly rounded) by K - 2 trim_b (scipy.stats.trim_mean); only
// the kept values are summed, so an extreme value cannot cancel against the rest.
template <int P>
__device__ __forceinline__ float robust_select(const CommArgs& a, float (&v)[P]) {
  constexpr OddEvenMergeNet<P> net{};
#pragma unroll
  for (int c = 0; c < net.n; ++c) {
    const float x = v[net.lo[c]], y = v[net.hi[c]];
    v[net.lo[c]] = fminf(x, y);
    v[net.hi[c]] = fmaxf(x, y);
  }
  if (a.agg == AGG_MEDIAN) {
    const int ilo = (a.K - 1) >> 1, ihi = a.K >> 1;
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int j = 0; j < P; ++j) {
      if (j == ilo) lo = v[j];
      if (j == ihi) hi = v[j];
    }
    return (a.K & 1) ? hi : (lo + hi) * 0.5f;
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < P; ++j)
    if (j >= a.trim_b && j < a.K - a.trim_b) s += v[j];
  return __fdiv_rn(s, float(a.K - 2 * a.trim_b));
}

// the rule's aggregate over all K workers at float4 index `off`: K peer loads (never the multicast address), then one
// sort per lane
template <int P>
__device__ __forceinline__ float4 robust_gather_v4(const CommArgs& a, size_t off) {
  float vx[P], vy[P], vz[P], vw[P];
  const float inf = __int_as_float(0x7f800000);
#pragma unroll
  for (int k = 0; k < P; ++k) {
    float4 xv = make_float4(inf, inf, inf, inf);
    if (k < a.K) xv = ld_sys_v4(a.x[k] + off);
    vx[k] = robust_canon(xv.x); vy[k] = robust_canon(xv.y); vz[k] = robust_canon(xv.z); vw[k] = robust_canon(xv.w);
  }
  return make_float4(robust_select<P>(a, vx), robust_select<P>(a, vy), robust_select<P>(a, vz), robust_select<P>(a, vw));
}
template <int P>
__device__ __forceinline__ float robust_gather_f32(const CommArgs& a, int i) {
  float v[P];
#pragma unroll
  for (int k = 0; k < P; ++k) v[k] = k < a.K ? robust_canon(ld_sys_f32(a.x[k] + i)) : __int_as_float(0x7f800000);
  return robust_select<P>(a, v);
}

// AGG_PAD = 0: the mean (sum; scaled by the caller).  AGG_PAD = 4 / 8 / 16: the robust rule on K <= AGG_PAD inputs.
template <int AGG_PAD>
__device__ __forceinline__ float4 reduce_v4(const CommArgs& a, size_t off, float rho, bool use_mc) {
  if constexpr (AGG_PAD == 0) return gather_v4(a, off, rho, use_mc);
  else return robust_gather_v4<AGG_PAD>(a, off);
}

// ---- DP-FedAvg noise: counter-based standard normals (Box-Muller on splitmix64 words) ----------------------------------
// Coordinates 2p and 2p + 1 of DP round t share the word w = F(F(key + (t + 1) G) + (p + 1) G), arithmetic mod 2^64, with
// F the splitmix64 finaliser and G = 0x9E3779B97F4A7C15.  u1 = (w[63:40] + 1) 2^-24 in (0, 1], u2 = w[23:0] 2^-24 in
// [0, 1), r = sqrt(-2 ln u1):  xi_2p = r cos(2 pi u2),  xi_2p+1 = r sin(2 pi u2).  algo/privacy.py (dp_noise) is the
// float64 numpy oracle.  The draw depends on (key, t, i) only: every rank, one-shot or two-shot, adds the same noise.
constexpr uint64_t DP_GAMMA = 0x9E3779B97F4A7C15ull;
__device__ __forceinline__ uint64_t dp_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ float2 dp_normal_pair(uint64_t round_key, uint64_t p) {
  const uint64_t w = dp_mix(round_key + (p + 1ull) * DP_GAMMA);
  // in double precision: the extension is built with --use_fast_math, whose single-precision log / sincos intrinsics
  // are off by ~1e-4 in the tails; rounded once to float, xi is within an ulp of the float64 oracle
  const double u1 = double((w >> 40) + 1ull) * 5.9604644775390625e-8;      // exact: 24-bit integers times 2^-24
  const double u2 = double(w & 0xFFFFFFull) * 5.9604644775390625e-8;
  const double r = sqrt(-2.0 * log(u1));
  double s, c;
  sincospi(2.0 * u2, &s, &c);
  return make_float2(float(r * c), float(r * s));
}
// DP: the mean plus dp_std * xi at float4 index `off` (a multiple of 4: coordinate pairs off / 2 and off / 2 + 1) or at
// coordinate i, in the round t = *dp_t the kernel was launched for (the last CTA advances it only after every CTA is done).
// Alignment padding (dp_valid) gets no noise.  (The kernel calls these through `DP ? noised : mean`, which keeps the other
// instantiations' code exactly as it was.)
__device__ __forceinline__ uint64_t dp_round_key(const CommArgs& a) {
  return dp_mix(a.dp_key + uint64_t(*a.dp_t + 1) * DP_GAMMA);
}
// noise std of coordinate i: dp_std for a parameter, 0 for padding
__device__ __forceinline__ float dp_std_at(const CommArgs& a, size_t i) {
  if (a.dp_valid == nullptr) return a.dp_std;
  return int(i % DP_CHUNK) < int(a.dp_valid[i / DP_CHUNK]) ? a.dp_std : 0.f;
}
template <bool DP>
__device__ __forceinline__ float4 dp_noised_v4(const CommArgs& a, size_t off, float4 mean) {
  const uint64_t key = dp_round_key(a);
  const float2 g0 = dp_normal_pair(key, off >> 1), g1 = dp_normal_pair(key, (off >> 1) + 1);
  return make_float4(fmaf(dp_std_at(a, off), g0.x, mean.x), fmaf(dp_std_at(a, off + 1), g0.y, mean.y),
                     fmaf(dp_std_at(a, off + 2), g1.x, mean.z), fmaf(dp_std_at(a, off + 3), g1.y, mean.w));
}
template <bool DP>
__device__ __forceinline__ float dp_noised_f32(const CommArgs& a, int i, float mean) {
  const float2 g = dp_normal_pair(dp_round_key(a), uint64_t(i >> 1));
  return fmaf(dp_std_at(a, size_t(i)), (i & 1) ? g.y : g.x, mean);
}

// ---- compressed client updates: stochastic QBITS-bit codes with one scale per Q_GROUP coordinates ----------------------
// (QSGD, Alistarh et al. 2017; FedPAQ, Reisizadeh et al. 2020; error feedback, Seide et al. 2014, Karimireddy et al. 2019)
// Worker k's update u = x_k - z (+ e_k) is cut into groups of Q_GROUP coordinates counted from the block start.  A group's
// scale is s = max|u| / L (L = 127 or 7) and its codes are q = clamp(floor(u / s + U), -L, L), U in [0, 1) the
// counter-based uniform of (key, k, t, i), so E[q s] = u.  A group holding a non-finite u gets s = NaN (fmaxf alone would
// drop a NaN) and codes 0: its dequantized values are NaN and the NaN guard fires.  An all-zero group gets s = 0, codes 0.
// Every float operation that decides a code is correctly rounded (the extension is built with --use_fast_math), so the
// codes equal the float32 numpy oracle (algo/compress.py: quantize) bit for bit.
// Coordinates 2p and 2p + 1 share the word w = F(F(F(key + (t + 1) G) + (k + 1) G) + (p + 1) G) (F, G as for the DP
// noise):  U_2p = w[63:40] 2^-24,  U_2p+1 = w[23:0] 2^-24.
//
// Work is split in tiles of COMM_THREADS * Q_SEG coordinates (64 groups) from the start of each slice (slices are whole
// groups); CTA b takes tiles b, b + grid, ... and thread i the Q_SEG coordinates at 16 i of a tile in the encoder, in the
// reduction and in the write-back alike.  So CTA b of every rank encodes exactly the groups CTA b of any peer reads, and
// the per-CTA barriers A and B cover the payload as they cover the floats.
constexpr int Q_TILE = COMM_THREADS * Q_SEG;
static_assert(Q_GROUP % Q_SEG == 0 && Q_TILE % Q_GROUP == 0, "a tile must hold whole groups");

__device__ __forceinline__ uint4 ld_sys_u32x4(const void* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ld_sys_u32x2(const void* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
// float4 at coordinate c (a multiple of 4) of a length-n slice: coordinates >= n read as 0 and are never written
__device__ __forceinline__ float4 q_ld4(const float* p, int c, int n) {
  if (c + 4 <= n) return *reinterpret_cast<const float4*>(p + c);
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = c + i < n ? p[c + i] : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ float4 q_ld4_sys(const float* p, int c, int n) {
  if (c + 4 <= n) return ld_sys_v4(p + c);
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = c + i < n ? ld_sys_f32(p + c + i) : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void q_st4(float* p, int c, int n, float4 v) {
  if (c + 4 <= n) {
    *reinterpret_cast<float4*>(p + c) = v;
    return;
  }
  const float w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (c + i < n) p[c + i] = w[i];
}
// bcast_v4 at coordinate c (a multiple of 4) of a length-n slice: coordinates >= n are not written
__device__ __forceinline__ void q_bcast4(float* mc, float* const* w, int world, int c, int n, float4 v) {
  if (c + 4 <= n) {
    bcast_v4(mc, w, world, size_t(c), v);
    return;
  }
  const float s[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (c + i < n) for (int p = 0; p < world; ++p) st_sys_f32(w[p] + c + i, s[i]);
}
__device__ __forceinline__ float4 q_f4(const float* v, int q) { return make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]); }
__device__ __forceinline__ void q_unf4(float* v, int q, float4 t) { v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }

// Slice s of a compressed round: whole groups (top-k rounds: whole tiles, unit = Q_TILE), coordinates [lo, hi).
struct QSlice {
  int lo, hi;
};
__device__ __forceinline__ QSlice q_slice(const CommArgs& a, int s, int unit = Q_GROUP) {
  const int ng = (a.n + unit - 1) / unit;
  const int per = a.two_shot ? (ng + a.world - 1) / a.world : ng;
  return {min(a.n, s * per * unit), min(a.n, (s + 1) * per * unit)};
}

// Phase 0: encode the local replicas' updates on this CTA's tiles of every slice, update e_j, and accumulate this
// thread's part of sum_j ||u_j - q_j s_j||^2 (err) and sum_j ||u_j||^2 (nrm).
template <int QBITS>
__device__ __forceinline__ void q_encode(const CommArgs& a, int nslices, float& err, float& nrm) {
  constexpr float L = QBITS == 8 ? 127.f : 7.f;
  const float inf = __int_as_float(0x7f800000);
  for (int s = 0; s < nslices; ++s) {
    const QSlice sl = q_slice(a, s);
    for (int tb = sl.lo + blockIdx.x * Q_TILE; tb < sl.hi; tb += gridDim.x * Q_TILE) {   // uniform across the CTA
      const int c0 = tb + Q_SEG * threadIdx.x;
      const bool active = c0 < sl.hi;
      float zv[Q_SEG];
#pragma unroll
      for (int q = 0; q < Q_SEG / 4; ++q) q_unf4(zv, q, active ? q_ld4(a.z, c0 + 4 * q, a.n) : make_float4(0.f, 0.f, 0.f, 0.f));
      for (int j = 0; j < a.n_local; ++j) {
        const int k = a.q_worker[j];
        float* ef = a.q_ef[j];
        float u[Q_SEG];
        float amax = 0.f;                          // +inf: the group holds a non-finite u
#pragma unroll
        for (int q = 0; q < Q_SEG / 4; ++q) {
          const float4 xv = active ? q_ld4(a.xl[j], c0 + 4 * q, a.n) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 ev = active && ef != nullptr ? q_ld4(ef, c0 + 4 * q, a.n) : make_float4(0.f, 0.f, 0.f, 0.f);
          u[4 * q + 0] = __fadd_rn(__fsub_rn(xv.x, zv[4 * q + 0]), ev.x);
          u[4 * q + 1] = __fadd_rn(__fsub_rn(xv.y, zv[4 * q + 1]), ev.y);
          u[4 * q + 2] = __fadd_rn(__fsub_rn(xv.z, zv[4 * q + 2]), ev.z);
          u[4 * q + 3] = __fadd_rn(__fsub_rn(xv.w, zv[4 * q + 3]), ev.w);
        }
#pragma unroll
        for (int i = 0; i < Q_SEG; ++i) amax = isfinite(u[i]) ? fmaxf(amax, fabsf(u[i])) : inf;
        // the Q_GROUP / Q_SEG = 8 threads of a group are adjacent lanes of one warp
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
        const float sc = amax == inf ? __int_as_float(0x7fc00000) : __fdiv_rn(amax, L);
        const bool coded = sc > 0.f && sc != inf;  // false for s = 0 and s = NaN: codes 0
        const uint64_t wkey = dp_mix(dp_mix(a.q_key + uint64_t(*a.q_t + 1) * DP_GAMMA) + uint64_t(k + 1) * DP_GAMMA);
        uint32_t packed[QBITS * Q_SEG / 32];
#pragma unroll
        for (int w = 0; w < QBITS * Q_SEG / 32; ++w) packed[w] = 0u;
#pragma unroll
        for (int p = 0; p < Q_SEG / 2; ++p) {
          const uint64_t w = dp_mix(wkey + uint64_t((c0 >> 1) + p + 1) * DP_GAMMA);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int i = 2 * p + h;
            const float U = float(uint32_t(h ? (w & 0xFFFFFFull) : (w >> 40))) * 5.9604644775390625e-8f;   // exact
            int q = 0;
            if (coded) q = int(fminf(fmaxf(floorf(__fadd_rn(__fdiv_rn(u[i], sc), U)), -L), L));
            const float e = __fsub_rn(u[i], __fmul_rn(float(q), sc));
            err = fmaf(e, e, err);
            nrm = fmaf(u[i], u[i], nrm);
            u[i] = e;
            packed[i * QBITS / 32] |= (uint32_t(q) & ((1u << QBITS) - 1u)) << ((i * QBITS) % 32);
          }
        }
        if (!active) continue;
        if constexpr (QBITS == 8)
          *reinterpret_cast<uint4*>(a.q_codes[k] + c0) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
        else
          *reinterpret_cast<uint2*>(a.q_codes[k] + c0 / 2) = make_uint2(packed[0], packed[1]);
        if ((threadIdx.x & (Q_GROUP / Q_SEG - 1)) == 0) a.q_scales[k][c0 / Q_GROUP] = sc;
        if (ef != nullptr) {
#pragma unroll
          for (int q = 0; q < Q_SEG / 4; ++q) q_st4(ef, c0 + 4 * q, a.n, q_f4(u, q));
        }
      }
    }
  }
}

// ---- secure aggregation: pairwise ChaCha20-masked fixed-point updates (SecAgg, Bonawitz et al. 2017) -----------------
// The instantiations are the compressed ones with QBITS = SA_QBITS: 32-bit codes on the compressed tiling, one ChaCha20
// block (16 words) per thread, coordinate segment and peer pair.  algo/secagg.py is the numpy oracle; the payloads and the
// FedAvg model equal it bit for bit.
constexpr int SA_QBITS = 32;
static_assert(Q_SEG == 16, "one ChaCha20 block masks one thread's segment");

// ChaCha20 block function (RFC 8439 §2.3) with key `key`, block counter `ctr` and nonce (n0, n1, 0), added to (SIGN = 1)
// or subtracted from (SIGN = -1) acc, mod 2^32
#define SA_QR(a, b, c, d)                                                    \
  a += b; d ^= a; d = __funnelshift_l(d, d, 16);                             \
  c += d; b ^= c; b = __funnelshift_l(b, b, 12);                             \
  a += b; d ^= a; d = __funnelshift_l(d, d, 8);                              \
  c += d; b ^= c; b = __funnelshift_l(b, b, 7);
__device__ __forceinline__ void sa_chacha_acc(const uint32_t (&key)[8], uint32_t ctr, uint32_t n0, uint32_t n1, bool add,
                                              uint32_t (&acc)[Q_SEG]) {
  uint32_t x0 = 0x61707865u, x1 = 0x3320646eu, x2 = 0x79622d32u, x3 = 0x6b206574u;
  uint32_t x4 = key[0], x5 = key[1], x6 = key[2], x7 = key[3], x8 = key[4], x9 = key[5], x10 = key[6], x11 = key[7];
  uint32_t x12 = ctr, x13 = n0, x14 = n1, x15 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    SA_QR(x0, x4, x8, x12) SA_QR(x1, x5, x9, x13) SA_QR(x2, x6, x10, x14) SA_QR(x3, x7, x11, x15)
    SA_QR(x0, x5, x10, x15) SA_QR(x1, x6, x11, x12) SA_QR(x2, x7, x8, x13) SA_QR(x3, x4, x9, x14)
  }
  const uint32_t w[Q_SEG] = {x0 + 0x61707865u, x1 + 0x3320646eu, x2 + 0x79622d32u, x3 + 0x6b206574u,
                             x4 + key[0], x5 + key[1], x6 + key[2], x7 + key[3], x8 + key[4], x9 + key[5], x10 + key[6],
                             x11 + key[7], x12 + ctr, x13 + n0, x14 + n1, x15};
#pragma unroll
  for (int i = 0; i < Q_SEG; ++i) acc[i] = add ? acc[i] + w[i] : acc[i] - w[i];
}
#undef SA_QR

// row of pair (i, j), i < j, in the key table: pairs in lexicographic order
__device__ __forceinline__ int sa_pair_row(int i, int j, int K) { return i * (2 * K - i - 1) / 2 + (j - i - 1); }

// Phase 0 of a SecAgg round: encode and mask the local replicas' updates on this CTA's tiles of every slice, and count
// this thread's clipped and non-finite coordinates.  The key table is read with uniform loads (every thread of the CTA
// reads the same 32 bytes).
__device__ __forceinline__ void sa_encode(const CommArgs& a, int nslices, uint32_t& clipped, uint32_t& nonfinite) {
  const float R = a.sa_clip;
  const float scale = __int_as_float((127 + a.sa_frac_bits) << 23);            // 2^f, exact
  const long long t = *a.q_t;
  const uint32_t n0 = uint32_t(t), n1 = uint32_t(uint64_t(t) >> 32);
  for (int s = 0; s < nslices; ++s) {
    const QSlice sl = q_slice(a, s);
    for (int tb = sl.lo + blockIdx.x * Q_TILE; tb < sl.hi; tb += gridDim.x * Q_TILE) {
      const int c0 = tb + Q_SEG * threadIdx.x;
      if (c0 >= sl.hi) continue;
      float zv[Q_SEG];
#pragma unroll
      for (int q = 0; q < Q_SEG / 4; ++q) q_unf4(zv, q, q_ld4(a.z, c0 + 4 * q, a.n));
      for (int j = 0; j < a.n_local; ++j) {
        const int k = a.q_worker[j];
        uint32_t acc[Q_SEG];
#pragma unroll
        for (int q = 0; q < Q_SEG / 4; ++q) {
          const float4 xv = q_ld4(a.xl[j], c0 + 4 * q, a.n);       // coordinates >= n: u = 0, code 0
          const float u4[4] = {__fsub_rn(xv.x, zv[4 * q]), __fsub_rn(xv.y, zv[4 * q + 1]), __fsub_rn(xv.z, zv[4 * q + 2]),
                               __fsub_rn(xv.w, zv[4 * q + 3])};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float u = u4[i];
            int code = 0;
            if (!isfinite(u)) {
              ++nonfinite;
            } else {
              clipped += fabsf(u) > R ? 1u : 0u;
              code = __float2int_rn(__fmul_rn(fminf(fmaxf(u, -R), R), scale));
            }
            acc[4 * q + i] = uint32_t(code);
          }
        }
        const uint32_t ctr = uint32_t(c0 / Q_SEG);
        for (int p = 0; p < a.K; ++p) {                            // uniform across the CTA
          if (p == k) continue;
          const uint4* kp = reinterpret_cast<const uint4*>(a.sa_keys + 8 * sa_pair_row(min(k, p), max(k, p), a.K));
          const uint4 ka = __ldg(kp), kb = __ldg(kp + 1);
          const uint32_t key[8] = {ka.x, ka.y, ka.z, ka.w, kb.x, kb.y, kb.z, kb.w};
          sa_chacha_acc(key, ctr, n0, n1, p > k, acc);
        }
        uint4* dst = reinterpret_cast<uint4*>(a.q_codes[k] + 4 * size_t(c0));   // one 64-byte segment per thread
#pragma unroll
        for (int q = 0; q < Q_SEG / 4; ++q) dst[q] = make_uint4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
      }
    }
  }
}

// pass 1 of a SecAgg round at this thread's Q_SEG coordinates c0..: S = sum_k y_k mod 2^32 read as int32 (= sum_k q_k),
// and acc = float(S) 2^-f, correctly rounded
__device__ __forceinline__ void sa_gather(const CommArgs& a, int c0, float (&acc)[Q_SEG]) {
  uint32_t s[Q_SEG];
#pragma unroll
  for (int i = 0; i < Q_SEG; ++i) s[i] = 0u;
#pragma unroll 2
  for (int k = 0; k < a.K; ++k) {
    const unsigned char* src = a.q_codes[k] + 4 * size_t(c0);
#pragma unroll
    for (int q = 0; q < Q_SEG / 4; ++q) {                          // four 16-byte loads per peer
      const uint4 v = ld_sys_u32x4(src + 16 * q);
      s[4 * q] += v.x; s[4 * q + 1] += v.y; s[4 * q + 2] += v.z; s[4 * q + 3] += v.w;
    }
  }
  const float inv = __int_as_float((127 - a.sa_frac_bits) << 23);             // 2^-f, exact
#pragma unroll
  for (int i = 0; i < Q_SEG; ++i) acc[i] = __fmul_rn(__int2float_rn(int(s[i])), inv);
}

// the sum over a CTA of a per-thread count, valid in thread 0 (integers: the order does not matter)
__device__ __forceinline__ uint32_t block_add_u32(uint32_t v, uint32_t* sm) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t r = 0u;
  if (threadIdx.x < 32) r = __reduce_add_sync(0xffffffffu, threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0u);
  __syncthreads();
  return r;
}

// sum over the K workers, in worker order, of their dequantized codes q_k s_k at this thread's Q_SEG coordinates c0..
template <int QBITS>
__device__ __forceinline__ void q_gather(const CommArgs& a, int c0, float (&acc)[Q_SEG]) {
#pragma unroll
  for (int i = 0; i < Q_SEG; ++i) acc[i] = 0.f;
#pragma unroll 4
  for (int k = 0; k < a.K; ++k) {
    const float sc = ld_sys_f32(a.q_scales[k] + c0 / Q_GROUP);
    uint32_t wd[QBITS * Q_SEG / 32];
    if constexpr (QBITS == 8) {                    // 16 bytes per peer and load
      const uint4 v = ld_sys_u32x4(a.q_codes[k] + c0);
      wd[0] = v.x; wd[1] = v.y; wd[2] = v.z; wd[3] = v.w;
    } else {                                       // 8 bytes
      const uint2 v = ld_sys_u32x2(a.q_codes[k] + c0 / 2);
      wd[0] = v.x; wd[1] = v.y;
    }
#pragma unroll
    for (int i = 0; i < Q_SEG; ++i) {
      const int q = int(wd[i * QBITS / 32] << (32 - QBITS - (i * QBITS) % 32)) >> (32 - QBITS);   // sign-extended code
      acc[i] = __fadd_rn(acc[i], __fmul_rn(float(q), sc));
    }
  }
}

// ---- top-k sparsified updates: the K workers' sparse payloads (TopKLayout) of one tile, summed in shared memory -------
__device__ __forceinline__ uint32_t ld_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_sys_u16(const uint16_t* p) {
  unsigned short v;
  asm volatile("ld.relaxed.sys.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return v;
}
// acc = sum over the K workers, in worker order, of their sparse updates s_k at this thread's Q_SEG coordinates of the
// tile starting at tb.  Run by the whole CTA (barriers inside): the entries of tile tb / Q_TILE of worker k are
// scatter-added into a shared-memory accumulator, one worker after the other; a worker's indices are distinct, so no two
// threads add to one coordinate at once.  Adding 0 is exact and the accumulator never holds -0, so skipping the
// unselected coordinates gives the dense sum in worker order bit for bit.
__device__ __forceinline__ void topk_gather(const CommArgs& a, int tb, float (&acc)[Q_SEG]) {
  __shared__ __align__(16) float s_acc[Q_TILE];
  const TopKLayout L = topk_layout(a.n, a.topk_k);
  const int t = tb / Q_TILE;
  float4* s4 = reinterpret_cast<float4*>(s_acc) + threadIdx.x * (Q_SEG / 4);
#pragma unroll
  for (int q = 0; q < Q_SEG / 4; ++q) s4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  for (int k = 0; k < a.K; ++k) {
    const uint32_t* p = reinterpret_cast<const uint32_t*>(a.q_codes[k]);
    const uint32_t o0 = ld_sys_u32(p + t), o1 = min(ld_sys_u32(p + t + 1), uint32_t(a.topk_k));
    const float* val = reinterpret_cast<const float*>(p + L.val);
    const uint16_t* idx = reinterpret_cast<const uint16_t*>(p + L.idx);
    for (uint32_t e = o0 + threadIdx.x; e < o1; e += blockDim.x) {
      const uint32_t i = ld_sys_u16(idx + e) & (Q_TILE - 1);
      s_acc[i] = __fadd_rn(s_acc[i], ld_sys_f32(val + e));
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < Q_SEG / 4; ++q) q_unf4(acc, q, s4[q]);
  __syncthreads();                                 // the next tile clears s_acc
}

// Server optimizer step from the pseudo-gradient d itself (compressed rounds: d is the dequantized mean update, not
// formed as (z + d) - z).  FedAvgM: z + lr m, which is z + d when beta = 0 and lr = 1.
__device__ __forceinline__ float fedopt_step_d(const CommArgs& a, float z, float d, float& m, float& v) {
  if (a.opt == FEDOPT_AVGM) {
    m = fmaf(a.beta1, m, d);
    return fmaf(a.lr, m, z);
  }
  m = fmaf(a.beta1, m, (1.f - a.beta1) * d);
  const float d2 = d * d;
  if (a.opt == FEDOPT_ADAGRAD) {
    v += d2;
  } else if (a.opt == FEDOPT_ADAM) {
    v = fmaf(a.beta2, v, (1.f - a.beta2) * d2);
  } else {
    const float s = v > d2 ? 1.f : (v < d2 ? -1.f : 0.f);
    v = fmaf(-(1.f - a.beta2) * d2, s, v);
  }
  return fmaf(a.lr, m / (sqrtf(v) + a.tau), z);
}

// Pass 1 of a compressed round on this CTA's tiles of slice my_slice: z' = z + (1/K) sum_k q_k s_k (or the server step
// along that d); one-shot stores z' (and m, v) locally, two-shot broadcasts them into every rank.
// TOPK: the top-k rounds' sum of sparse payloads on whole-tile slices.
template <bool FEDOPT, int QBITS, bool TOPK = false>
__device__ __forceinline__ void q_reduce(const CommArgs& a, int my_slice, float inv_k, float& dual, float& bad) {
  const QSlice sl = q_slice(a, my_slice, TOPK ? Q_TILE : Q_GROUP);
  const bool adaptive = FEDOPT && a.opt != FEDOPT_AVGM;
  for (int tb = sl.lo + blockIdx.x * Q_TILE; tb < sl.hi; tb += gridDim.x * Q_TILE) {
    const int c0 = tb + Q_SEG * threadIdx.x;
    float acc[Q_SEG];
    if constexpr (TOPK) topk_gather(a, tb, acc);   // the whole CTA, before the partial tile's idle threads leave
    if (c0 >= sl.hi) continue;
    if constexpr (QBITS == SA_QBITS) sa_gather(a, c0, acc);
    else if constexpr (!TOPK) q_gather<QBITS>(a, c0, acc);
#pragma unroll
    for (int q = 0; q < Q_SEG / 4; ++q) {
      const int c = c0 + 4 * q;
      if (c >= a.n) break;
      const float4 zo = q_ld4(a.z, c, a.n);
      float4 d = q_f4(acc, q);
      d = make_float4(__fmul_rn(d.x, inv_k), __fmul_rn(d.y, inv_k), __fmul_rn(d.z, inv_k), __fmul_rn(d.w, inv_k));
      float4 zs, mv, vv;
      if constexpr (FEDOPT) {
        mv = q_ld4(a.m, c, a.n);
        vv = adaptive ? q_ld4(a.v, c, a.n) : make_float4(0.f, 0.f, 0.f, 0.f);
        zs = make_float4(fedopt_step_d(a, zo.x, d.x, mv.x, vv.x), fedopt_step_d(a, zo.y, d.y, mv.y, vv.y),
                         fedopt_step_d(a, zo.z, d.z, mv.z, vv.z), fedopt_step_d(a, zo.w, d.w, mv.w, vv.w));
      } else {
        zs = make_float4(__fadd_rn(zo.x, d.x), __fadd_rn(zo.y, d.y), __fadd_rn(zo.z, d.z), __fadd_rn(zo.w, d.w));
      }
      if (!a.two_shot) {
        dual_nan_v4(zo, zs, dual, bad);
        q_st4(a.z, c, a.n, zs);
        if constexpr (FEDOPT) {
          q_st4(a.m, c, a.n, mv);
          if (adaptive) q_st4(a.v, c, a.n, vv);
        }
      } else {                                     // dual + NaN check from the landed weights in pass 2
        q_bcast4(a.mc_x, a.xw, a.world, c, a.n, zs);
        if constexpr (FEDOPT) {
          q_bcast4(a.mc_m, a.mw, a.world, c, a.n, mv);
          if (adaptive) q_bcast4(a.mc_v, a.vw, a.world, c, a.n, vv);
        }
      }
    }
  }
}

// Pass 2 of a compressed round (FedAvg's, on the compressed tiling): one-shot writes z into every local replica,
// two-shot copies the broadcast weights of every slice into z and takes the dual residual and NaN count from them.
__device__ __forceinline__ void q_write_back(const CommArgs& a, int nslices, float& dual, float& bad, int unit) {
  for (int s = 0; s < nslices; ++s) {
    const QSlice sl = q_slice(a, s, unit);
    for (int tb = sl.lo + blockIdx.x * Q_TILE; tb < sl.hi; tb += gridDim.x * Q_TILE) {
      const int c0 = tb + Q_SEG * threadIdx.x;
      if (c0 >= sl.hi) continue;
#pragma unroll
      for (int q = 0; q < Q_SEG / 4; ++q) {
        const int c = c0 + 4 * q;
        if (c >= a.n) break;
        if (a.two_shot) {
          const float4 zn = q_ld4_sys(a.xl[0], c, a.n);
          dual_nan_v4(q_ld4(a.z, c, a.n), zn, dual, bad);
          q_st4(a.z, c, a.n, zn);
        } else {
          const float4 zv = q_ld4(a.z, c, a.n);
          for (int j = 0; j < a.n_local; ++j) q_st4(a.xl[j], c, a.n, zv);
        }
      }
    }
  }
}

// ---- client sampling: the participant set of round t and its sample-count weights --------------------------------------
// Worker k draws h_k = F(F(key + (t + 1) G) + (k + 1) G) (F, G as for the DP noise); the round takes the samp_S workers
// with the smallest (h_k, k), by integer ranks.  w_k = n_k / sum_{j in P} n_j, the integer sum rounded once to float and
// the quotient correctly rounded (__fdiv_rn: the extension is built with --use_fast_math), so the set and the weights equal
// algo/sampling.py (participants, weights) exactly.  Every CTA computes them for itself, in shared memory.
struct SampSet {
  const float* const* x;             // [np] the participants' slices, in worker order
  const float* w;                    // [np] their weights
  int np;
};
__device__ __forceinline__ SampSet samp_select(const CommArgs& a) {
  __shared__ unsigned long long s_h[COMM_MAX_K];
  __shared__ int s_in[COMM_MAX_K];
  __shared__ const float* s_x[COMM_MAX_K];
  __shared__ float s_w[COMM_MAX_K];
  __shared__ int s_np;
  const int k = threadIdx.x;
  if (k < a.K) {
    const uint64_t rk = dp_mix(a.samp_key + uint64_t(*a.samp_t + 1) * DP_GAMMA);
    s_h[k] = dp_mix(rk + uint64_t(k + 1) * DP_GAMMA);
  }
  __syncthreads();
  if (k < a.K) {
    const unsigned long long h = s_h[k];
    int rank = 0;
    for (int j = 0; j < a.K; ++j) rank += (s_h[j] < h || (s_h[j] == h && j < k)) ? 1 : 0;
    s_in[k] = rank < a.samp_S ? 1 : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long total = 0;
    int np = 0;
    for (int j = 0; j < a.K; ++j) {
      if (!s_in[j]) continue;
      total += a.client_n[j];
      s_x[np++] = a.x[j];
    }
    const float ft = float(total);
    for (int j = 0, i = 0; j < a.K; ++j)
      if (s_in[j]) s_w[i++] = __fdiv_rn(float(a.client_n[j]), ft);
    s_np = np;
  }
  __syncthreads();
  return {s_x, s_w, s_np};
}
// sum_{k in P} w_k x_k at float4 index `off` / coordinate i, in worker order; each term rounded, then added (no fma), as
// the ATen oracle forms it.  Non-participants are not read.
__device__ __forceinline__ float4 samp_gather_v4(const SampSet& ss, size_t off) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int i = 0; i < ss.np; ++i) {
    const float w = ss.w[i];
    const float4 xv = ld_sys_v4(ss.x[i] + off);
    acc.x = __fadd_rn(acc.x, __fmul_rn(w, xv.x)); acc.y = __fadd_rn(acc.y, __fmul_rn(w, xv.y));
    acc.z = __fadd_rn(acc.z, __fmul_rn(w, xv.z)); acc.w = __fadd_rn(acc.w, __fmul_rn(w, xv.w));
  }
  return acc;
}
__device__ __forceinline__ float samp_gather_f32(const SampSet& ss, int i) {
  float acc = 0.f;
  for (int p = 0; p < ss.np; ++p) acc = __fadd_rn(acc, __fmul_rn(ss.w[p], ld_sys_f32(ss.x[p] + i)));
  return acc;
}
// pass 1's aggregate at float4 index `off`: the weighted sum of the participants (SAMP) or reduce_v4's
template <int AGG_PAD, bool SAMP>
__device__ __forceinline__ float4 pass1_v4(const CommArgs& a, size_t off, float rho, bool use_mc, const SampSet& ss) {
  if constexpr (SAMP) return samp_gather_v4(ss, off);
  else return reduce_v4<AGG_PAD>(a, off, rho, use_mc);
}

// Phase C (the last CTA, world > 1): every rank posts the NW words w[] of its round statistics into row PAD_PAYLOAD of
// every peer; thread 0 then replaces w[] by their sums over the ranks in rank order, as T (float, or uint32_t for counts
// passed as bit patterns), so every rank reports the same values.  w is shared memory, written by thread 0 before the call.
template <typename T, int NW>
__device__ __forceinline__ void exchange_sum(const CommArgs& a, uint32_t epoch, float* w, int* s_abort) {
  __syncthreads();
  if (threadIdx.x < a.world) {
    float* pay = reinterpret_cast<float*>(a.ctrl[threadIdx.x] + PAD_PAYLOAD) + 4 * a.rank;
    for (int i = 0; i < NW; ++i) st_sys_f32(pay + i, w[i]);
    peer_post_wait(a.ctrl, a.rank, PAD_FLAG_C, epoch, a.timeout_cycles, a.out + OUT_STATUS, s_abort);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float* pay = reinterpret_cast<const float*>(a.ctrl[a.rank] + PAD_PAYLOAD);
    T s[NW] = {};
    for (int r = 0; r < a.world; ++r) {
#pragma unroll
      for (int i = 0; i < NW; ++i) {
        const float v = ld_sys_f32(pay + 4 * r + i);
        if constexpr (std::is_same<T, float>::value) s[i] += v;
        else s[i] += __float_as_uint(v);
      }
    }
#pragma unroll
    for (int i = 0; i < NW; ++i) {
      if constexpr (std::is_same<T, float>::value) w[i] = s[i];
      else w[i] = __uint_as_float(s[i]);
    }
  }
}

// FEDOPT = false: FedAvg / FedProx / ADMM (a.mode).  FEDOPT = true: FedAvg (mode 0) whose new model is a server optimizer
// step from z instead of the plain mean.  Pass 1 forms the step from the reduced mean, z and the state m (and v): one-shot
// stores z, m, v locally; two-shot rank r broadcasts slice r of the new weights, of m and of v into every rank, so every rank
// ends the round with the same z, m and v.  Pass 2 is FedAvg's.
// AGG_PAD > 0: the robust instantiations (modes 0 / 1): pass 1 takes the median / trimmed mean of the K workers instead of
// their mean (with FEDOPT, as the server optimizer's aggregate); everything else is shared with the mean.
// DP: the DP-FedAvg instantiations (mode 0, the mean, AGG_PAD = 0): pass 1 adds dp_std * xi to the mean before the optional
// server step (one-shot, two-shot and the scalar tail alike); phase C exchanges the clip statistics of dp_clip_kernel
// across ranks, and the last CTA advances the round counter dp_t.
// QBITS = 8 / 4: the compressed instantiations (mode 0, the mean): phase 0, before barrier A, encodes the local replicas'
// updates into the payload arenas; pass 1 reduces the K workers' payloads instead of their floats, and both passes walk the
// compressed tiling (no separate scalar tail); phase C exchanges the quantization statistics and advances q_t.
// QBITS = SA_QBITS: the secure-aggregation instantiations (mode 0, the mean), on the compressed skeleton: phase 0 encodes
// and masks the local replicas' updates into 32-bit payloads; pass 1 sums the K payloads as integers mod 2^32 and decodes;
// phase C exchanges the integer clipped / non-finite counts, adds the latter to the non-finite count and advances q_t.
// SAMP: the client-sampling instantiations (mode 0, the mean, AGG_PAD = 0): every CTA selects round *samp_t's participants
// and their weights first; pass 1 (one-shot, two-shot and the scalar tail) forms the weighted sum of the participants out of
// peer memory with P2P loads only (multimem.ld_reduce would add every bound device with weight 1; the two-shot broadcast
// may still use multimem.st); pass 2 is FedAvg's, so every replica, participant or not, receives z; the last CTA advances
// samp_t.
// TOPK: the top-k instantiations (mode 0, the mean), on the compressed skeleton with whole-tile slices: topk_select_kernel
// has written the payloads before this launch; pass 1 scatter-adds the K workers' entries of each tile into shared memory
// in worker order (P2P loads only) and applies the compressed rounds' epilogue; phase C exchanges the selection statistics.
template <bool FEDOPT, int AGG_PAD, bool DP = false, int QBITS = 0, bool SAMP = false, bool TOPK = false>
__global__ void __launch_bounds__(COMM_THREADS, 1) block_reduce_kernel(const CommArgs a) {
  constexpr bool TILED = QBITS != 0 || TOPK;     // both passes walk the compressed tiling
  __shared__ float sm[32];
  __shared__ int s_abort;
  __shared__ int s_last;
  if (threadIdx.x == 0) { s_abort = 0; s_last = 0; }
  __syncthreads();
  SampSet ss{};
  if constexpr (SAMP) ss = samp_select(a);
  const uint32_t epoch = a.sync[0] + 1;
  const float rho = a.rho_dev != nullptr ? __ldg(a.rho_dev) : a.rho;
  const float inv_scale = (AGG_PAD > 0 || SAMP) ? 1.f : a.mode == 2 ? 1.f / (float(a.K) * rho) : 1.f / float(a.K);
  const int n4 = a.n >> 2;
  const int nslices = a.two_shot ? a.world : 1;
  const int chunk4 = a.two_shot ? (n4 + a.world - 1) / a.world : n4;
  const int my_slice = a.two_shot ? a.rank : 0;
  const int stride = gridDim.x * blockDim.x;
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const bool use_mc = !SAMP && a.mc_x != nullptr && (a.mode != 2 || a.mc_y != nullptr);

  // ---- 0 (compressed rounds): encode the local replicas' updates; per-CTA partial statistics in CTA order ------
  if constexpr (QBITS == SA_QBITS) {             // SecAgg: integer counts of clipped and non-finite coordinates
    uint32_t clipped = 0u, nonfinite = 0u;
    sa_encode(a, nslices, clipped, nonfinite);
    clipped = block_add_u32(clipped, reinterpret_cast<uint32_t*>(sm));      // (its barriers also publish the payload)
    nonfinite = block_add_u32(nonfinite, reinterpret_cast<uint32_t*>(sm));
    if (threadIdx.x == 0) {
      reinterpret_cast<uint32_t*>(a.q_part)[2 * blockIdx.x + 0] = clipped;
      reinterpret_cast<uint32_t*>(a.q_part)[2 * blockIdx.x + 1] = nonfinite;
    }
    if (a.world > 1) __threadfence_system();
  } else if constexpr (QBITS != 0) {
    float err = 0.f, nrm = 0.f;
    q_encode<QBITS>(a, nslices, err, nrm);
    err = block_add(err, sm);                      // (its barriers also make the CTA's payload visible to all its threads)
    nrm = block_add(nrm, sm);
    if (threadIdx.x == 0) {
      a.q_part[2 * blockIdx.x + 0] = err;
      a.q_part[2 * blockIdx.x + 1] = nrm;
    }
    if (a.world > 1) __threadfence_system();
  }

  // ---- A: inputs of every rank are final (their producers precede this kernel in stream order) ----------------
  cta_peer_barrier(a.ctrl, a.world, a.rank, PAD_FLAG_A, epoch, a.timeout_cycles, a.out + OUT_STATUS, &s_abort);

  // ---- 1: reduce, scale, new z, dual residual ---------------------------------------------------------------------
  float dual = 0.f, bad = 0.f;
  if constexpr (TILED) {
    // SecAgg, top-k: 1/K correctly rounded (the extension is built with --use_fast_math), as the oracle's float32(1) / K
    q_reduce<FEDOPT, QBITS, TOPK>(a, my_slice, (QBITS == SA_QBITS || TOPK) ? __frcp_rn(float(a.K)) : inv_scale, dual, bad);
  } else {
    const int lo = my_slice * chunk4;
    const int hi = min(n4, lo + chunk4);
    const bool adaptive = FEDOPT && a.opt != FEDOPT_AVGM;
    const bool dual_here = !(a.two_shot && a.mode == 0);   // two-shot FedAvg takes the dual residual and NaN count from
                                                            // the finished weights in pass 2
    // two elements per thread and iteration: their (remote) loads are issued back to back, so twice as many bytes are in
    // flight per thread — the pass is bound by NVLink round trips, not by issue slots
    for (int i = lo + t0; i < hi; i += 2 * stride) {
      const int i1 = i + stride;
      const bool has1 = i1 < hi;
      const size_t off0 = 4 * size_t(i), off1 = 4 * size_t(has1 ? i1 : i);
      float4 accs[2];
      accs[0] = pass1_v4<AGG_PAD, SAMP>(a, off0, rho, use_mc, ss);
      accs[1] = has1 ? pass1_v4<AGG_PAD, SAMP>(a, off1, rho, use_mc, ss) : accs[0];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (u == 1 && !has1) break;
        const size_t off = u == 0 ? off0 : off1;
        const float4 acc = accs[u];
        const float4 zn = DP ? dp_noised_v4<DP>(a, off, make_float4(acc.x * inv_scale, acc.y * inv_scale, acc.z * inv_scale,
                                                                     acc.w * inv_scale))
                             : make_float4(acc.x * inv_scale, acc.y * inv_scale, acc.z * inv_scale, acc.w * inv_scale);
        // the new value zs: the aggregate itself, or the server step from z along it (which also updates m and v)
        const float4 zo = (FEDOPT || dual_here) ? *reinterpret_cast<const float4*>(a.z + off) : zn;
        float4 zs = zn, mv, vv;
        if constexpr (FEDOPT) {
          mv = *reinterpret_cast<const float4*>(a.m + off);
          vv = adaptive ? *reinterpret_cast<const float4*>(a.v + off) : make_float4(0.f, 0.f, 0.f, 0.f);
          zs = fedopt_step_v4(a, zo, zn, mv, vv);
        }
        if (dual_here) dual_nan_v4(zo, zs, dual, bad);
        if (!a.two_shot) {
          *reinterpret_cast<float4*>(a.z + off) = zs;
          if constexpr (FEDOPT) {
            *reinterpret_cast<float4*>(a.m + off) = mv;
            if (adaptive) *reinterpret_cast<float4*>(a.v + off) = vv;
          }
        } else {                                   // slice r into every rank: FedAvg's weights, else the consensus vector
          if (a.mode == 0) bcast_v4(a.mc_x, a.xw, a.world, off, zs);
          else bcast_v4(a.mc_z, a.zw, a.world, off, zs);
          if constexpr (FEDOPT) {
            bcast_v4(a.mc_m, a.mw, a.world, off, mv);
            if (adaptive) bcast_v4(a.mc_v, a.vw, a.world, off, vv);
          }
        }
      }
    }
  }
  // scalar tail (n % 4 elements): every rank reduces it for itself, one-shot style
  const int tail0 = n4 << 2;
  if (!TILED && blockIdx.x == 0 && tail0 + int(threadIdx.x) < a.n) {
    const int i = tail0 + threadIdx.x;
    float acc = 0.f;
    if constexpr (AGG_PAD > 0) {
      acc = robust_gather_f32<AGG_PAD>(a, i);
    } else if constexpr (SAMP) {
      acc = samp_gather_f32(ss, i);
    } else if (use_mc) {
      acc = multimem_ld_reduce_f32(a.mc_x + i);
      if (a.mode == 2) acc = fmaf(rho, acc, multimem_ld_reduce_f32(a.mc_y + i));
    } else {
      for (int k = 0; k < a.K; ++k) {
        const float xv = ld_sys_f32(a.x[k] + i);
        acc += a.mode == 2 ? fmaf(rho, xv, ld_sys_f32(a.y[k] + i)) : xv;
      }
    }
    float zn = DP ? dp_noised_f32<DP>(a, i, acc * inv_scale) : acc * inv_scale;
    if constexpr (FEDOPT) {                        // every rank steps its own copy of the tail
      float mv = a.m[i], vv = a.opt != FEDOPT_AVGM ? a.v[i] : 0.f;
      zn = fedopt_step(a, a.z[i], zn, mv, vv);
      a.m[i] = mv;
      if (a.opt != FEDOPT_AVGM) a.v[i] = vv;
    }
    const float d = a.z[i] - zn;
    if (!a.two_shot || a.mode == 0 || a.rank == 0) dual = fmaf(d, d, dual);     // two-shot FedProx/ADMM: the dual parts are summed over ranks
    if (!isfinite(zn)) bad += 1.f;
    a.z[i] = zn;
  }
  if (a.world > 1) __threadfence_system();

  // ---- B: every peer has finished reading my x / y, and its broadcast has landed here ------------------------
  cta_peer_barrier(a.ctrl, a.world, a.rank, PAD_FLAG_B, epoch, a.timeout_cycles, a.out + OUT_STATUS, &s_abort);

  // ---- 2: local epilogue in place -------------------------------------------------------------------------------
  float pr[COMM_MAX_LOCAL];
#pragma unroll
  for (int j = 0; j < COMM_MAX_LOCAL; ++j) pr[j] = 0.f;
  if constexpr (TILED) q_write_back(a, nslices, dual, bad, TOPK ? Q_TILE : Q_GROUP);
  for (int s = 0; s < (TILED ? 0 : nslices); ++s) {
    const int lo = s * chunk4;
    const int hi = min(n4, lo + chunk4);
    for (int i = lo + t0; i < hi; i += stride) {
      const size_t off = 4 * size_t(i);
      if (a.mode == 0) {
        if (a.two_shot) {                        // weights already hold the average: keep a copy as next round's z_old,
          const float4 zn = ld_sys_v4(a.xl[0] + off);          // and take the dual residual + NaN check from it (the full vector
          dual_nan_v4(*reinterpret_cast<const float4*>(a.z + off), zn, dual, bad);   // is local now: no cross-rank sum needed)
          *reinterpret_cast<float4*>(a.z + off) = zn;
        } else {
          const float4 zv = *reinterpret_cast<const float4*>(a.z + off);
          for (int j = 0; j < a.n_local; ++j) *reinterpret_cast<float4*>(a.xl[j] + off) = zv;
        }
      } else {
        const float4 zv = a.two_shot ? ld_sys_v4(a.z + off) : *reinterpret_cast<const float4*>(a.z + off);
#pragma unroll
        for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
          if (j < a.n_local) {
            const float4 xv = *reinterpret_cast<const float4*>(a.xl[j] + off);
            const float4 yd = make_float4(rho * (xv.x - zv.x), rho * (xv.y - zv.y), rho * (xv.z - zv.z), rho * (xv.w - zv.w));
            pr[j] = fmaf(yd.x, yd.x, fmaf(yd.y, yd.y, fmaf(yd.z, yd.z, fmaf(yd.w, yd.w, pr[j]))));
            if (a.mode == 2) {
              float4 yv = *reinterpret_cast<float4*>(a.yl[j] + off);
              yv.x += yd.x; yv.y += yd.y; yv.z += yd.z; yv.w += yd.w;
              *reinterpret_cast<float4*>(a.yl[j] + off) = yv;
            }
          }
        }
      }
    }
  }
  if (!TILED && blockIdx.x == 0 && tail0 + int(threadIdx.x) < a.n) {
    const int i = tail0 + threadIdx.x;
    const float zv = a.z[i];
#pragma unroll
    for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
      if (j < a.n_local) {
        if (a.mode == 0) {
          a.xl[j][i] = zv;
        } else {
          const float yd = rho * (a.xl[j][i] - zv);
          pr[j] = fmaf(yd, yd, pr[j]);
          if (a.mode == 2) a.yl[j][i] += yd;
        }
      }
    }
  }

  // ---- block partials -> device accumulators; the last CTA finishes the scalars ---------------------------------
  dual = block_add(dual, sm);
  bad = block_add(bad, sm);
  if (threadIdx.x == 0) {
    if (dual != 0.f) atomicAdd(a.scratch + 0, dual);
    if (bad != 0.f) atomicAdd(a.scratch + 1, bad);
  }
  if (a.mode != 0) {
#pragma unroll
    for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
      if (j < a.n_local) {                      // uniform across the CTA: the barriers inside block_add are safe
        const float v = block_add(pr[j], sm);
        if (threadIdx.x == 0 && v != 0.f) atomicAdd(a.scratch + 4 + j, v);
      }
    }
  }
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicAdd(reinterpret_cast<unsigned*>(a.scratch + 2), 1u);
    s_last = (t == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;

  // ---- C: exchange the round's statistics over the ranks and write the record (one CTA) ---------------------------
  // A round exchanges one set of words at most: FedProx / ADMM their dual and primal parts and non-finite counts (FedAvg's
  // are complete on every rank already), DP rounds the clip statistics of the local replicas, compressed rounds the
  // quantization statistics and SecAgg rounds the clipped / non-finite counts, both summed over the CTAs in CTA order.
  __shared__ float s_c[3];
  float dual_sq = 0.f, primal = 0.f, nonfinite = 0.f;   // thread 0
  if (threadIdx.x == 0) {
    __threadfence();
    for (int j = 0; j < a.n_local; ++j) primal += sqrtf(__ldcg(a.scratch + 4 + j));
    dual_sq = __ldcg(a.scratch + 0);
    nonfinite = __ldcg(a.scratch + 1);
    for (int j = 0; j < COMM_SCRATCH_FLOATS; ++j) a.scratch[j] = 0.f;      // self-cleaning: no memset per launch
    if constexpr (DP) {
      float clipped = 0.f, norms = 0.f;
      for (int j = 0; j < a.n_local; ++j) {
        norms += a.dp_stats[j];
        clipped += a.dp_stats[COMM_MAX_LOCAL + j];
      }
      s_c[0] = clipped;
      s_c[1] = norms;
    } else if constexpr (QBITS == SA_QBITS) {      // integers, as uint32 bit patterns
      uint32_t c = 0u, b = 0u;
      for (int i = 0; i < int(gridDim.x); ++i) {
        c += __ldcg(reinterpret_cast<const unsigned int*>(a.q_part) + 2 * i + 0);
        b += __ldcg(reinterpret_cast<const unsigned int*>(a.q_part) + 2 * i + 1);
      }
      s_c[0] = __uint_as_float(c);
      s_c[1] = __uint_as_float(b);
    } else if constexpr (TOPK) {                   // topk_select_kernel summed them over the CTAs in CTA order
      s_c[0] = __ldcg(a.q_part + 0);
      s_c[1] = __ldcg(a.q_part + 1);
    } else if constexpr (QBITS != 0) {
      float e = 0.f, u = 0.f;
      for (int b = 0; b < int(gridDim.x); ++b) {
        e += __ldcg(a.q_part + 2 * b + 0);
        u += __ldcg(a.q_part + 2 * b + 1);
      }
      s_c[0] = e;
      s_c[1] = u;
    } else {
      s_c[0] = dual_sq;
      s_c[1] = primal;
      s_c[2] = nonfinite;
    }
  }
  using Word = typename std::conditional<QBITS == SA_QBITS, uint32_t, float>::type;
  constexpr int NW = (DP || TILED) ? 2 : 3;
  if (a.world > 1 && (DP || TILED || a.mode != 0)) exchange_sum<Word, NW>(a, epoch, s_c, &s_abort);
  if (threadIdx.x == 0) {
    if constexpr (DP) {
      a.out[OUT_DP_CLIPPED] = s_c[0];
      a.out[OUT_DP_NORM_SUM] = s_c[1];
      *a.dp_t += 1;                                // every CTA has read t: the next round (or graph replay) draws t + 1
    } else if constexpr (QBITS == SA_QBITS) {
      a.out[OUT_SA_CLIPPED] = s_c[0];
      a.out[OUT_SA_NONFINITE] = s_c[1];
      nonfinite += float(__float_as_uint(s_c[1]));  // so the NaN guard fires although the non-finite updates' codes are 0
      *a.q_t += 1;                                 // every CTA has read t: the next round (or graph replay) masks with t + 1
    } else if constexpr (QBITS != 0) {
      a.out[OUT_Q_ERR_SQ] = s_c[0];
      a.out[OUT_Q_NORM_SQ] = s_c[1];
      *a.q_t += 1;                                 // every CTA has read t: the next round (or graph replay) draws t + 1
    } else if constexpr (TOPK) {
      a.out[OUT_Q_ERR_SQ] = s_c[0];
      a.out[OUT_Q_NORM_SQ] = s_c[1];
    } else if (a.world > 1 && a.mode != 0) {
      if (a.two_shot) {                            // one-shot: every rank already holds the full dual residual and NaN count
        dual_sq = s_c[0];
        nonfinite = s_c[2];
      }
      primal = s_c[1];
    }
    if constexpr (SAMP) *a.samp_t += 1;            // every CTA has selected: the next round (or graph replay) samples t + 1
    a.out[OUT_DUAL_SQ] = dual_sq;
    a.out[OUT_PRIMAL] = primal;
    a.out[OUT_NONFINITE] = nonfinite;
    a.out[OUT_RHO] = rho;                          // OUT_STATUS is sticky: only ever written on a timeout
    a.out[OUT_EPOCH] = float(epoch);
    a.out[OUT_TWO_SHOT] = float(a.two_shot);
    __threadfence();
    a.sync[0] = epoch;
  }
}

// one CTA per SM (132 on an H100 SXM) x 512 threads, at most COMM_MAX_BLOCKS; read once per process
static int comm_max_blocks() {
  static const int m = [] {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms < 1 ? 1 : (sms > COMM_MAX_BLOCKS ? COMM_MAX_BLOCKS : sms);
  }();
  return m;
}

// block_reduce_kernel's instantiation for a round, as an index into the launcher's table: the mean, the robust rules on
// <= 4, <= 8 and <= 16 workers, the DP mean, 8-bit codes, 4-bit codes, the sampled weighted mean, secure aggregation and
// top-k payloads, plus REDUCE_VARIANTS with a server optimizer
constexpr int REDUCE_VARIANTS = 10;
static int reduce_variant(const CommArgs& a) {
  int v;
  if (a.topk_k != 0) v = 9;
  else if (a.sa) v = 8;
  else if (a.samp_S != 0 || a.samp_t != nullptr) v = 7;
  else if (a.qbits != 0) v = a.qbits == 8 ? 5 : 6;
  else if (a.dp) v = 4;
  else if (a.agg == AGG_MEAN) v = 0;
  else v = a.K <= 4 ? 1 : a.K <= 8 ? 2 : 3;
  return (a.opt != FEDOPT_NONE ? REDUCE_VARIANTS : 0) + v;
}

void block_reduce_launch(const CommArgs& args_in, cudaStream_t s) {
  CommArgs args = args_in;
  if (args.K < 1 || args.K > COMM_MAX_K || args.n_local > COMM_MAX_LOCAL || args.world > COMM_MAX_WORLD)
    throw std::runtime_error("fedb200: block_reduce: too many contributions / replicas / ranks");
  if (args.two_shot && (args.world <= 1 || args.n_local != 1 || args.K != args.world))
    throw std::runtime_error("fedb200: two-shot aggregation needs one replica per rank");
  if (args.opt != FEDOPT_NONE &&
      (args.opt > FEDOPT_YOGI || args.mode != 0 || args.m == nullptr || (args.opt != FEDOPT_AVGM && args.v == nullptr)))
    throw std::runtime_error("fedb200: block_reduce: server optimizer needs mode 0 and its state vectors");
  if (args.agg != AGG_MEAN) {
    if (args.agg != AGG_MEDIAN && args.agg != AGG_TRIMMED)
      throw std::runtime_error("fedb200: block_reduce: unknown aggregation rule");
    if (args.K > COMM_MAX_K_ROBUST)
      throw std::runtime_error("fedb200: block_reduce: robust aggregation supports at most 16 workers");
    if (args.mode == 2) throw std::runtime_error("fedb200: block_reduce: robust aggregation needs mode 0 or 1");
    if (args.agg == AGG_TRIMMED && (args.trim_b < 0 || 2 * args.trim_b >= args.K))
      throw std::runtime_error("fedb200: block_reduce: trimmed mean needs 0 <= 2 trim_b < K");
  }
  if (args.dp && (args.agg != AGG_MEAN || args.mode != 0 || args.dp_t == nullptr || args.dp_stats == nullptr))
    throw std::runtime_error("fedb200: block_reduce: DP needs mode 0, the mean, a round counter and clip statistics");
  if (args.qbits != 0) {
    if (args.qbits != 8 && args.qbits != 4) throw std::runtime_error("fedb200: block_reduce: compressed rounds take 8 or 4 bits");
    if (args.agg != AGG_MEAN || args.mode != 0 || args.dp || args.q_t == nullptr || args.q_part == nullptr)
      throw std::runtime_error("fedb200: block_reduce: compression needs mode 0, the mean without DP, a round counter and "
                               "a statistics buffer");
    if (args.two_shot && (args.xw[args.world - 1] == nullptr || (args.opt != FEDOPT_NONE && args.mw[args.world - 1] == nullptr)))
      throw std::runtime_error("fedb200: block_reduce: two-shot compressed rounds need P2P broadcast targets");
  }
  const bool samp = args.samp_S != 0 || args.samp_t != nullptr;
  if (samp) {
    if (args.samp_S < 1 || args.samp_S > args.K)
      throw std::runtime_error("fedb200: block_reduce: client sampling needs 1 <= S <= K participants");
    if (args.samp_t == nullptr || args.client_n == nullptr)
      throw std::runtime_error("fedb200: block_reduce: client sampling needs a round counter and the sample counts");
    if (args.mode != 0 || args.agg != AGG_MEAN || args.dp || args.qbits != 0)
      throw std::runtime_error("fedb200: block_reduce: client sampling needs mode 0 and the mean, without DP or compression");
  }
  if (args.sa) {
    if (args.mode != 0 || args.agg != AGG_MEAN || args.dp || args.qbits != 0 || samp)
      throw std::runtime_error("fedb200: block_reduce: secure aggregation needs mode 0 and the mean, without DP, "
                               "compression or sampling");
    if (args.K < 2) throw std::runtime_error("fedb200: block_reduce: secure aggregation needs at least 2 workers");
    if (args.sa_keys == nullptr || args.q_t == nullptr || args.q_part == nullptr)
      throw std::runtime_error("fedb200: block_reduce: secure aggregation needs the pair keys, a round counter and a "
                               "statistics buffer");
    if (args.sa_frac_bits < 0 || args.sa_frac_bits > SA_MAX_FRAC_BITS || !(args.sa_clip > 0.f))
      throw std::runtime_error("fedb200: block_reduce: secure aggregation needs 0 <= f <= 126 and a clip > 0");
    for (int k = 0; k < args.K; ++k)
      if (args.q_codes[k] == nullptr) throw std::runtime_error("fedb200: block_reduce: secure aggregation needs K payloads");
    if (args.two_shot && (args.xw[args.world - 1] == nullptr || (args.opt != FEDOPT_NONE && args.mw[args.world - 1] == nullptr)))
      throw std::runtime_error("fedb200: block_reduce: two-shot secure aggregation needs P2P broadcast targets");
  }
  if (args.topk_k != 0) {
    if (args.mode != 0 || args.agg != AGG_MEAN || args.dp || args.qbits != 0 || samp || args.sa)
      throw std::runtime_error("fedb200: block_reduce: top-k rounds need mode 0 and the mean, without DP, compression, "
                               "sampling or secure aggregation");
    if (args.topk_k < 1 || args.topk_k > args.n || args.q_part == nullptr)
      throw std::runtime_error("fedb200: block_reduce: top-k rounds need 1 <= k <= n and the selection statistics");
    for (int k = 0; k < args.K; ++k)
      if (args.q_codes[k] == nullptr) throw std::runtime_error("fedb200: block_reduce: top-k rounds need K payloads");
    if (args.two_shot && (args.xw[args.world - 1] == nullptr || (args.opt != FEDOPT_NONE && args.mw[args.world - 1] == nullptr)))
      throw std::runtime_error("fedb200: block_reduce: two-shot top-k rounds need P2P broadcast targets");
  }
  static const void* const kernels[2 * REDUCE_VARIANTS] = {
      (const void*)block_reduce_kernel<false, 0>, (const void*)block_reduce_kernel<false, 4>,
      (const void*)block_reduce_kernel<false, 8>, (const void*)block_reduce_kernel<false, 16>,
      (const void*)block_reduce_kernel<false, 0, true>, (const void*)block_reduce_kernel<false, 0, false, 8>,
      (const void*)block_reduce_kernel<false, 0, false, 4>, (const void*)block_reduce_kernel<false, 0, false, 0, true>,
      (const void*)block_reduce_kernel<false, 0, false, SA_QBITS>,
      (const void*)block_reduce_kernel<false, 0, false, 0, false, true>,
      (const void*)block_reduce_kernel<true, 0>, (const void*)block_reduce_kernel<true, 4>,
      (const void*)block_reduce_kernel<true, 8>, (const void*)block_reduce_kernel<true, 16>,
      (const void*)block_reduce_kernel<true, 0, true>, (const void*)block_reduce_kernel<true, 0, false, 8>,
      (const void*)block_reduce_kernel<true, 0, false, 4>, (const void*)block_reduce_kernel<true, 0, false, 0, true>,
      (const void*)block_reduce_kernel<true, 0, false, SA_QBITS>,
      (const void*)block_reduce_kernel<true, 0, false, 0, false, true>};
  const void* kernel = kernels[reduce_variant(args)];
  int cap = comm_max_blocks();
  if (args.max_blocks > 0 && args.max_blocks < cap) cap = args.max_blocks;
  const int n4 = args.n >> 2;
  const int work4 = args.two_shot ? (n4 + args.world - 1) / args.world : n4;
  int want = (work4 + COMM_THREADS - 1) / COMM_THREADS;
  if (args.qbits != 0 || args.sa) {                    // one tile of COMM_THREADS * Q_SEG coordinates per CTA and step
    const int ng = (args.n + Q_GROUP - 1) / Q_GROUP;
    const int per = args.two_shot ? (ng + args.world - 1) / args.world : ng;
    want = (per * Q_GROUP + Q_TILE - 1) / Q_TILE;
  }
  if (args.topk_k != 0) {                              // whole tiles per slice
    const int nt = (args.n + Q_TILE - 1) / Q_TILE;
    want = args.two_shot ? (nt + args.world - 1) / args.world : nt;
  }
  int grid = want < 1 ? 1 : (want > cap ? cap : want);
  if (args.timeout_cycles <= 0) args.timeout_cycles = 240000000000LL;   // ~2 min at 2 GHz
  void* kargs[] = {(void*)&args};
  // Plain launch: a CTA only ever waits for the SAME-numbered CTA of its peers (never for another CTA of its own grid), so
  // co-residency of the grid is not required and a cooperative launch would only add launch cost.
  cudaError_t e = cudaLaunchKernel(kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: block_reduce launch: ") + cudaGetErrorString(e));
  count_launch();
}

// ------------------------------------------------------------------------------------------------------------------
// DP-FedAvg update clipping (McMahan et al. 2018) — see DPClipArgs in fedb200.h
// ------------------------------------------------------------------------------------------------------------------
// Pass 1 reads z and every local replica once (4 n (n_local + 1) bytes); each CTA stores its partial sums of squares, and
// after grid.sync() every CTA adds the partials in CTA order, so the norms are deterministic and equal in every CTA.
// Squares are summed in double: no finite float32 update can overflow it, so a non-finite norm means a non-finite input.
// Pass 2 rewrites only the replicas over the bound: x <- z + s (x - z), s = C / ||x - z||, in double (an update near the
// float range cannot overflow x - z).  A non-finite norm is never clipped, so NaN / Inf reach the aggregation kernel (and
// its non-finite count) untouched.
__device__ __forceinline__ double warp_add_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double block_add_d(double v, double* sm) {
  v = warp_add_d(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x < 32) {
    r = threadIdx.x < (blockDim.x >> 5) ? sm[threadIdx.x] : 0.0;
    r = warp_add_d(r);
  }
  __syncthreads();
  return r;  // valid in thread 0
}
__global__ void __launch_bounds__(COMM_THREADS, 1) dp_clip_kernel(const DPClipArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double sm[32];
  __shared__ double s_scale[COMM_MAX_LOCAL];
  double* part = reinterpret_cast<double*>(a.stats + DP_PART);     // [COMM_MAX_LOCAL][COMM_MAX_BLOCKS]
  const int n4 = a.n >> 2;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;
  double acc[COMM_MAX_LOCAL];
#pragma unroll
  for (int j = 0; j < COMM_MAX_LOCAL; ++j) acc[j] = 0.0;
  for (int i = tid; i < n4; i += nth) {
    const float4 zv = reinterpret_cast<const float4*>(a.z)[i];
#pragma unroll
    for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
      if (j < a.n_local) {
        const float4 xv = reinterpret_cast<const float4*>(a.x[j])[i];
        const double dx = double(xv.x) - zv.x, dy = double(xv.y) - zv.y, dz = double(xv.z) - zv.z,
                     dw = double(xv.w) - zv.w;
        acc[j] = fma(dx, dx, fma(dy, dy, fma(dz, dz, fma(dw, dw, acc[j]))));
      }
    }
  }
  for (int i = (n4 << 2) + tid; i < a.n; i += nth) {
    const float zv = a.z[i];
#pragma unroll
    for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
      if (j < a.n_local) {
        const double d = double(a.x[j][i]) - zv;
        acc[j] = fma(d, d, acc[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < COMM_MAX_LOCAL; ++j) {
    if (j < a.n_local) {                           // uniform across the CTA: the barriers inside block_add_d are safe
      const double v = block_add_d(acc[j], sm);
      if (threadIdx.x == 0) part[j * COMM_MAX_BLOCKS + blockIdx.x] = v;
    }
  }
  __threadfence();
  grid.sync();

  if (threadIdx.x < a.n_local) {
    const int j = threadIdx.x;
    double s = 0.0;
    for (int b = 0; b < int(gridDim.x); ++b) s += __ldcg(part + j * COMM_MAX_BLOCKS + b);
    const double norm = sqrt(s);
    const bool clip = isfinite(norm) && norm > double(a.bound);
    s_scale[j] = clip ? double(a.bound) / norm : 0.0;
    if (blockIdx.x == 0) {
      a.stats[DP_NORM + j] = float(norm);
      a.stats[DP_CLIPPED + j] = clip ? 1.f : 0.f;
    }
  }
  __syncthreads();
  for (int j = 0; j < a.n_local; ++j) {
    const double s = s_scale[j];
    if (s == 0.0) continue;                        // within the bound (or non-finite): not written at all
    float* x = a.x[j];
    for (int i = tid; i < n4; i += nth) {
      const float4 zv = reinterpret_cast<const float4*>(a.z)[i];
      float4 xv = reinterpret_cast<const float4*>(x)[i];
      xv = make_float4(float(fma(s, double(xv.x) - zv.x, zv.x)), float(fma(s, double(xv.y) - zv.y, zv.y)),
                       float(fma(s, double(xv.z) - zv.z, zv.z)), float(fma(s, double(xv.w) - zv.w, zv.w)));
      reinterpret_cast<float4*>(x)[i] = xv;
    }
    for (int i = (n4 << 2) + tid; i < a.n; i += nth) x[i] = float(fma(s, double(x[i]) - a.z[i], double(a.z[i])));
  }
}

void dp_clip_launch(const DPClipArgs& args, cudaStream_t s) {
  if (args.n_local < 1 || args.n_local > COMM_MAX_LOCAL || args.n < 1)
    throw std::runtime_error("fedb200: dp_clip: bad replica count or block length");
  int cap = comm_max_blocks();
  if (args.max_blocks > 0 && args.max_blocks < cap) cap = args.max_blocks;
  const int want = ((args.n >> 2) + COMM_THREADS - 1) / COMM_THREADS;
  const int grid = want < 1 ? 1 : (want > cap ? cap : want);
  void* kargs[] = {(void*)&args};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)dp_clip_kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: dp_clip launch: ") + cudaGetErrorString(e));
  count_launch();
}

// ------------------------------------------------------------------------------------------------------------------
// Top-k selection of the local replicas' updates (Stich et al. 2018; Lin et al. 2018) — see TopKArgs in fedb200.h
// ------------------------------------------------------------------------------------------------------------------
static_assert(TOPK_TILE == Q_TILE, "a top-k tile is a tile of the compressed tiling");

__device__ __forceinline__ uint32_t topk_key(float u) { return __float_as_uint(u) & 0x7fffffffu; }

// float4 at coordinate c (a multiple of 4) of a length-n vector, from L2 (written by other CTAs of this grid); coordinates
// >= n read as 0
__device__ __forceinline__ float4 ldcg4(const float* p, int c, int n) {
  if (c + 4 <= n) return __ldcg(reinterpret_cast<const float4*>(p + c));
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = c + i < n ? __ldcg(p + c + i) : 0.f;
  return make_float4(v[0], v[1], v[2], v[3]);
}

// exclusive prefix sum over the CTA of one uint32 per thread; *total gets the CTA's sum.  s holds COMM_THREADS / 32 + 1
// words.
__device__ __forceinline__ uint32_t block_exscan_u32(uint32_t v, uint32_t* s, uint32_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s[w] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0u;
    for (int i = 0; i < int(blockDim.x >> 5); ++i) {
      const uint32_t t = s[i];
      s[i] = run;
      run += t;
    }
    s[COMM_THREADS / 32] = run;
  }
  __syncthreads();
  const uint32_t r = s[w] + incl - v;
  *total = s[COMM_THREADS / 32];
  __syncthreads();
  return r;
}

// histogram update of one warp-wide batch of bins (bin TOPK_RADIX = no count): lanes with the same bin add once
__device__ __forceinline__ void topk_hist_add(uint32_t* h, uint32_t bin) {
  const unsigned peers = __match_any_sync(0xffffffffu, bin);
  if (bin < TOPK_RADIX && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(h + bin, uint32_t(__popc(peers)));
}

__global__ void __launch_bounds__(COMM_THREADS, 1) topk_select_kernel(const TopKArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ uint32_t s_hist[COMM_MAX_LOCAL * TOPK_RADIX];
  __shared__ uint32_t s_thr[COMM_MAX_LOCAL];     // replica j's threshold key, digit by digit
  __shared__ uint32_t s_need[COMM_MAX_LOCAL];    // keys still to select at or below the digits fixed so far
  __shared__ uint32_t s_scan[COMM_THREADS / 32 + 1];
  __shared__ float sm[32];
  const TopKLayout L = topk_layout(a.n, a.k);
  const int T = L.tiles;
  uint32_t* hist = reinterpret_cast<uint32_t*>(a.ws);                    // [4][COMM_MAX_LOCAL][TOPK_RADIX]
  uint32_t* cnt_gt = hist + 4 * COMM_MAX_LOCAL * TOPK_RADIX;             // [n_local][T] keys above the threshold
  uint32_t* cnt_eq = cnt_gt + a.n_local * T;                            // [n_local][T] keys equal to it
  uint32_t* take_eq = cnt_eq + a.n_local * T;                           // [n_local][T] of those, selected
  const int lane = threadIdx.x & 31;
  const int wtid = blockIdx.x * blockDim.x + threadIdx.x - lane;        // warp-uniform loops: every lane takes part
  const int nth = gridDim.x * blockDim.x;
  const int n4 = a.n >> 2;
  if (threadIdx.x < COMM_MAX_LOCAL) {
    s_thr[threadIdx.x] = 0u;
    s_need[threadIdx.x] = uint32_t(a.k);
  }

  // ---- radix select of the k-th largest key, 8 bits per pass from bit 24 (keys have 31 bits) -------------------
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t hmask = pass == 0 ? 0u : 0xffffffffu << (shift + 8);
    for (int i = threadIdx.x; i < a.n_local * TOPK_RADIX; i += blockDim.x) s_hist[i] = 0u;
    __syncthreads();
    for (int j = 0; j < a.n_local; ++j) {
      const uint32_t pre = s_thr[j];
      uint32_t* h = s_hist + j * TOPK_RADIX;
      float* u = a.ef[j] != nullptr ? a.ef[j] : a.u[j];
      for (int b = wtid; b < n4; b += nth) {
        const int i = b + lane;
        float4 uv = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool on = i < n4;
        if (on && pass == 0) {                     // materialise u = (x - z) + e once
          const float4 xv = reinterpret_cast<const float4*>(a.x[j])[i];
          const float4 zv = reinterpret_cast<const float4*>(a.z)[i];
          const float4 ev = a.ef[j] != nullptr ? reinterpret_cast<const float4*>(a.ef[j])[i] : uv;
          uv = make_float4(__fadd_rn(__fsub_rn(xv.x, zv.x), ev.x), __fadd_rn(__fsub_rn(xv.y, zv.y), ev.y),
                           __fadd_rn(__fsub_rn(xv.z, zv.z), ev.z), __fadd_rn(__fsub_rn(xv.w, zv.w), ev.w));
          reinterpret_cast<float4*>(u)[i] = uv;
        } else if (on) {
          uv = __ldcg(reinterpret_cast<const float4*>(u) + i);
        }
        const float w4[4] = {uv.x, uv.y, uv.z, uv.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t key = topk_key(w4[q]);
          topk_hist_add(h, on && (key & hmask) == pre ? (key >> shift) & (TOPK_RADIX - 1) : TOPK_RADIX);
        }
      }
      for (int b = (n4 << 2) + wtid; b < a.n; b += nth) {   // scalar tail (n % 4 coordinates)
        const int i = b + lane;
        const bool on = i < a.n;
        float uv = 0.f;
        if (on && pass == 0) {
          uv = __fadd_rn(__fsub_rn(a.x[j][i], a.z[i]), a.ef[j] != nullptr ? a.ef[j][i] : 0.f);
          u[i] = uv;
        } else if (on) {
          uv = __ldcg(u + i);
        }
        const uint32_t key = topk_key(uv);
        topk_hist_add(h, on && (key & hmask) == pre ? (key >> shift) & (TOPK_RADIX - 1) : TOPK_RADIX);
      }
    }
    __syncthreads();
    uint32_t* gh = hist + pass * COMM_MAX_LOCAL * TOPK_RADIX;
    for (int i = threadIdx.x; i < a.n_local * TOPK_RADIX; i += blockDim.x)
      if (s_hist[i] != 0u) atomicAdd(gh + i, s_hist[i]);
    grid.sync();
    for (int i = threadIdx.x; i < a.n_local * TOPK_RADIX; i += blockDim.x) s_hist[i] = __ldcg(gh + i);
    __syncthreads();                             // (the walk below then costs shared-memory latency, not L2 round trips)
    if (threadIdx.x < a.n_local) {               // every CTA fixes the same digit: the largest d with count(>= d) >= need
      const int j = threadIdx.x;
      const uint32_t need = s_need[j];
      uint32_t above = 0u;
      int d = TOPK_RADIX - 1;
      for (; d > 0; --d) {
        const uint32_t c = s_hist[j * TOPK_RADIX + d];
        if (above + c >= need) break;
        above += c;
      }
      s_need[j] = need - above;
      s_thr[j] |= uint32_t(d) << shift;
    }
    __syncthreads();
  }

  // ---- per tile: keys above and equal to the threshold ------------------------------------------------------------
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    const int c0 = t * TOPK_TILE + Q_SEG * threadIdx.x;
    for (int j = 0; j < a.n_local; ++j) {
      const float* u = a.ef[j] != nullptr ? a.ef[j] : a.u[j];
      const uint32_t thr = s_thr[j];
      uint32_t gt = 0u, eq = 0u;
#pragma unroll
      for (int q = 0; q < Q_SEG / 4; ++q) {
        const int c = c0 + 4 * q;
        const float4 uv = ldcg4(u, c, a.n);
        const float w4[4] = {uv.x, uv.y, uv.z, uv.w};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const uint32_t key = topk_key(w4[r]);
          if (c + r < a.n) {
            gt += key > thr ? 1u : 0u;
            eq += key == thr ? 1u : 0u;
          }
        }
      }
      uint32_t tot;
      block_exscan_u32((eq << 16) | gt, s_scan, &tot);   // <= 8192 each: the halves do not carry into each other
      if (threadIdx.x == 0) {
        cnt_gt[j * T + t] = tot & 0xffffu;
        cnt_eq[j * T + t] = tot >> 16;
      }
    }
  }
  grid.sync();

  // ---- CTA j scans replica j's tiles: tile offsets, and the equal keys each tile takes in index order ------------
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 4 * COMM_MAX_LOCAL * TOPK_RADIX; i += nth)
    hist[i] = 0u;                                // every CTA has read the histograms: clean for the next launch
  if (blockIdx.x < a.n_local) {
    const int j = blockIdx.x;
    const uint32_t need = s_need[j];
    uint32_t* off = a.pay[j];
    uint32_t run_sel = 0u, run_eq = 0u;
    for (int base = 0; base < T; base += blockDim.x) {
      const int t = base + threadIdx.x;
      const uint32_t gt = t < T ? __ldcg(cnt_gt + j * T + t) : 0u;
      const uint32_t eq = t < T ? __ldcg(cnt_eq + j * T + t) : 0u;
      uint32_t tot_eq, tot_sel;
      const uint32_t eq_before = run_eq + block_exscan_u32(eq, s_scan, &tot_eq);
      const uint32_t take = eq_before >= need ? 0u : min(eq, need - eq_before);
      const uint32_t sel_before = run_sel + block_exscan_u32(gt + take, s_scan, &tot_sel);
      if (t < T) {
        off[t] = sel_before;
        take_eq[j * T + t] = take;
      }
      run_eq += tot_eq;
      run_sel += tot_sel;
    }
    if (threadIdx.x == 0) off[T] = run_sel;      // = k
  }
  grid.sync();

  // ---- per tile: entries in index order, error feedback, statistics --------------------------------------------------
  float err = 0.f, nrm = 0.f;
  for (int t = blockIdx.x; t < T; t += gridDim.x) {
    const int c0 = t * TOPK_TILE + Q_SEG * threadIdx.x;
    for (int j = 0; j < a.n_local; ++j) {
      float* u = a.ef[j] != nullptr ? a.ef[j] : a.u[j];
      const uint32_t thr = s_thr[j];
      const uint32_t take = __ldcg(take_eq + j * T + t);
      float v[Q_SEG];
      uint32_t gt = 0u, eq = 0u;
#pragma unroll
      for (int q = 0; q < Q_SEG / 4; ++q) q_unf4(v, q, ldcg4(u, c0 + 4 * q, a.n));
#pragma unroll
      for (int i = 0; i < Q_SEG; ++i) {
        const uint32_t key = topk_key(v[i]);
        if (c0 + i < a.n) {
          gt += key > thr ? 1u : 0u;
          eq += key == thr ? 1u : 0u;
        }
      }
      uint32_t tot;
      const uint32_t ex = block_exscan_u32((eq << 16) | gt, s_scan, &tot);
      uint32_t eq_seen = ex >> 16;
      uint32_t pos = __ldcg(a.pay[j] + t) + (ex & 0xffffu) + min(eq_seen, take);
      float* val = reinterpret_cast<float*>(a.pay[j] + L.val);
      uint16_t* idx = reinterpret_cast<uint16_t*>(a.pay[j] + L.idx);
#pragma unroll
      for (int i = 0; i < Q_SEG; ++i) {
        const int c = c0 + i;
        if (c >= a.n) break;
        const uint32_t key = topk_key(v[i]);
        bool sel = key > thr;
        if (key == thr) sel = eq_seen++ < take;
        nrm = fmaf(v[i], v[i], nrm);
        if (sel) {
          val[pos] = v[i];
          idx[pos] = uint16_t(c - t * TOPK_TILE);
          ++pos;
          if (a.ef[j] != nullptr) u[c] = 0.f;     // e <- u - s: 0 where selected, u (already stored) elsewhere
        } else {
          err = fmaf(v[i], v[i], err);
        }
      }
    }
  }
  err = block_add(err, sm);
  nrm = block_add(nrm, sm);
  if (threadIdx.x == 0) {
    a.stats[2 + 2 * blockIdx.x] = err;
    a.stats[3 + 2 * blockIdx.x] = nrm;
  }
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) {     // in CTA order: the same bits on every run
    float e = 0.f, s = 0.f;
    for (int b = 0; b < int(gridDim.x); ++b) {
      e += __ldcg(a.stats + 2 + 2 * b);
      s += __ldcg(a.stats + 3 + 2 * b);
    }
    a.stats[0] = e;
    a.stats[1] = s;
  }
}

void topk_select_launch(const TopKArgs& args, cudaStream_t s) {
  if (args.n_local < 1 || args.n_local > COMM_MAX_LOCAL || args.n < 1 || args.k < 1 || args.k > args.n)
    throw std::runtime_error("fedb200: topk_select: needs 1 to 16 replicas and 1 <= k <= n");
  int cap = comm_max_blocks();
  if (args.max_blocks > 0 && args.max_blocks < cap) cap = args.max_blocks;
  if (cap < args.n_local) throw std::runtime_error("fedb200: topk_select: needs at least one CTA per replica");
  const int want = ((args.n >> 2) + COMM_THREADS - 1) / COMM_THREADS;
  const int grid = want < args.n_local ? args.n_local : (want > cap ? cap : want);
  void* kargs[] = {(void*)&args};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)topk_select_kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: topk_select launch: ") + cudaGetErrorString(e));
  count_launch();
}

// ------------------------------------------------------------------------------------------------------------------
// Barzilai-Borwein adaptive rho (consensus_multi.py:242-278) — see BBArgs in fedb200.h
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(COMM_THREADS, 1) bb_update_kernel(const BBArgs a) {
  cg::grid_group grid = cg::this_grid();
  __shared__ float sm[32];
  __shared__ int s_abort;
  if (threadIdx.x == 0) s_abort = 0;
  __syncthreads();
  const uint32_t epoch = a.sync[0] + 1;
  const int n4 = a.n >> 2;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nth = gridDim.x * blockDim.x;
  float* dots = a.scratch;                         // [n_local][8]
  float* rho_turn = a.scratch + 8 * COMM_MAX_LOCAL + 8;   // [n_local]

  if (!a.seed_only) {
    // ---- six dots per local worker: a = y - yhat0, b = x - z, c = x - x0 ----------------------------------------
    for (int j = 0; j < a.n_local; ++j) {
      float d[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int i = tid; i < n4; i += nth) {
        const float4 xv = reinterpret_cast<const float4*>(a.x[j])[i];
        const float4 yv = reinterpret_cast<const float4*>(a.y[j])[i];
        const float4 hv = reinterpret_cast<const float4*>(a.yhat0[j])[i];
        const float4 ov = reinterpret_cast<const float4*>(a.x0[j])[i];
        const float4 zv = reinterpret_cast<const float4*>(a.z)[i];
        const float av[4] = {yv.x - hv.x, yv.y - hv.y, yv.z - hv.z, yv.w - hv.w};
        const float bv[4] = {xv.x - zv.x, xv.y - zv.y, xv.z - zv.z, xv.w - zv.w};
        const float cv[4] = {xv.x - ov.x, xv.y - ov.y, xv.z - ov.z, xv.w - ov.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          d[0] = fmaf(av[q], av[q], d[0]); d[1] = fmaf(av[q], bv[q], d[1]); d[2] = fmaf(bv[q], bv[q], d[2]);
          d[3] = fmaf(av[q], cv[q], d[3]); d[4] = fmaf(bv[q], cv[q], d[4]); d[5] = fmaf(cv[q], cv[q], d[5]);
        }
      }
      for (int i = (n4 << 2) + tid; i < a.n; i += nth) {
        const float av = a.y[j][i] - a.yhat0[j][i], bv = a.x[j][i] - a.z[i], cv = a.x[j][i] - a.x0[j][i];
        d[0] = fmaf(av, av, d[0]); d[1] = fmaf(av, bv, d[1]); d[2] = fmaf(bv, bv, d[2]);
        d[3] = fmaf(av, cv, d[3]); d[4] = fmaf(bv, cv, d[4]); d[5] = fmaf(cv, cv, d[5]);
      }
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const float v = block_add(d[q], sm);
        if (threadIdx.x == 0) atomicAdd(dots + 8 * j + q, v);
      }
    }
    grid.sync();

    // ---- gather the rows of all K workers, replay the sequential rule (every rank computes the same thing) ----
    if (blockIdx.x == 0) {
      float* my_rows = reinterpret_cast<float*>(a.ctrl[a.rank] + PAD_BBROWS);
      if (a.world > 1) {
        if (threadIdx.x < a.world) {
          float* rows = reinterpret_cast<float*>(a.ctrl[threadIdx.x] + PAD_BBROWS);
          for (int j = 0; j < a.n_local; ++j)
            for (int q = 0; q < 6; ++q) st_sys_f32(rows + 8 * a.worker[j] + q, __ldcg(dots + 8 * j + q));
          peer_post_wait(a.ctrl, a.rank, PAD_FLAG_D, epoch, a.timeout_cycles, a.out + OUT_STATUS, &s_abort);
        }
      } else if (threadIdx.x == 0) {
        for (int j = 0; j < a.n_local; ++j)
          for (int q = 0; q < 6; ++q) my_rows[8 * a.worker[j] + q] = __ldcg(dots + 8 * j + q);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        double rho = double(*a.rho_dev);
        for (int ck = 0; ck < a.K; ++ck) {
          const float* r = my_rows + 8 * ck;
          const double aa = ld_sys_f32(r + 0), ab = ld_sys_f32(r + 1), bb = ld_sys_f32(r + 2);
          const double ac = ld_sys_f32(r + 3), bc = ld_sys_f32(r + 4), cc = ld_sys_f32(r + 5);
          for (int j = 0; j < a.n_local; ++j)
            if (a.worker[j] == ck) rho_turn[j] = float(rho);     // the penalty in force at this worker's turn
          const double d11 = aa + 2.0 * rho * ab + rho * rho * bb, d12 = ac + rho * bc, d22 = cc;
          double alpha = 0.0, aSD = 0.0, aMG = 0.0, tested = 0.0, rhonew = rho;
          if (fabs(d12) > a.epsilon && d11 > a.epsilon && d22 > a.epsilon) {
            tested = 1.0;
            alpha = d12 / sqrt(d11 * d22);
            aSD = d11 / d22;
            aMG = d12 / d22;
            const double ahat = (2.0 * aMG > aSD) ? aMG : aSD - 0.5 * aMG;
            if (alpha >= a.alphacorrmin && ahat < a.rhomax) rhonew = ahat;
          }
          rho = rhonew;
          float* lg = a.log + 8 * ck;
          lg[0] = float(d11); lg[1] = float(d12); lg[2] = float(d22); lg[3] = float(alpha); lg[4] = float(aSD);
          lg[5] = float(aMG); lg[6] = float(tested); lg[7] = float(rho);
        }
        *a.rho_dev = float(rho);
        __threadfence();
      }
    }
    grid.sync();
  }

  // ---- carry forward: yhat0_k <- y_k + rho_k (x_k - z), x0_k <- x_k -----------------------------------------------
  for (int j = 0; j < a.n_local; ++j) {
    const float rk = a.seed_only ? 0.f : __ldcg(rho_turn + j);
    for (int i = tid; i < n4; i += nth) {
      const float4 xv = reinterpret_cast<const float4*>(a.x[j])[i];
      if (!a.seed_only) {
        const float4 yv = reinterpret_cast<const float4*>(a.y[j])[i];
        const float4 zv = reinterpret_cast<const float4*>(a.z)[i];
        reinterpret_cast<float4*>(a.yhat0[j])[i] = make_float4(fmaf(rk, xv.x - zv.x, yv.x), fmaf(rk, xv.y - zv.y, yv.y),
                                                               fmaf(rk, xv.z - zv.z, yv.z), fmaf(rk, xv.w - zv.w, yv.w));
      }
      reinterpret_cast<float4*>(a.x0[j])[i] = xv;
    }
    for (int i = (n4 << 2) + tid; i < a.n; i += nth) {
      if (!a.seed_only) a.yhat0[j][i] = fmaf(rk, a.x[j][i] - a.z[i], a.y[j][i]);
      a.x0[j][i] = a.x[j][i];
    }
  }
  if (a.seed_only) return;
  grid.sync();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int j = 0; j < BB_SCRATCH_FLOATS; ++j) a.scratch[j] = 0.f;
    __threadfence();
    a.sync[0] = epoch;
  }
}

void bb_update_launch(const BBArgs& args_in, cudaStream_t s) {
  BBArgs args = args_in;
  if (args.K < 1 || args.K > COMM_MAX_K || args.n_local > COMM_MAX_LOCAL || args.world > COMM_MAX_WORLD)
    throw std::runtime_error("fedb200: bb_update: limits exceeded");
  int cap = comm_max_blocks();
  if (args.max_blocks > 0 && args.max_blocks < cap) cap = args.max_blocks;
  int want = ((args.n >> 2) + COMM_THREADS - 1) / COMM_THREADS;
  int grid = want < 1 ? 1 : (want > cap ? cap : want);
  if (args.timeout_cycles <= 0) args.timeout_cycles = 240000000000LL;
  void* kargs[] = {(void*)&args};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)bb_update_kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: bb_update launch: ") + cudaGetErrorString(e));
  count_launch();
}

}  // namespace fedb200

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
//   C. the last CTA to finish exchanges the scalars (dual part, primal part, #non-finite) through the control pads
//      and writes the result record.
//
// CTA b works on the SAME index set on every rank and in both passes, so barriers A and B only involve CTA b of each
// rank (threads 0..world-1 signal / poll one peer each): there is no grid-wide barrier in the kernel.
//
// mode: 0 = FedAvg (z = sum x / K, write-back), 1 = FedProx (no write-back), 2 = ADMM (z = sum(y + rho x)/(K rho)).
// Reference sites: /root/reference/src/federated_multi.py:203-217, fedprox_multi.py:211-232, consensus_multi.py:242-299.
#include "fedb200.h"

#include <cooperative_groups.h>
#include <cstdlib>
#include <stdexcept>
#include <string>

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

__global__ void __launch_bounds__(COMM_THREADS, 1) block_reduce_kernel(const CommArgs a) {
  __shared__ float sm[32];
  __shared__ int s_abort;
  __shared__ int s_last;
  if (threadIdx.x == 0) { s_abort = 0; s_last = 0; }
  __syncthreads();
  const uint32_t epoch = a.sync[0] + 1;
  const float rho = a.rho_dev != nullptr ? __ldg(a.rho_dev) : a.rho;
  const float inv_scale = a.mode == 2 ? 1.f / (float(a.K) * rho) : 1.f / float(a.K);
  const int n4 = a.n >> 2;
  const int nslices = a.two_shot ? a.world : 1;
  const int chunk4 = a.two_shot ? (n4 + a.world - 1) / a.world : n4;
  const int my_slice = a.two_shot ? a.rank : 0;
  const int stride = gridDim.x * blockDim.x;
  const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
  const bool use_mc = a.mc_x != nullptr && (a.mode != 2 || a.mc_y != nullptr);

  // ---- A: inputs of every rank are final (their producers precede this kernel in stream order) ----------------
  cta_peer_barrier(a.ctrl, a.world, a.rank, PAD_FLAG_A, epoch, a.timeout_cycles, a.out + OUT_STATUS, &s_abort);

  // ---- 1: reduce, scale, new z, dual residual ---------------------------------------------------------------------
  float dual = 0.f, bad = 0.f;
  {
    const int lo = my_slice * chunk4;
    const int hi = min(n4, lo + chunk4);
    // two elements per thread and iteration: their (remote) loads are issued back to back, so twice as many bytes are in
    // flight per thread — the pass is bound by NVLink round trips, not by issue slots
    for (int i = lo + t0; i < hi; i += 2 * stride) {
      const int i1 = i + stride;
      const bool has1 = i1 < hi;
      const size_t off0 = 4 * size_t(i), off1 = 4 * size_t(has1 ? i1 : i);
      float4 accs[2];
      accs[0] = gather_v4(a, off0, rho, use_mc);
      accs[1] = has1 ? gather_v4(a, off1, rho, use_mc) : accs[0];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (u == 1 && !has1) break;
        const size_t off = u == 0 ? off0 : off1;
        const float4 acc = accs[u];
        const float4 zn = make_float4(acc.x * inv_scale, acc.y * inv_scale, acc.z * inv_scale, acc.w * inv_scale);
        if (!(a.two_shot && a.mode == 0)) {       // two-shot FedAvg takes both from the finished weights in pass 2
          const float4 zo = *reinterpret_cast<const float4*>(a.z + off);
          const float dx = zo.x - zn.x, dy = zo.y - zn.y, dz = zo.z - zn.z, dw = zo.w - zn.w;
          dual = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, dual))));
          if (!(isfinite(zn.x) && isfinite(zn.y) && isfinite(zn.z) && isfinite(zn.w))) bad += 1.f;
        }
        if (!a.two_shot) {
          *reinterpret_cast<float4*>(a.z + off) = zn;
        } else if (a.mode == 0) {                 // broadcast the averaged weights into every rank's replica
          if (a.mc_x != nullptr) multimem_st_v4(a.mc_x + off, zn);
          else for (int p = 0; p < a.world; ++p) st_sys_v4(a.xw[p] + off, zn);
        } else {                                   // broadcast the consensus vector
          if (a.mc_z != nullptr) multimem_st_v4(a.mc_z + off, zn);
          else for (int p = 0; p < a.world; ++p) st_sys_v4(a.zw[p] + off, zn);
        }
      }
    }
  }
  // scalar tail (n % 4 elements): every rank reduces it for itself, one-shot style
  const int tail0 = n4 << 2;
  if (blockIdx.x == 0 && tail0 + int(threadIdx.x) < a.n) {
    const int i = tail0 + threadIdx.x;
    float acc = 0.f;
    if (use_mc) {
      acc = multimem_ld_reduce_f32(a.mc_x + i);
      if (a.mode == 2) acc = fmaf(rho, acc, multimem_ld_reduce_f32(a.mc_y + i));
    } else {
      for (int k = 0; k < a.K; ++k) {
        const float xv = ld_sys_f32(a.x[k] + i);
        acc += a.mode == 2 ? fmaf(rho, xv, ld_sys_f32(a.y[k] + i)) : xv;
      }
    }
    const float zn = acc * inv_scale;
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
  for (int s = 0; s < nslices; ++s) {
    const int lo = s * chunk4;
    const int hi = min(n4, lo + chunk4);
    for (int i = lo + t0; i < hi; i += stride) {
      const size_t off = 4 * size_t(i);
      if (a.mode == 0) {
        if (a.two_shot) {                        // weights already hold the average: keep a copy as next round's z_old,
          const float4 zn = ld_sys_v4(a.xl[0] + off);          // and take the dual residual + NaN check from it (the full vector
          const float4 zo = *reinterpret_cast<const float4*>(a.z + off);   // is local now: no cross-rank sum needed)
          const float dx = zo.x - zn.x, dy = zo.y - zn.y, dz = zo.z - zn.z, dw = zo.w - zn.w;
          dual = fmaf(dx, dx, fmaf(dy, dy, fmaf(dz, dz, fmaf(dw, dw, dual))));
          if (!(isfinite(zn.x) && isfinite(zn.y) && isfinite(zn.z) && isfinite(zn.w))) bad += 1.f;
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
  if (blockIdx.x == 0 && tail0 + int(threadIdx.x) < a.n) {
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

  // ---- C: exchange and finish the scalars (one CTA) -------------------------------------------------------------
  __shared__ float s_vals[3];
  if (threadIdx.x == 0) {
    __threadfence();
    float local = 0.f;
    for (int j = 0; j < a.n_local; ++j) local += sqrtf(__ldcg(a.scratch + 4 + j));
    s_vals[0] = __ldcg(a.scratch + 0);
    s_vals[1] = local;
    s_vals[2] = __ldcg(a.scratch + 1);
    for (int j = 0; j < COMM_SCRATCH_FLOATS; ++j) a.scratch[j] = 0.f;      // self-cleaning: no memset per launch
  }
  __syncthreads();
  float dual_sq = s_vals[0], primal = s_vals[1], nonfinite = s_vals[2];
  if (a.world > 1 && a.mode != 0) {          // FedAvg: every rank already holds the complete dual residual and NaN count
    if (threadIdx.x < a.world) {
      float* pay = reinterpret_cast<float*>(a.ctrl[threadIdx.x] + PAD_PAYLOAD) + 4 * a.rank;
      st_sys_f32(pay + 0, dual_sq);
      st_sys_f32(pay + 1, primal);
      st_sys_f32(pay + 2, nonfinite);
      __threadfence_system();
      st_release_sys(a.ctrl[threadIdx.x] + PAD_FLAG_C + a.rank, epoch);
      if (s_abort == 0 && !wait_flag(a.ctrl[a.rank] + PAD_FLAG_C + threadIdx.x, epoch, a.timeout_cycles)) {
        a.out[OUT_STATUS] = 100.f + float(threadIdx.x);
        atomicExch(&s_abort, 1);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const float* pay = reinterpret_cast<const float*>(a.ctrl[a.rank] + PAD_PAYLOAD);
      float d = 0.f, p = 0.f, b = 0.f;
      for (int r = 0; r < a.world; ++r) {
        d += ld_sys_f32(pay + 4 * r + 0);
        p += ld_sys_f32(pay + 4 * r + 1);
        b += ld_sys_f32(pay + 4 * r + 2);
      }
      if (a.two_shot) dual_sq = d;      // one-shot: every rank already holds the full sum
      primal = p;
      nonfinite = a.two_shot ? b : nonfinite;
    }
  }
  if (threadIdx.x == 0) {
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

static int env_int_c(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return v ? std::atoi(v) : dflt;
}

static int comm_max_blocks(const void* kernel) {
  int dev = 0, sms = 0, per = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, COMM_THREADS, 0);
  int m = sms * (per < 1 ? 1 : 1);                    // one CTA per SM (132 on an H100 SXM) x 512 threads
  if (m > COMM_MAX_BLOCKS) m = COMM_MAX_BLOCKS;
  const int cap = env_int_c("FEDB200_COMM_BLOCKS", 0);
  if (cap > 0 && cap < m) m = cap;
  return m < 1 ? 1 : m;
}

void block_reduce_launch(const CommArgs& args_in, cudaStream_t s) {
  CommArgs args = args_in;
  if (args.K < 1 || args.K > COMM_MAX_K || args.n_local > COMM_MAX_LOCAL || args.world > COMM_MAX_WORLD)
    throw std::runtime_error("fedb200: block_reduce: too many contributions / replicas / ranks");
  if (args.two_shot && (args.world <= 1 || args.n_local != 1 || args.K != args.world))
    throw std::runtime_error("fedb200: two-shot aggregation needs one replica per rank");
  static int max_blocks = 0;
  if (max_blocks == 0) max_blocks = comm_max_blocks((const void*)block_reduce_kernel);
  int cap = max_blocks;
  if (args.max_blocks > 0 && args.max_blocks < cap) cap = args.max_blocks;
  const int n4 = args.n >> 2;
  const int work4 = args.two_shot ? (n4 + args.world - 1) / args.world : n4;
  int want = (work4 + COMM_THREADS - 1) / COMM_THREADS;
  int grid = want < 1 ? 1 : (want > cap ? cap : want);
  if (args.timeout_cycles <= 0) args.timeout_cycles = 240000000000LL;   // ~2 min at 2 GHz
  void* kargs[] = {(void*)&args};
  // Plain launch: a CTA only ever waits for the SAME-numbered CTA of its peers (never for another CTA of its own grid), so
  // co-residency of the grid is not required and a cooperative launch only adds launch cost.  FEDB200_COMM_COOP=1 restores
  // it (A/B runs).
  static const int coop = env_int_c("FEDB200_COMM_COOP", 0);
  cudaError_t e;
  if (coop) e = cudaLaunchCooperativeKernel((void*)block_reduce_kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  else e = cudaLaunchKernel((void*)block_reduce_kernel, dim3(grid), dim3(COMM_THREADS), kargs, 0, s);
  if (e != cudaSuccess) throw std::runtime_error(std::string("fedb200: block_reduce launch: ") + cudaGetErrorString(e));
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
  unsigned* ticket = reinterpret_cast<unsigned*>(a.scratch + 8 * COMM_MAX_LOCAL);
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
          __threadfence_system();
          st_release_sys(a.ctrl[threadIdx.x] + PAD_FLAG_D + a.rank, epoch);
          if (!wait_flag(a.ctrl[a.rank] + PAD_FLAG_D + threadIdx.x, epoch, a.timeout_cycles)) {
            a.out[OUT_STATUS] = 100.f + float(threadIdx.x);
            atomicExch(&s_abort, 1);
          }
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
    (void)ticket;
    __threadfence();
    a.sync[0] = epoch;
  }
}

void bb_update_launch(const BBArgs& args_in, cudaStream_t s) {
  BBArgs args = args_in;
  if (args.K < 1 || args.K > COMM_MAX_K || args.n_local > COMM_MAX_LOCAL || args.world > COMM_MAX_WORLD)
    throw std::runtime_error("fedb200: bb_update: limits exceeded");
  static int max_blocks = 0;
  if (max_blocks == 0) max_blocks = comm_max_blocks((const void*)bb_update_kernel);
  int cap = max_blocks;
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

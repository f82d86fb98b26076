// Launcher declarations shared by the .cu translation units (torch-free) and bindings.cpp (torch glue).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fedb200 {

// every kernel launcher bumps this; bindings expose it so benchmarks can report `gpu_launches`
void count_launch(int n = 1);
long long launch_count();

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------
// A training step is ~200 short kernels: launch latency + CTA ramp-up of kernel N+1 is hidden behind
// the tail of kernel N by letting N+1 become resident early.  Every kernel launched through launch_pdl() executes
// pdl_launch_dependents() first (lets ITS successor start scheduling) and pdl_wait() before its first global-memory
// access (blocks until the predecessor grid has completed and flushed).  Opt-in with FEDB200_PDL=1: inside the
// CUDA-graph step the launch gaps are already hidden.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

// ---- wgmma implicit GEMM (gemm_wgmma.cu) -----------------------------------------------------------
int pick_block_n(int M, int N);
void linear_tf32(const float* x, const float* w, const float* bias, float* out, int M, int N, int K, int ldx, int ldw,
                 int ldo, int act, cudaStream_t stream);
bool conv_geometry_supported(int H_out, int W_out, int C_in, int stride);
void conv2d_nhwc_tf32(const float* x, const float* w, float* y, float* stats, int NB, int H, int W, int C_in, int C_out,
                      int kh, int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream);
// y += conv(x, w) (experimental: residual-gradient accumulation fused into the data-gradient convolution)
void conv2d_nhwc_accumulate_tf32(const float* x, const float* w, float* y, int NB, int H, int W, int C_in, int C_out, int kh,
                                 int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream);
// same kernel with bias + optional ELU in the epilogue (no statistics, no split-K): VAE / CPC convolutions
void conv2d_nhwc_bias_act_tf32(const float* x, const float* w, const float* bias, int act, float* y, int NB, int H, int W,
                               int C_in, int C_out, int kh, int kw, int stride, int pad, int dil, int H_out, int W_out,
                               cudaStream_t stream);

// phase-packed stride-1 conv stored straight into the pixel-shuffled [N, 2Ho, 2Wo, C4/4] result (stride-2 dgrad, transposed conv)
bool conv_shuffle_supported(int H_out, int W_out, int C_in, int Ci_out);
void conv2d_nhwc_shuffle_tf32(const float* x, const float* w, float* out, int NB, int H, int W, int C_in, int C4, int kh, int kw,
                              int pad, int H_out, int W_out, cudaStream_t stream);
// `branches` dilated convolutions of one input as one launch writing the concatenated output (CPC encoder stem)
bool conv_multidil_supported(int H_out, int W_out, int C_in, int stride, int branches);
void conv2d_nhwc_multidil_tf32(const float* x, const float* w, const float* bias, int act, float* y, int NB, int H, int W, int C_in,
                               int C_out, int branches, int kh, int kw, int stride, const int* dils, const int* pads, int H_out,
                               int W_out, cudaStream_t stream);
// weight gradient on wgmma (operands gathered K-major into shared memory, split over the pixel range, red.add into dw)
bool conv_wgrad_supported(int C_x, int C_out, int stride, int W_out, int H_out);
void conv_wgrad_tf32(const float* x, const float* dy, float* dw, int NB, int H, int W, int C_x, int C_w, int C_out, int kh,
                     int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream);


// ---- flat-vector kernels (flat_kernels.cu) ---------------------------------------------------------
void adam_prox(float* x, const float* g, float* m, float* v, const int* step_dev, int n, float lr, float b1, float b2,
               float eps, const float* z, const float* y, float rho, float l1, float l2, cudaStream_t s,
               const float* rho_dev = nullptr);
void bump_step(int* step_dev, cudaStream_t s);
void l1_l2(const float* g, int n, float* out2, cudaStream_t s);
void make_pair(const float* g, const float* gprev, const float* d, float t, float trust, float* y, float* sv, int n,
               float* out3, cudaStream_t s);
void welford(const float* g, float* mean, float* m2, int n, float inv_n, float* out1, cudaStream_t s);
void penalty_value(const float* x, const float* z, const float* y, float rho, float l1, float l2, int n, float* out1,
                   cudaStream_t s);
void penalty_grad(float* g, const float* x, const float* z, const float* y, float rho, float l1, float l2, int n,
                  cudaStream_t s);
void multi_dot(const float* const* a, const float* const* b, int npairs, int n, float* out, cudaStream_t s);
void lbfgs_two_loop(const float* Y, const float* S, const int* order, int k, int n, int ld, const float* g, float hdiag,
                    float* d, float* work, cudaStream_t s);
size_t lbfgs_two_loop_work_floats(int k);

// ---- elementwise / normalisation (elementwise_kernels.cu) ------------------------------------------
void normalize_u8_nhwc(const uint8_t* in, float* out, int npix, int c_out, const float* mean3, const float* std3,
                       int to_nchw, int H, int W, cudaStream_t s);
void col_stats(const float* y, float* stats, int M, int C, cudaStream_t s);
// stats: [2C] sums (+ one uint counter behind them when self_clean: the kernel zeroes the buffer after the last read)
void bn_elu_fwd(const float* y, float* stats, const float* gamma, const float* beta, const float* residual,
                float* out, float* running_mean, float* running_var, float* save_mean, float* save_invstd, int M, int C,
                float eps, float momentum, int act, int self_clean, cudaStream_t s);
// out == nullptr (allowed when the layer had no residual input): ELU' is recomputed from y, gamma, beta
void bn_elu_bwd_reduce(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                       const float* gamma, const float* beta, float* sums, int M, int C, int act, int sums_clean, cudaStream_t s);
void bn_elu_bwd_apply(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, float* sums, float* dy, float* dres, float* dgamma,
                      float* dbeta, int M, int C, int act, int self_clean, cudaStream_t s);
// experimental single-kernel backward for small tensors (returns false when not applicable; sums: [2C] scratch)
bool bn_elu_bwd_fused(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, float* sums, float* dy, float* dres, float* dgamma,
                      float* dbeta, int M, int C, int act, cudaStream_t s);
// experimental fused classifier head: avg-pool over HW + Linear (true fp32), O <= 32 outputs
void head_fwd(const float* x, const float* w, const float* bias, float* pooled, float* logits, int NB, int HW, int C, int O,
              cudaStream_t s);
void head_bwd(const float* dlogits, const float* w, float* dx, int NB, int HW, int C, int O, cudaStream_t s);
void avgpool_nhwc(const float* x, float* out, int NB, int HW, int C, cudaStream_t s);
void avgpool_nhwc_bwd(const float* dout, float* dx, int NB, int HW, int C, cudaStream_t s);
void weight_krsc_flip(const float* w, float* out, int C_out, int C_in, int kh, int kw, cudaStream_t s);
// ConvTranspose2d(4, 2, 1) weight [Ci, Co, 4, 4] (strided) -> phase-packed KRSC filter [4 * Co, 3, 3, Ci]
void convT_pack(const float* w, float* out, int Ci, int Co, long long s_ci, long long s_co, long long s_r, long long s_s, cudaStream_t s);

// ---- losses (loss_kernels.cu) --------------------------------------------------------------------
void cross_entropy_fwd(const float* logits, const long long* labels, float* loss, float* probs, int B, int C,
                       cudaStream_t s);
void cross_entropy_bwd(const float* probs, const long long* labels, const float* gout, float* dlogits, int B, int C,
                       cudaStream_t s);
void vae_loss_fwd(const float* recon, const float* x, int n, const float* mu, const float* logvar, int nl, float* out,
                  cudaStream_t s);
void vae_loss_bwd(const float* recon, const float* x, int n, const float* mu, const float* logvar, int nl,
                  const float* gout, float* drecon, float* dmu, float* dlogvar, cudaStream_t s);

// ---- small / awkward operators in true fp32 (aux_kernels.cu) ---------------------------------------
void gemm_f32(const float* a, const float* b, const float* bias, float* c, int M, int N, int K, long long sa_i, long long sa_k,
              long long sb_k, long long sb_j, int ldc, int act, int accumulate, cudaStream_t s);
void act_bwd_bias(const float* dout, const float* out, float* dz, float* db, long long total, int C, int act, cudaStream_t s);
void maxpool2x2_fwd(const float* x, float* y, unsigned char* idx, int N, int C, int H, int W, int nhwc, cudaStream_t s);
void maxpool2x2_bwd(const float* dy, const unsigned char* idx, float* dx, int N, int C, int H, int W, int nhwc, cudaStream_t s);
void argmax_count(const float* logits, const long long* labels, long long* counter, int B, int C, cudaStream_t s);
int info_nce_max_p();
int info_nce_scratch_floats();
void info_nce_fwd(const float* Z, const float* Zh, int R, int P, float* scratch, float* loss, float* coef, cudaStream_t s);
void info_nce_bwd(const float* Z, const float* Zh, const float* coef, const float* gout, float* dZ, float* dZh, int R, int P,
                  cudaStream_t s);
void gauss_nll_rows_fwd(const float* x, const float* mu, const float* s2, float* rows, int nrows, int B, int D, cudaStream_t s);
void gauss_nll_rows_bwd(const float* x, const float* mu, const float* s2, const float* grow, float* dmu, float* ds2, int nrows,
                        int B, int D, cudaStream_t s);
bool smallconv_supported(int Ci, int Co, int k);
void smallconv_fwd(const float* x, const float* w, const float* bias, float* y, unsigned char* pidx, int NB, int Ci, int H, int W,
                   int Co, int k, int pad, int act, int pool, cudaStream_t s);
void smallconv_dgrad(const float* dz, const float* w, float* dx, int NB, int Ci, int H, int W, int Co, int k, int pad, cudaStream_t s);
void smallconv_wgrad(const float* dz, const float* x, float* dw, float* db, int NB, int Ci, int H, int W, int Co, int k, int pad,
                     cudaStream_t s);
void smallconv_unpool_actbwd(const float* dy, const float* yout, const unsigned char* pidx, float* dz, long long planes, int Ho, int Wo,
                             int act, int pool, cudaStream_t s);

// ---- fused block collectives (comm_kernels.cu) -------------------------------------------------------
constexpr int COMM_MAX_K = 64;       // contributions (workers) per aggregation
constexpr int COMM_MAX_LOCAL = 16;   // replicas hosted by one process
constexpr int COMM_MAX_WORLD = 16;   // processes meeting through peer memory
constexpr int COMM_THREADS = 512;
constexpr int COMM_MAX_BLOCKS = 160; // CTAs per aggregation kernel (one per SM: 132 on an H100 SXM)

// Control pad (uint32 words; one pad per rank, mapped into every peer).  Flags hold the epoch of the aggregation that
// last signalled them (monotonic, compared with >=), so nothing is ever reset.
constexpr int PAD_FLAG_A = 0;                                                 // [COMM_MAX_BLOCKS][COMM_MAX_WORLD]  per-CTA: inputs final
constexpr int PAD_FLAG_B = PAD_FLAG_A + COMM_MAX_BLOCKS * COMM_MAX_WORLD;     // [COMM_MAX_BLOCKS][COMM_MAX_WORLD]  per-CTA: reads / broadcasts done
constexpr int PAD_FLAG_C = PAD_FLAG_B + COMM_MAX_BLOCKS * COMM_MAX_WORLD;     // [COMM_MAX_WORLD]  scalars posted
constexpr int PAD_FLAG_D = PAD_FLAG_C + COMM_MAX_WORLD;                       // [COMM_MAX_WORLD]  Barzilai-Borwein rows posted
constexpr int PAD_PAYLOAD = PAD_FLAG_D + COMM_MAX_WORLD;                      // [COMM_MAX_WORLD][4] floats: dual^2 part, primal part, #non-finite
constexpr int PAD_BBROWS = PAD_PAYLOAD + 4 * COMM_MAX_WORLD;                  // [COMM_MAX_K][8] floats: six dots per worker
constexpr int COMM_PAD_WORDS = 8192;
static_assert(PAD_BBROWS + 8 * COMM_MAX_K <= COMM_PAD_WORDS, "control pad too small");

// out record of an aggregation (floats): what the host reads back, once per round
constexpr int OUT_DUAL_SQ = 0, OUT_PRIMAL = 1, OUT_NONFINITE = 2, OUT_STATUS = 3, OUT_RHO = 4, OUT_EPOCH = 5, OUT_TWO_SHOT = 6;
constexpr int COMM_OUT_FLOATS = 8;
// device scratch (floats): [0] dual^2, [1] #non-finite, [2] ticket (as uint), [4 + j] per-replica primal^2; self-cleaning
constexpr int COMM_SCRATCH_FLOATS = 4 + COMM_MAX_LOCAL;

struct CommArgs {
  int mode;                          // 0 FedAvg, 1 FedProx, 2 ADMM
  int K, n_local, world, rank;
  int n;                             // floats in the block slice
  int two_shot;                      // 1: rank r reduces slice r of the vector and broadcasts it (n_local == 1, world > 1)
  int max_blocks;                    // grid cap (0 = one CTA per SM)
  float rho;                         // penalty when rho_dev == nullptr
  const float* rho_dev;              // device-resident penalty (adaptive ADMM): read by the kernel, never by the host
  const float* x[COMM_MAX_K];        // x_k slices of ALL workers (local or peer-mapped pointers)
  const float* y[COMM_MAX_K];        // y_k slices (ADMM) or nullptr
  float* xl[COMM_MAX_LOCAL];         // this process' replicas (writable aliases of the matching x[...])
  float* yl[COMM_MAX_LOCAL];
  float* xw[COMM_MAX_WORLD];         // two-shot FedAvg: rank p's x slice (broadcast target over P2P)
  float* zw[COMM_MAX_WORLD];         // two-shot FedProx / ADMM: rank p's z slice
  float* mc_x;                       // multicast address of the x slice (NVLS: multimem.ld_reduce / multimem.st) or nullptr
  float* mc_y;
  float* mc_z;
  float* z;                          // local copy of the consensus vector (in/out)
  float* out;                        // [COMM_OUT_FLOATS] result record
  float* scratch;                    // [COMM_SCRATCH_FLOATS] device accumulators (zero between launches)
  uint32_t* ctrl[COMM_MAX_WORLD];    // control pads of every rank (peer-mapped), COMM_PAD_WORDS words each
  uint32_t* sync;                    // local: [0] = epoch of the last completed collective
  long long timeout_cycles;          // per barrier; a timeout sets out[OUT_STATUS] = 100 + missing rank and lets the kernel end
};
void block_reduce_launch(const CommArgs& args, cudaStream_t s);

// Barzilai-Borwein / spectral penalty update of consensus ADMM as ONE kernel (SURVEY G20, X4): six dots per worker
// straight from (x, y, yhat0, x0, z), rows exchanged through the control pads, the reference's sequential
// accept/reject rule replayed identically on every rank, rho written to device memory, yhat0 / x0 carried forward.
struct BBArgs {
  int K, n_local, world, rank, n;
  int seed_only;                     // 1: x0 <- x only (round 0)
  int max_blocks;
  float epsilon, alphacorrmin, rhomax;
  const float* x[COMM_MAX_LOCAL];
  const float* y[COMM_MAX_LOCAL];
  float* yhat0[COMM_MAX_LOCAL];
  float* x0[COMM_MAX_LOCAL];
  int worker[COMM_MAX_LOCAL];        // global worker id of local replica j
  const float* z;
  float* rho_dev;                    // in/out: the shared penalty of this block
  float* log;                        // [K][8]: d11, d12, d22, alpha, alphaSD, alphaMG, tested(0/1), rho after this worker's turn
  float* scratch;                    // [8 * COMM_MAX_LOCAL + 8] zero between launches: dots + ticket + rho_turn
  uint32_t* ctrl[COMM_MAX_WORLD];
  uint32_t* sync;
  float* out;                        // status goes to out[OUT_STATUS]
  long long timeout_cycles;
};
constexpr int BB_SCRATCH_FLOATS = 8 * COMM_MAX_LOCAL + 8 + COMM_MAX_LOCAL;
void bb_update_launch(const BBArgs& args, cudaStream_t s);

}  // namespace fedb200

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
// Tile orientation of the convolution kernel: ROW = 128 pixels x BLOCK_N channels (igemm_wgmma_kernel), PIXEL = 64 / 128
// channels x 256 pixels (igemm_wgmma_pix_kernel, C_out 64 or 128); AUTO = the choice of pick_conv_orientation.  PIXEL runs
// the window-reuse main loop where conv_window_reuse allows it and the per-tap loop elsewhere; PIXEL_PERTAP always runs the
// per-tap loop (A/B tests and benchmarks).
enum { CONV_ORIENT_AUTO = -1, CONV_ORIENT_ROW = 0, CONV_ORIENT_PIXEL = 1, CONV_ORIENT_PIXEL_PERTAP = 2 };
// The orientation conv2d_nhwc_tf32 uses by itself for this shape (stride-1/2, no split-K).
int pick_conv_orientation(int NB, int H_out, int W_out, int C_out, int stride);
// Whether a pixel-major convolution of this shape runs the window-reuse main loop (one input box per filter column serves
// all kh filter rows).
bool conv_window_reuse(int H_out, int W_out, int C_in, int C_out, int kh, int stride, int dil);
void conv2d_nhwc_tf32(const float* x, const float* w, float* y, float* stats, int NB, int H, int W, int C_in, int C_out,
                      int kh, int kw, int stride, int pad, int dil, int H_out, int W_out, cudaStream_t stream,
                      int orient = CONV_ORIENT_AUTO);
// same kernel with bias + optional ELU in the epilogue (no statistics, no split-K): VAE / CPC convolutions
void conv2d_nhwc_bias_act_tf32(const float* x, const float* w, const float* bias, int act, float* y, int NB, int H, int W,
                               int C_in, int C_out, int kh, int kw, int stride, int pad, int dil, int H_out, int W_out,
                               cudaStream_t stream);
// y = act(BN_eval(conv(x, w)) + residual) with BatchNorm on its running statistics (inference); residual: [NB*H_out*W_out, C_out]
// or nullptr.  One launch without split-K, else the split-K convolution + an in-place bn_elu_fwd (running-statistics mode).
void conv2d_nhwc_bn_eval_tf32(const float* x, const float* w, const float* gamma, const float* beta, const float* mean,
                              const float* var, float eps, const float* residual, int act, float* y, int NB, int H, int W,
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

// ---- ResNet stem: 3 -> 64 channels, 3 x 3, stride 1, padding 1, + training-mode BatchNorm + ELU (stem_kernels.cu) ----------
// STORE_Y: y [N,H,32,64] and its batch statistics added into stats [sum 64 | sumsq 64 | counter]; STATS_ONLY: the statistics
// alone; APPLY: out = act(BN(conv(x))) from the complete statistics, save_mean / save_invstd, the running-statistics update
// (running_mean may be nullptr) and, with self_clean, the reset of stats and its counter, as bn_elu_fwd does.
enum { STEM_STORE_Y = 0, STEM_STATS_ONLY = 1, STEM_APPLY = 2 };
bool stem_conv_supported(int H, int W, int C_in, int C_out);
void stem_conv_bn(int mode, const float* x, const float* w, float* out, float* stats, const float* gamma, const float* beta,
                  float* running_mean, float* running_var, float* save_mean, float* save_invstd, int NB, int H, float eps,
                  float momentum, int act, int self_clean, cudaStream_t stream);


// ---- flat-vector kernels (flat_kernels.cu) ---------------------------------------------------------
void adam_prox(float* x, const float* g, float* m, float* v, const int* step_dev, int n, float lr, float b1, float b2,
               float eps, const float* z, const float* y, float rho, float l1, float l2, cudaStream_t s,
               const float* rho_dev = nullptr, const float* lr_dev = nullptr, float weight_decay = 0.f,
               const float* norm_dev = nullptr, float clip = 0.f);
// buf == nullptr: no momentum (momentum must then be 0)
void sgd_prox(float* x, const float* g, float* buf, int n, float lr, float momentum, bool nesterov, float weight_decay,
              const float* z, const float* y, float rho, float l1, float l2, cudaStream_t s, const float* rho_dev,
              const float* lr_dev = nullptr, const float* norm_dev = nullptr, float clip = 0.f);
// gradient norm for clipping: ws = [norm, sum of norms, clipped steps, steps, partials[grad_norm_blocks(n)]]
constexpr int kGradNormHeader = 4;
int grad_norm_blocks(int n);
void grad_norm(const float* g, int n, float* ws, unsigned int* ticket, float clip, cudaStream_t s);
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
// at most kTwoLoopMaxHist pairs (the kernel keeps the row indices in shared memory); longer histories take the ATen path
constexpr int kTwoLoopMaxHist = 32;
void lbfgs_two_loop(const float* Y, const float* S, const int* order, int k, int n, int ld, const float* g, float hdiag,
                    float* d, float* work, cudaStream_t s);
size_t lbfgs_two_loop_work_floats(int k);

// ---- elementwise / normalisation (elementwise_kernels.cu) ------------------------------------------
void normalize_u8_nhwc(const uint8_t* in, float* out, int npix, int c_out, const float* mean3, const float* std3,
                       int to_nchw, int H, int W, cudaStream_t s);
// n samples of training augmentation (random 4-pixel-padded crop + horizontal flip) + normalisation, NCHW or NHWC (3
// channels) out.  rows: int64 indices of the samples in `in` (device-resident dataset), or nullptr when `in` already holds
// the n samples.  Sample i draws from (key, counter + i); the draw is documented in data/cifar.py (augment_draws).
void augment_normalize_u8(const uint8_t* in, const int64_t* rows, float* out, int n, int H, int W, uint64_t key,
                          uint64_t counter, const float* mean3, const float* std3, int to_nchw, cudaStream_t s);
// n samples mixed with their partners n-1-i (mixup: lam_f a + mlam_f b; cutmix: the partner's pixels inside
// [y0, y1) x [x0, x1)), after the optional augmentation (augment != 0, drawn from (key, counter + i)) and normalisation,
// NCHW or NHWC (3 channels) out; lam_out[0] = lam_eff.  rows as for augment_normalize_u8.  The draw is made on the host
// (data/cifar.py: mix_draws).
void mix_normalize_u8(const uint8_t* in, const int64_t* rows, float* out, float* lam_out, int n, int H, int W, int augment,
                      uint64_t key, uint64_t counter, const float* mean3, const float* std3, int to_nchw, int cutmix,
                      float lam_f, float mlam_f, int y0, int y1, int x0, int x1, float lam_eff, cudaStream_t s);
void col_stats(const float* y, float* stats, int M, int C, cudaStream_t s);
// stats: [2C] sums (+ one uint counter behind them when self_clean: the kernel zeroes the buffer after the last read)
// use_running: eval-mode BatchNorm on running_mean / running_var (read only); stats, save_mean / save_invstd, momentum and
// self_clean are unused, and out may equal y
void bn_elu_fwd(const float* y, float* stats, const float* gamma, const float* beta, const float* residual,
                float* out, float* running_mean, float* running_var, float* save_mean, float* save_invstd, int M, int C,
                float eps, float momentum, int act, int self_clean, cudaStream_t s, int use_running = 0);
// out == nullptr (allowed when the layer had no residual input): ELU' is recomputed from y, gamma, beta
void bn_elu_bwd_reduce(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                       const float* gamma, const float* beta, float* sums, int M, int C, int act, int sums_clean, cudaStream_t s);
void bn_elu_bwd_apply(const float* dout, const float* out, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, float* sums, float* dy, float* dres, float* dgamma,
                      float* dbeta, int M, int C, int act, int self_clean, cudaStream_t s);

// ---- GroupNorm + residual + ELU (norm_kernels.cu) ----------------------------------------------------
// y, residual, out: [N, HW, C] (NHWC); mean / rstd: [N, G].  Scratch: part [N, S, 2, C] with S = gn_splits(N, HW, C),
// table [N, 2, C] (scale | shift), ab [2, N, G].  Needs C % 4 == 0, C <= 1024, G | C, G <= 256.
int gn_splits(int N, int HW, int C);
void gn_elu_fwd(const float* y, const float* gamma, const float* beta, const float* residual, float* out, float* mean,
                float* rstd, float* part, float* table, int N, int HW, int C, int G, float eps, int act, cudaStream_t s);
// out == nullptr (allowed when the layer had no residual input): ELU' is recomputed from y, gamma, beta.  dres, dgamma,
// dbeta may be nullptr; dgamma / dbeta are overwritten, not accumulated.
void gn_elu_bwd(const float* dout, const float* out, const float* y, const float* mean, const float* rstd, const float* gamma,
                const float* beta, float* part, float* ab, float* dy, float* dres, float* dgamma, float* dbeta, int N, int HW,
                int C, int G, int act, cudaStream_t s);
// fused classifier head: avg-pool over HW + Linear (true fp32), O <= 32 outputs
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
// soft-target cross-entropy: targets lam s(y_i) + (1 - lam) s(y_{B-1-i}), s(y) = (1 - eps) onehot(y) + eps / C; lam is a
// device scalar (nullptr = 1).  The mean loss is summed in a fixed order (no atomics); dlogits = (p - q) gout / B.
void soft_ce_fwd(const float* logits, const long long* labels, const float* lam, float eps, float* loss, float* probs, int B,
                 int C, cudaStream_t s);
void soft_ce_bwd(const float* probs, const long long* labels, const float* lam, float eps, const float* gout, float* dlogits,
                 int B, int C, cudaStream_t s);
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
// Every kind of round posts its statistics into the same PAD_PAYLOAD row (FedProx / ADMM: dual^2 part, primal part,
// #non-finite; DP: #clipped, sum of norms; compressed: quantization statistics; SecAgg: clipped / non-finite counts).  A
// rank posts into a peer's row again only in a later round, after passing that round's barrier A with the peer; the
// peer's kernel for that round started only after its kernel that read the row had finished (launches on a stream run in
// order), so a round never overwrites words a peer has yet to read, whatever kind either round is.
constexpr int PAD_FLAG_A = 0;                                                 // [COMM_MAX_BLOCKS][COMM_MAX_WORLD]  per-CTA: inputs final
constexpr int PAD_FLAG_B = PAD_FLAG_A + COMM_MAX_BLOCKS * COMM_MAX_WORLD;     // [COMM_MAX_BLOCKS][COMM_MAX_WORLD]  per-CTA: reads / broadcasts done
constexpr int PAD_FLAG_C = PAD_FLAG_B + COMM_MAX_BLOCKS * COMM_MAX_WORLD;     // [COMM_MAX_WORLD]  statistics posted
constexpr int PAD_FLAG_D = PAD_FLAG_C + COMM_MAX_WORLD;                       // [COMM_MAX_WORLD]  Barzilai-Borwein rows posted
constexpr int PAD_PAYLOAD = PAD_FLAG_D + COMM_MAX_WORLD;                      // [COMM_MAX_WORLD][4] words: a round's statistics
constexpr int PAD_BBROWS = PAD_PAYLOAD + 4 * COMM_MAX_WORLD;                  // [COMM_MAX_K][8] floats: six dots per worker
constexpr int COMM_PAD_WORDS = 8192;
static_assert(PAD_BBROWS + 8 * COMM_MAX_K <= COMM_PAD_WORDS, "control pad too small");

// out record of an aggregation (floats): what the host reads back, once per round.  DP rounds add the number of clipped
// workers and the sum of their pre-clip update norms, over all K; compressed rounds the sums over all K of
// ||u_k - q_k s_k||^2 and ||u_k||^2.
constexpr int OUT_DUAL_SQ = 0, OUT_PRIMAL = 1, OUT_NONFINITE = 2, OUT_STATUS = 3, OUT_RHO = 4, OUT_EPOCH = 5, OUT_TWO_SHOT = 6;
constexpr int OUT_DP_CLIPPED = 8, OUT_DP_NORM_SUM = 9;
constexpr int OUT_Q_ERR_SQ = 10, OUT_Q_NORM_SQ = 11;
// secure-aggregation rounds: the number of clipped and of non-finite coordinates over all K, as uint32 bit patterns
// (integers: float counts stop being exact above 2^24)
constexpr int OUT_SA_CLIPPED = 12, OUT_SA_NONFINITE = 13;
constexpr int COMM_OUT_FLOATS = 14;
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
  // ---- server optimizer (FedOpt instantiation only; mode must be 0): d = mean - z is a pseudo-gradient, the step replaces
  // the plain mean as the new model.  m / v persist across rounds in device memory.
  int opt;                           // FEDOPT_NONE selects the FedAvg / FedProx / ADMM kernel
  float lr, beta1, beta2, tau;       // avgm: beta1 is the momentum
  float* m;                          // local server state slices: momentum / first moment, second moment (adaptive only)
  float* v;
  float* mw[COMM_MAX_WORLD];         // two-shot: rank p's m / v slice (broadcast targets over P2P)
  float* vw[COMM_MAX_WORLD];
  float* mc_m;                       // multicast addresses of the m / v slices (multimem.st) or nullptr
  float* mc_v;
  // ---- robust aggregation (modes 0 / 1, with or without a server optimizer): a per-coordinate order statistic over the
  // K workers replaces the mean.  Computed in registers, so K <= COMM_MAX_K_ROBUST; peers are read over P2P even when a
  // multicast object is bound (no in-switch order statistics).
  int agg;                           // AGG_MEAN selects the instantiations above
  int trim_b;                        // AGG_TRIMMED: values dropped at each end (0 <= 2 trim_b < K)
  // ---- client-level differential privacy (DP-FedAvg, McMahan et al. 2018; mode 0 with the mean, with or without a server
  // optimizer): the replicas were clipped by dp_clip_kernel; the Gaussian noise dp_std * xi(key, t, i) is added to the mean.
  int dp;                            // 0 selects the instantiations above
  float dp_std;                      // noise std of the mean: sigma C / K
  unsigned long long dp_key;         // key of the run's noise stream
  long long* dp_t;                   // device: index t of this DP round over the run; the last CTA increments it
  const float* dp_stats;             // dp_clip_kernel's [DP_NORM ..) record: per-replica norms, then clipped flags
  // per DP_CHUNK-float chunk of the slice, how many of its leading floats are parameters (the rest is the arena's
  // alignment padding, which gets no noise and stays zero); nullptr: every float is a parameter
  const unsigned char* dp_valid;
  // ---- compressed client updates (QSGD / FedPAQ, mode 0 with the mean, with or without a server optimizer): before barrier
  // A every rank quantizes its local replicas' updates u_k = x_k - z (+ e_k) into payload arenas — one scale per Q_GROUP
  // coordinates, stochastically rounded qbits-bit codes — and pass 1 reads the K workers' payloads instead of their floats.
  int qbits;                         // 0 selects the instantiations above; 8 or 4
  unsigned long long q_key;          // key of the run's rounding stream
  long long* q_t;                    // device: index t of this compressed round over the run; the last CTA increments it
  int q_worker[COMM_MAX_LOCAL];      // global worker id k of local replica j (keys the rounding draw)
  unsigned char* q_codes[COMM_MAX_K];   // codes of ALL workers (local or peer-mapped): one byte per coordinate (8-bit)
                                        // or two codes per byte, the even coordinate in the low nibble (4-bit)
  float* q_scales[COMM_MAX_K];       // one scale per group of Q_GROUP coordinates, counted from the block start
  float* q_ef[COMM_MAX_LOCAL];       // error feedback e_j of local replica j (in/out), or nullptr (off)
  float* q_part;                     // [Q_PART_FLOATS] per-CTA partial statistics (each launch overwrites what it reads)
  // ---- client sampling with sample-count weights (FedAvg partial participation, McMahan et al. 2017; mode 0 with the
  // mean, with or without a server optimizer, without DP or compression): round t = *samp_t takes the samp_S workers with
  // the smallest (h_k, k), h_k = F(F(samp_key + (t + 1) G) + (k + 1) G), and z = sum_{k in P} w_k x_k with
  // w_k = n_k / sum_{j in P} n_j.  Only participants are read (over P2P); every replica receives z.
  int samp_S;                        // 0 selects the instantiations above; else 1..K participants per round
  unsigned long long samp_key;       // key of the run's sampling stream
  long long* samp_t;                 // device: index t of this sampled round over the run; the last CTA increments it
  const int* client_n;               // device: [K] sample counts n_k of the workers' shards
  // ---- secure aggregation (SecAgg, Bonawitz et al. 2017; mode 0 with the mean, with or without a server optimizer,
  // without DP, compression or sampling): before barrier A every rank encodes its local replicas' updates u = x_k - z as
  // int32 fixed-point codes q = rint(clamp(u, -R, R) 2^f) and uploads y_k = q_k + sum_{j>k} m_kj - sum_{j<k} m_jk
  // (mod 2^32), m_ij the ChaCha20 keystream of pair key ij under nonce t.  The masks cancel in the sum, so pass 1 decodes
  // z' = z + (float(sum_k y_k) 2^-f) / K exactly.  The rounds use the compressed rounds' q_codes (as 4-byte words, one
  // per coordinate), q_t (the nonce t), q_worker and q_part (per-CTA integer counts).
  int sa;                            // 0 selects the instantiations above
  int sa_frac_bits;                  // f: K rint(R 2^f) <= 2^31 - 1, 0 <= f <= 126
  float sa_clip;                     // R
  const uint32_t* sa_keys;           // device: [K (K - 1) / 2][8] pair keys, pairs (i < j) in lexicographic order
  // ---- top-k sparsified updates (mode 0 with the mean, with or without a server optimizer, without DP, compression,
  // sampling or SecAgg): topk_select_kernel has written every local worker's sparse payload (layout: TopKLayout) and its
  // statistics (q_part[0], q_part[1]); pass 1 scatter-adds the K workers' entries tile by tile into shared memory, in
  // worker order.  The payload pointers of ALL K workers go in q_codes.
  int topk_k;                        // 0 selects the instantiations above; else k_sel entries per worker
};
constexpr int Q_GROUP = 128;                             // coordinates per scale
constexpr int Q_SEG = 16;                                // coordinates per thread and tile in the compressed instantiations
constexpr int Q_PART_FLOATS = 2 * COMM_MAX_BLOCKS;
constexpr int DP_CHUNK = 32;
constexpr int FEDOPT_NONE = 0, FEDOPT_AVGM = 1, FEDOPT_ADAGRAD = 2, FEDOPT_ADAM = 3, FEDOPT_YOGI = 4;
constexpr int AGG_MEAN = 0, AGG_MEDIAN = 1, AGG_TRIMMED = 2;
constexpr int COMM_MAX_K_ROBUST = 16;
constexpr int SA_MAX_FRAC_BITS = 126;                   // 2^f and 2^-f stay normal floats
// block_reduce_launch picks the instantiation: the mean, a robust rule, DP, compressed codes (qbits), client sampling
// (samp_S), secure aggregation (sa) or top-k payloads (topk_k); it rejects combinations the kernel does not implement.
void block_reduce_launch(const CommArgs& args, cudaStream_t s);

// ---- top-k sparse payload of one worker and block (int32 words; algo/compress.py: topk_select is the oracle) ----------
// words [0, T]: uint32 tile offsets (T = ceil(n / TOPK_TILE) tiles from the block start; offset T = k), then from word
// val the k float32 values, then from word idx the k uint16 in-tile offsets, two per word (the lower index in the low
// half).  Entries are in ascending coordinate order.  Sections start at 16-byte boundaries.
constexpr int TOPK_TILE = COMM_THREADS * Q_SEG;          // 8192 coordinates: one tile of the compressed tiling
struct TopKLayout {
  int tiles, val, idx, words;
};
__host__ __device__ inline TopKLayout topk_layout(int n, int k) {
  const int T = (n + TOPK_TILE - 1) / TOPK_TILE;
  const int val = (T + 1 + 3) & ~3;
  const int idx = val + ((k + 3) & ~3);
  return {T, val, idx, idx + (((k + 1) / 2 + 3) & ~3)};
}

// Top-k selection of the local replicas' updates as ONE cooperative kernel touching no peer memory.  Per replica j:
// u = (x_j - z) + e_j is materialised into e_j (error feedback) or u[j]; the k-th largest key bits(u) & 0x7fffffff is
// found by a 4-digit radix select (global integer histograms, grid.sync() between digits); each tile counts its keys above
// and equal to it, replica j's tile offsets are scanned by CTA j, and every tile writes its entries in index order by an
// in-CTA prefix scan (ties go to the lower index).  With error feedback e_j <- u - s_j.  q_part[0] / q_part[1] receive
// sum_j ||u_j - s_j||^2 and sum_j ||u_j||^2, summed in a fixed order: the same bits on every run.
struct TopKArgs {
  int n, n_local, k, max_blocks;
  const float* x[COMM_MAX_LOCAL];    // this process' replicas
  const float* z;                    // the server model the round started from
  float* ef[COMM_MAX_LOCAL];         // error feedback e_j (in / out), or nullptr (off: u goes to u[j])
  float* u[COMM_MAX_LOCAL];          // scratch for u_j when error feedback is off
  uint32_t* pay[COMM_MAX_LOCAL];     // the replicas' payloads (TopKLayout)
  int* ws;                           // [topk_ws_ints(n, n_local)] workspace; its histograms are zero between launches
  float* stats;                      // [TOPK_STATS_FLOATS] (the aggregation's q_part): [0] err, [1] norm, per-CTA partials
};
constexpr int TOPK_RADIX = 256;
constexpr int TOPK_STATS_FLOATS = 2 + 2 * COMM_MAX_BLOCKS;
inline int topk_ws_ints(int n, int n_local) {
  return 4 * COMM_MAX_LOCAL * TOPK_RADIX + 3 * n_local * ((n + TOPK_TILE - 1) / TOPK_TILE);
}
void topk_select_launch(const TopKArgs& args, cudaStream_t s);

// DP-FedAvg update clipping on the local replicas, as ONE cooperative kernel touching no peer memory: ||x_j - z|| per
// replica, grid.sync(), then x_j <- z + (C / ||x_j - z||) (x_j - z) for the replicas over the bound C only (the others are
// not written).  Norms and clipped flags go to the stats record, which the DP aggregation kernel that follows reads.
struct DPClipArgs {
  int n, n_local, max_blocks;
  float bound;                       // C
  float* x[COMM_MAX_LOCAL];          // this process' replicas
  const float* z;                    // the server model the round started from
  float* stats;                      // [DP_STATS_FLOATS]
};
// stats record (floats): per-CTA partial sums of squares as doubles [COMM_MAX_LOCAL][COMM_MAX_BLOCKS] (2 floats each),
// then per replica the pre-clip norm [COMM_MAX_LOCAL] and the clipped flag (0 / 1) [COMM_MAX_LOCAL].  Every launch
// overwrites what it reads: no cleaning.
constexpr int DP_PART = 0;
constexpr int DP_NORM = 2 * COMM_MAX_LOCAL * COMM_MAX_BLOCKS;
constexpr int DP_CLIPPED = DP_NORM + COMM_MAX_LOCAL;
constexpr int DP_STATS_FLOATS = DP_CLIPPED + COMM_MAX_LOCAL;
void dp_clip_launch(const DPClipArgs& args, cudaStream_t s);

// SCAFFOLD control variates (flat_kernels.cu), one launch per step for all local replicas j (blockIdx.y = j):
//  * scaffold_cv:   c_j <- (c_j - c) + s_j (z - x_j) for the replicas with s_j != 0 (s_j = 0: sat out, not written);
//  * scaffold_corr: d_j <- c - c_j for every replica, and norm_sq[j] = ||d_j||^2 summed in a fixed order (per-CTA partials
//    in ws[j * scaffold_corr_blocks(n) + cta], the last CTA of replica j, by its ticket, sums them in CTA order and
//    resets the ticket).  No floating-point atomics: the same bits on every run.
struct ScaffoldArgs {
  int n, n_local;
  float* ci[COMM_MAX_LOCAL];         // c_j (cv: in/out; corr: in)
  const float* x[COMM_MAX_LOCAL];    // cv: x_j after the round's local steps
  float* d[COMM_MAX_LOCAL];          // corr: the correction d_j (out)
  float scale[COMM_MAX_LOCAL];       // cv: s_j = 1 / (tau_j lr), 0 = sat out
  const float* c;                    // the server control variate
  const float* z;                    // cv: the server model the round started from
  float* ws;                         // corr: [n_local * scaffold_corr_blocks(n)] partials
  unsigned int* tickets;             // corr: [n_local], zero between launches
  float* norm_sq;                    // corr: [n_local]
};
int scaffold_corr_blocks(int n);
void scaffold_cv_launch(const ScaffoldArgs& args, cudaStream_t s);
void scaffold_corr_launch(const ScaffoldArgs& args, cudaStream_t s);

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
  float* scratch;                    // [BB_SCRATCH_FLOATS] zero between launches: dots, 8 unused words, rho_turn
  uint32_t* ctrl[COMM_MAX_WORLD];
  uint32_t* sync;
  float* out;                        // status goes to out[OUT_STATUS]
  long long timeout_cycles;
};
constexpr int BB_SCRATCH_FLOATS = 8 * COMM_MAX_LOCAL + 8 + COMM_MAX_LOCAL;
void bb_update_launch(const BBArgs& args, cudaStream_t s);

}  // namespace fedb200

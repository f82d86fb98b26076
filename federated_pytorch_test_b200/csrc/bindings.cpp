// Torch glue for the sm_90a kernels: tensor checks, stream selection, pybind.  All math lives in the .cu files.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cstdlib>

#include "fedb200.h"

namespace fb = fedb200;
using torch::Tensor;

static cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
static const float* fptr(const Tensor& t) { return t.data_ptr<float>(); }
static float* fptr_mut(Tensor& t) { return t.data_ptr<float>(); }
static const float* opt_ptr(const c10::optional<Tensor>& t) { return (t.has_value() && t->defined()) ? t->data_ptr<float>() : nullptr; }

#define CHECK_F32_CUDA(x) TORCH_CHECK((x).is_cuda() && (x).scalar_type() == torch::kFloat32, #x " must be a CUDA float32 tensor")
#define CHECK_CONTIG(x) TORCH_CHECK((x).is_contiguous(), #x " must be contiguous")

// ---------------------------------------------------------------------------------------------- flat ops
void adam_prox(Tensor x, Tensor g, Tensor m, Tensor v, Tensor step, double lr, double b1, double b2, double eps,
               c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2,
               c10::optional<Tensor> rho_dev, c10::optional<Tensor> lr_dev, double weight_decay,
               c10::optional<Tensor> norm_dev, double clip) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_CONTIG(g); CHECK_CONTIG(m); CHECK_CONTIG(v);
  c10::cuda::CUDAGuard guard(x.device());
  fb::adam_prox(fptr_mut(x), fptr(g), fptr_mut(m), fptr_mut(v), step.data_ptr<int>(), (int)x.numel(), (float)lr, (float)b1,
                (float)b2, (float)eps, opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, cur_stream(), opt_ptr(rho_dev),
                opt_ptr(lr_dev), (float)weight_decay, opt_ptr(norm_dev), (float)clip);
}
void sgd_prox(Tensor x, Tensor g, c10::optional<Tensor> buf, double lr, double momentum, bool nesterov, double weight_decay,
              c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2,
              c10::optional<Tensor> rho_dev, c10::optional<Tensor> lr_dev, c10::optional<Tensor> norm_dev, double clip) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_CONTIG(g);
  const bool has_buf = buf.has_value() && buf->defined();
  TORCH_CHECK(has_buf == (momentum != 0.0), "sgd_prox: a momentum buffer is passed exactly when momentum != 0");
  if (has_buf) { CHECK_CONTIG(*buf); TORCH_CHECK(buf->numel() == x.numel(), "sgd_prox: buf must have x's length"); }
  c10::cuda::CUDAGuard guard(x.device());
  fb::sgd_prox(fptr_mut(x), fptr(g), has_buf ? buf->data_ptr<float>() : nullptr, (int)x.numel(), (float)lr, (float)momentum,
               nesterov, (float)weight_decay, opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, cur_stream(),
               opt_ptr(rho_dev), opt_ptr(lr_dev), opt_ptr(norm_dev), (float)clip);
}
int64_t grad_norm_blocks(int64_t n) { return fb::grad_norm_blocks((int)n); }
void grad_norm(Tensor g, Tensor ws, Tensor ticket, double clip) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_F32_CUDA(ws); CHECK_CONTIG(ws);
  TORCH_CHECK(ticket.is_cuda() && ticket.scalar_type() == torch::kInt32 && ticket.numel() == 1,
              "grad_norm: ticket must be one CUDA int32");
  TORCH_CHECK(ws.numel() >= fb::kGradNormHeader + fb::grad_norm_blocks((int)g.numel()),
              "grad_norm: ws needs ", fb::kGradNormHeader, " + grad_norm_blocks(n) floats");
  c10::cuda::CUDAGuard guard(g.device());
  fb::grad_norm(fptr(g), (int)g.numel(), fptr_mut(ws), reinterpret_cast<unsigned int*>(ticket.data_ptr<int>()), (float)clip,
                cur_stream());
}
void bump_step(Tensor step) {
  c10::cuda::CUDAGuard guard(step.device());
  fb::bump_step(step.data_ptr<int>(), cur_stream());
}
Tensor l1_l2(Tensor g) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g);
  c10::cuda::CUDAGuard guard(g.device());
  auto out = torch::empty({2}, g.options());
  fb::l1_l2(fptr(g), (int)g.numel(), fptr_mut(out), cur_stream());
  return out;
}
// x is read or written element for element alongside ref: the same dtype, device and length, contiguous.  The messages
// are string literals only: with the torch this extension is built against, a TORCH_CHECK message formatted from
// run-time values (c10::str) crashes the process instead of raising.
#define CHECK_LIKE(x, ref)                                                                                     \
  do {                                                                                                         \
    CHECK_F32_CUDA(x); CHECK_CONTIG(x);                                                                        \
    TORCH_CHECK((x).device() == (ref).device(), #x " must be on the device of " #ref);                        \
    TORCH_CHECK((x).numel() == (ref).numel(), #x " must have the length of " #ref);                           \
  } while (0)
#define CHECK_OPT_LIKE(x, ref)                                                                                 \
  do {                                                                                                         \
    if ((x).has_value() && (x)->defined()) CHECK_LIKE((*x), ref);                                              \
  } while (0)

std::vector<Tensor> make_pair(Tensor g, Tensor gprev, Tensor d, double t, double trust) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_LIKE(gprev, g); CHECK_LIKE(d, g);
  c10::cuda::CUDAGuard guard(g.device());
  auto y = torch::empty_like(g), s = torch::empty_like(g);
  auto out = torch::empty({3}, g.options());
  fb::make_pair(fptr(g), fptr(gprev), fptr(d), (float)t, (float)trust, fptr_mut(y), fptr_mut(s), (int)g.numel(), fptr_mut(out), cur_stream());
  return {y, s, out};
}
Tensor welford(Tensor g, Tensor mean, Tensor m2, int64_t n_iter) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_LIKE(mean, g); CHECK_LIKE(m2, g);
  TORCH_CHECK(n_iter >= 1, "welford: n_iter must be >= 1");
  c10::cuda::CUDAGuard guard(g.device());
  auto out = torch::empty({1}, g.options());
  fb::welford(fptr(g), fptr_mut(mean), fptr_mut(m2), (int)g.numel(), 1.0f / (float)n_iter, fptr_mut(out), cur_stream());
  return out;
}
Tensor penalty_value(Tensor x, c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x);
  CHECK_OPT_LIKE(z, x); CHECK_OPT_LIKE(y, x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty({1}, x.options());
  fb::penalty_value(fptr(x), opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, (int)x.numel(), fptr_mut(out), cur_stream());
  return out;
}
void penalty_grad(Tensor g, Tensor x, c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_LIKE(x, g);
  CHECK_OPT_LIKE(z, g); CHECK_OPT_LIKE(y, g);
  c10::cuda::CUDAGuard guard(g.device());
  fb::penalty_grad(fptr_mut(g), fptr(x), opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, (int)g.numel(), cur_stream());
}
Tensor multi_dot(std::vector<Tensor> a, std::vector<Tensor> b) {
  TORCH_CHECK(a.size() == b.size() && !a.empty() && a.size() <= 8, "multi_dot: 1..8 pairs");
  c10::cuda::CUDAGuard guard(a[0].device());
  std::vector<const float*> pa, pb;
  for (size_t i = 0; i < a.size(); ++i) {
    CHECK_F32_CUDA(a[i]); CHECK_CONTIG(a[i]); CHECK_F32_CUDA(b[i]); CHECK_CONTIG(b[i]);
    TORCH_CHECK(a[i].device() == a[0].device() && b[i].device() == a[0].device(), "multi_dot: all vectors on one device");
    TORCH_CHECK(a[i].numel() == a[0].numel() && b[i].numel() == a[0].numel(), "multi_dot: equal lengths required");
    pa.push_back(fptr(a[i])); pb.push_back(fptr(b[i]));
  }
  auto out = torch::empty({(int64_t)a.size()}, a[0].options());
  fb::multi_dot(pa.data(), pb.data(), (int)a.size(), (int)a[0].numel(), fptr_mut(out), cur_stream());
  return out;
}
// order: the rows of Y and S to use, oldest pair first.  It is checked here and copied to the device with the call.
Tensor lbfgs_two_loop(Tensor Y, Tensor S, std::vector<int64_t> order, Tensor g, double hdiag) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g);
  CHECK_F32_CUDA(Y); CHECK_CONTIG(Y); CHECK_F32_CUDA(S); CHECK_CONTIG(S);
  TORCH_CHECK(Y.dim() == 2 && S.sizes() == Y.sizes(), "lbfgs_two_loop: Y and S must be [m, n] of one shape");
  TORCH_CHECK(Y.device() == g.device() && S.device() == g.device(), "lbfgs_two_loop: Y, S and g on one device");
  TORCH_CHECK(Y.size(1) == g.numel(), "lbfgs_two_loop: the rows of Y must have the length of g");
  const int64_t m = Y.size(0);
  const int k = (int)order.size(), n = (int)g.numel();
  TORCH_CHECK(k >= 1 && k <= m && k <= fb::kTwoLoopMaxHist,
              "lbfgs_two_loop: 1 to min(rows of Y, kTwoLoopMaxHist = 32) pairs");
  for (int64_t r : order) TORCH_CHECK(r >= 0 && r < m, "lbfgs_two_loop: every order entry must be a row of Y");
  std::vector<int> rows(order.begin(), order.end());
  c10::cuda::CUDAGuard guard(g.device());
  auto dev_order = torch::tensor(rows, torch::kInt32).to(g.device());
  auto d = torch::empty_like(g);
  auto work = torch::empty({(int64_t)fb::lbfgs_two_loop_work_floats(k)}, g.options());
  fb::lbfgs_two_loop(fptr(Y), fptr(S), dev_order.data_ptr<int>(), k, n, (int)Y.size(1), fptr(g), (float)hdiag, fptr_mut(d),
                     fptr_mut(work), cur_stream());
  return d;
}

// ---------------------------------------------------------------------------------------------- elementwise
Tensor normalize_u8(Tensor u8, std::vector<double> mean, std::vector<double> stdv, int64_t c_out, bool to_nchw) {
  TORCH_CHECK(u8.is_cuda() && u8.scalar_type() == torch::kUInt8 && u8.dim() == 4 && u8.size(3) == 3 && u8.is_contiguous(),
              "normalize_u8 expects a contiguous CUDA uint8 [N,H,W,3] tensor");
  c10::cuda::CUDAGuard guard(u8.device());
  const int64_t N = u8.size(0), H = u8.size(1), W = u8.size(2);
  float m3[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s3[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(u8.device());
  Tensor out = to_nchw ? torch::empty({N, 3, H, W}, opts) : torch::empty({N, H, W, c_out}, opts);
  fb::normalize_u8_nhwc(u8.data_ptr<uint8_t>(), fptr_mut(out), (int)(N * H * W), (int)c_out, m3, s3, to_nchw ? 1 : 0, (int)H, (int)W, cur_stream());
  return out;
}
// key: the 64-bit augmentation key, bit pattern passed as int64.  rows: optional int64 indices into u8 (every index must be
// a valid row); without them u8 holds the batch itself.
Tensor augment_normalize_u8(Tensor u8, c10::optional<Tensor> rows, int64_t key, int64_t counter, std::vector<double> mean,
                            std::vector<double> stdv, bool to_nchw) {
  TORCH_CHECK(u8.is_cuda() && u8.scalar_type() == torch::kUInt8 && u8.dim() == 4 && u8.size(3) == 3 && u8.is_contiguous(),
              "augment_normalize_u8 expects a contiguous CUDA uint8 [N,H,W,3] tensor");
  TORCH_CHECK(counter >= 0, "augment_normalize_u8: negative counter");
  c10::cuda::CUDAGuard guard(u8.device());
  int64_t N = u8.size(0);
  const int64_t H = u8.size(1), W = u8.size(2);
  const int64_t* rp = nullptr;
  if (rows.has_value() && rows->defined()) {
    TORCH_CHECK(rows->is_cuda() && rows->device() == u8.device() && rows->scalar_type() == torch::kInt64 && rows->dim() == 1 &&
                    rows->is_contiguous(),
                "augment_normalize_u8: rows must be a contiguous int64 vector on the images' device");
    N = rows->numel();
    rp = rows->data_ptr<int64_t>();
  }
  TORCH_CHECK(N * H * W < (int64_t(1) << 31), "augment_normalize_u8: batch too large");
  float m3[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s3[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(u8.device());
  Tensor out = to_nchw ? torch::empty({N, 3, H, W}, opts) : torch::empty({N, H, W, 3}, opts);
  if (N == 0) return out;
  fb::augment_normalize_u8(u8.data_ptr<uint8_t>(), rp, fptr_mut(out), (int)N, (int)H, (int)W, (uint64_t)key, (uint64_t)counter,
                           m3, s3, to_nchw ? 1 : 0, cur_stream());
  return out;
}
// Mixup / CutMix input stage: returns {batch, lam} with lam a one-float32 tensor holding lam_eff.  key: the augmentation key
// (used with augment), rows as for augment_normalize_u8.  lam_f / mlam_f / lam_eff arrive as doubles holding float32 values.
std::vector<Tensor> mix_normalize_u8(Tensor u8, c10::optional<Tensor> rows, bool augment, int64_t key, int64_t counter,
                                     std::vector<double> mean, std::vector<double> stdv, bool to_nchw, bool cutmix,
                                     double lam_f, double mlam_f, int64_t y0, int64_t y1, int64_t x0, int64_t x1,
                                     double lam_eff) {
  TORCH_CHECK(u8.is_cuda() && u8.scalar_type() == torch::kUInt8 && u8.dim() == 4 && u8.size(3) == 3 && u8.is_contiguous(),
              "mix_normalize_u8 expects a contiguous CUDA uint8 [N,H,W,3] tensor");
  TORCH_CHECK(counter >= 0, "mix_normalize_u8: negative counter");
  c10::cuda::CUDAGuard guard(u8.device());
  int64_t N = u8.size(0);
  const int64_t H = u8.size(1), W = u8.size(2);
  TORCH_CHECK(0 <= y0 && y0 <= y1 && y1 <= H && 0 <= x0 && x0 <= x1 && x1 <= W, "mix_normalize_u8: box outside the image");
  const int64_t* rp = nullptr;
  if (rows.has_value() && rows->defined()) {
    TORCH_CHECK(rows->is_cuda() && rows->device() == u8.device() && rows->scalar_type() == torch::kInt64 && rows->dim() == 1 &&
                    rows->is_contiguous(),
                "mix_normalize_u8: rows must be a contiguous int64 vector on the images' device");
    N = rows->numel();
    rp = rows->data_ptr<int64_t>();
  }
  TORCH_CHECK(N * H * W < (int64_t(1) << 31), "mix_normalize_u8: batch too large");
  float m3[3] = {(float)mean[0], (float)mean[1], (float)mean[2]}, s3[3] = {(float)stdv[0], (float)stdv[1], (float)stdv[2]};
  auto opts = torch::TensorOptions().dtype(torch::kFloat32).device(u8.device());
  Tensor out = to_nchw ? torch::empty({N, 3, H, W}, opts) : torch::empty({N, H, W, 3}, opts);
  Tensor lam = torch::empty({1}, opts);
  fb::mix_normalize_u8(u8.data_ptr<uint8_t>(), rp, fptr_mut(out), fptr_mut(lam), (int)N, (int)H, (int)W, augment ? 1 : 0,
                       (uint64_t)key, (uint64_t)counter, m3, s3, to_nchw ? 1 : 0, cutmix ? 1 : 0, (float)lam_f, (float)mlam_f,
                       (int)y0, (int)y1, (int)x0, (int)x1, (float)lam_eff, cur_stream());
  return {out, lam};
}
void col_stats(Tensor y, Tensor stats) {
  CHECK_F32_CUDA(y); CHECK_CONTIG(y);
  c10::cuda::CUDAGuard guard(y.device());
  const int C = (int)y.size(-1);
  fb::col_stats(fptr(y), fptr_mut(stats), (int)(y.numel() / C), C, cur_stream());
}
// y, out: [M, C] views of NHWC tensors.  Returns (out, save_mean, save_invstd).
// use_running: eval-mode BatchNorm on the running statistics (left unchanged); stats may be None and (out, None, None) is returned.
std::vector<Tensor> bn_elu_fwd(Tensor y, c10::optional<Tensor> stats, Tensor gamma, Tensor beta, c10::optional<Tensor> residual,
                               c10::optional<Tensor> running_mean, c10::optional<Tensor> running_var, double eps,
                               double momentum, bool act, bool self_clean, bool use_running) {
  CHECK_F32_CUDA(y); CHECK_CONTIG(y);
  c10::cuda::CUDAGuard guard(y.device());
  const int C = (int)y.size(-1);
  const int M = (int)(y.numel() / C);
  auto out = torch::empty_like(y);
  float* rm = (running_mean.has_value() && running_mean->defined()) ? running_mean->data_ptr<float>() : nullptr;
  float* rv = (running_var.has_value() && running_var->defined()) ? running_var->data_ptr<float>() : nullptr;
  if (use_running) {
    TORCH_CHECK(rm != nullptr && rv != nullptr, "bn_elu_fwd: use_running needs running_mean and running_var");
    fb::bn_elu_fwd(fptr(y), nullptr, fptr(gamma), fptr(beta), opt_ptr(residual), fptr_mut(out), rm, rv, nullptr, nullptr, M, C,
                   (float)eps, 0.f, act ? 1 : 0, 0, cur_stream(), 1);
    return {out, Tensor(), Tensor()};
  }
  TORCH_CHECK(stats.has_value() && stats->defined(), "bn_elu_fwd: stats required");
  auto sm = torch::empty({C}, y.options()), si = torch::empty({C}, y.options());
  TORCH_CHECK(stats->numel() >= 2 * C + (self_clean ? 1 : 0), "stats buffer too small");
  fb::bn_elu_fwd(fptr(y), stats->data_ptr<float>(), fptr(gamma), fptr(beta), opt_ptr(residual), fptr_mut(out), rm, rv, fptr_mut(sm),
                 fptr_mut(si), M, C, (float)eps, (float)momentum, act ? 1 : 0, self_clean ? 1 : 0, cur_stream());
  return {out, sm, si};
}
// ResNet stem (stem_kernels.cu).  x: [N,H,32,3] contiguous, w: [64,3,3,3] contiguous (KRSC), stats: [sum | sumsq | counter].
// mode STORE_Y returns (y); STATS_ONLY returns (); APPLY returns (out, save_mean, save_invstd).
bool stem_conv_supported(int64_t H, int64_t W, int64_t C_in, int64_t C_out) {
  return fb::stem_conv_supported((int)H, (int)W, (int)C_in, (int)C_out);
}
std::vector<Tensor> stem_conv_bn(Tensor x, Tensor w, Tensor stats, int64_t mode, c10::optional<Tensor> gamma,
                                 c10::optional<Tensor> beta, c10::optional<Tensor> running_mean, c10::optional<Tensor> running_var,
                                 double eps, double momentum, bool act, bool self_clean) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_F32_CUDA(w); CHECK_CONTIG(w); CHECK_F32_CUDA(stats);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == 3 && w.size(0) == 64 && w.size(1) == 3 && w.size(2) == 3 &&
                  w.size(3) == 3 && fb::stem_conv_supported((int)x.size(1), (int)x.size(2), 3, 64),
              "stem_conv_bn: x [N,H,32,3] with H % 4 == 0, w [64,3,3,3]");
  TORCH_CHECK(stats.numel() >= 2 * 64 + 1 && stats.is_contiguous(), "stem_conv_bn: stats buffer too small");
  TORCH_CHECK(x.size(0) * x.size(1) * x.size(2) * 64 < (int64_t(1) << 31), "stem_conv_bn: batch too large");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1);
  if (mode == fb::STEM_STATS_ONLY) {
    fb::stem_conv_bn(fb::STEM_STATS_ONLY, fptr(x), fptr(w), nullptr, fptr_mut(stats), nullptr, nullptr, nullptr, nullptr, nullptr,
                     nullptr, NB, H, 0.f, 0.f, 0, 0, cur_stream());
    return {};
  }
  auto out = torch::empty({NB, H, x.size(2), 64}, x.options());
  if (mode == fb::STEM_STORE_Y) {
    fb::stem_conv_bn(fb::STEM_STORE_Y, fptr(x), fptr(w), fptr_mut(out), fptr_mut(stats), nullptr, nullptr, nullptr, nullptr,
                     nullptr, nullptr, NB, H, 0.f, 0.f, 0, 0, cur_stream());
    return {out};
  }
  TORCH_CHECK(mode == fb::STEM_APPLY, "stem_conv_bn: mode must be 0 (STORE_Y), 1 (STATS_ONLY) or 2 (APPLY)");
  TORCH_CHECK(gamma.has_value() && gamma->defined() && beta.has_value() && beta->defined(), "stem_conv_bn: APPLY needs gamma and beta");
  CHECK_F32_CUDA((*gamma)); CHECK_F32_CUDA((*beta));
  float* rm = (running_mean.has_value() && running_mean->defined()) ? running_mean->data_ptr<float>() : nullptr;
  float* rv = (running_var.has_value() && running_var->defined()) ? running_var->data_ptr<float>() : nullptr;
  TORCH_CHECK((rm == nullptr) == (rv == nullptr), "stem_conv_bn: running_mean and running_var go together");
  auto sm = torch::empty({64}, x.options()), si = torch::empty({64}, x.options());
  fb::stem_conv_bn(fb::STEM_APPLY, fptr(x), fptr(w), fptr_mut(out), fptr_mut(stats), fptr(*gamma), fptr(*beta), rm, rv,
                   fptr_mut(sm), fptr_mut(si), NB, H, (float)eps, (float)momentum, act ? 1 : 0, self_clean ? 1 : 0, cur_stream());
  return {out, sm, si};
}
// Returns (dy, dres or undefined); accumulates into dgamma / dbeta when given.
std::vector<Tensor> bn_elu_bwd(Tensor dout, c10::optional<Tensor> out, Tensor y, Tensor mean, Tensor invstd, Tensor gamma,
                               c10::optional<Tensor> beta, c10::optional<Tensor> dgamma, c10::optional<Tensor> dbeta,
                               bool want_dres, bool act, c10::optional<Tensor> sums_buf) {
  CHECK_F32_CUDA(dout); CHECK_CONTIG(dout); CHECK_CONTIG(y);
  c10::cuda::CUDAGuard guard(y.device());
  const int C = (int)y.size(-1);
  const int M = (int)(y.numel() / C);
  const float* outp = nullptr;
  if (out.has_value() && out->defined()) { CHECK_CONTIG((*out)); outp = out->data_ptr<float>(); }
  const float* betap = opt_ptr(beta);
  // sums_buf: a zeroed per-layer [2C + 1] buffer that the apply kernel leaves zeroed again (no memset node per layer)
  const bool persistent = sums_buf.has_value() && sums_buf->defined();
  if (persistent) TORCH_CHECK(sums_buf->numel() == 2 * C + 1 && sums_buf->is_contiguous(), "bn_elu_bwd: sums buffer must be [2C + 1]");
  auto sums = persistent ? *sums_buf : torch::empty({2 * C + 1}, y.options());
  auto dy = torch::empty_like(y);
  Tensor dres;
  if (want_dres) dres = torch::empty_like(y);
  float* dg = (dgamma.has_value() && dgamma->defined()) ? dgamma->data_ptr<float>() : nullptr;
  float* db = (dbeta.has_value() && dbeta->defined()) ? dbeta->data_ptr<float>() : nullptr;
  fb::bn_elu_bwd_reduce(fptr(dout), outp, fptr(y), fptr(mean), fptr(invstd), fptr(gamma), betap, fptr_mut(sums), M, C,
                        act ? 1 : 0, persistent ? 1 : 0, cur_stream());
  fb::bn_elu_bwd_apply(fptr(dout), outp, fptr(y), fptr(mean), fptr(invstd), fptr(gamma), betap, fptr_mut(sums), fptr_mut(dy),
                       want_dres ? dres.data_ptr<float>() : nullptr, dg, db, M, C, act ? 1 : 0, persistent ? 1 : 0, cur_stream());
  return {dy, dres};
}
// GroupNorm + residual + ELU.  y, residual: [N,H,W,C] contiguous.  Returns (out, mean [N,G], rstd [N,G]).
static void check_gn(const Tensor& y, const Tensor& gamma, int64_t groups) {
  CHECK_F32_CUDA(y); CHECK_CONTIG(y);
  TORCH_CHECK(y.dim() == 4, "GroupNorm kernels: y must be [N,H,W,C]");
  CHECK_F32_CUDA(gamma); CHECK_CONTIG(gamma);
  TORCH_CHECK(gamma.numel() == y.size(3), "GroupNorm kernels: gamma must hold C values");
  TORCH_CHECK(groups >= 1 && y.size(3) % groups == 0, "GroupNorm kernels: the group count must divide C");
}
std::vector<Tensor> gn_elu_fwd(Tensor y, Tensor gamma, Tensor beta, c10::optional<Tensor> residual, int64_t groups, double eps,
                               bool act) {
  check_gn(y, gamma, groups);
  CHECK_F32_CUDA(beta); CHECK_CONTIG(beta);
  if (residual.has_value() && residual->defined()) {
    CHECK_F32_CUDA((*residual)); CHECK_CONTIG((*residual));
    TORCH_CHECK(residual->sizes() == y.sizes(), "gn_elu_fwd: residual must have y's shape");
  }
  c10::cuda::CUDAGuard guard(y.device());
  const int N = (int)y.size(0), HW = (int)(y.size(1) * y.size(2)), C = (int)y.size(3), G = (int)groups;
  auto out = torch::empty_like(y);
  auto mean = torch::empty({N, G}, y.options()), rstd = torch::empty({N, G}, y.options());
  auto part = torch::empty({(int64_t)N * fb::gn_splits(N, HW, C) * 2 * C}, y.options());
  auto table = torch::empty({(int64_t)N * 2 * C}, y.options());
  fb::gn_elu_fwd(fptr(y), fptr(gamma), fptr(beta), opt_ptr(residual), fptr_mut(out), fptr_mut(mean), fptr_mut(rstd),
                 fptr_mut(part), fptr_mut(table), N, HW, C, G, (float)eps, act ? 1 : 0, cur_stream());
  return {out, mean, rstd};
}
// Returns (dy, dres or undefined, dgamma or undefined, dbeta or undefined).
std::vector<Tensor> gn_elu_bwd(Tensor dout, c10::optional<Tensor> out, Tensor y, Tensor mean, Tensor rstd, Tensor gamma,
                               c10::optional<Tensor> beta, int64_t groups, bool want_dres, bool act, bool want_affine) {
  check_gn(y, gamma, groups);
  CHECK_F32_CUDA(dout); CHECK_CONTIG(dout);
  TORCH_CHECK(dout.sizes() == y.sizes(), "gn_elu_bwd: dout must have y's shape");
  const int N = (int)y.size(0), HW = (int)(y.size(1) * y.size(2)), C = (int)y.size(3), G = (int)groups;
  TORCH_CHECK(mean.numel() == (int64_t)N * G && rstd.numel() == (int64_t)N * G && mean.is_contiguous() && rstd.is_contiguous(),
              "gn_elu_bwd: mean / rstd must be [N, G]");
  const float* outp = nullptr;
  if (out.has_value() && out->defined()) {
    CHECK_CONTIG((*out));
    TORCH_CHECK(out->sizes() == y.sizes(), "gn_elu_bwd: out must have y's shape");
    outp = out->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(y.device());
  auto part = torch::empty({(int64_t)N * fb::gn_splits(N, HW, C) * 2 * C}, y.options());
  auto ab = torch::empty({2 * (int64_t)N * G}, y.options());
  auto dy = torch::empty_like(y);
  Tensor dres, dgamma, dbeta;
  if (want_dres) dres = torch::empty_like(y);
  if (want_affine) { dgamma = torch::empty_like(gamma); dbeta = torch::empty_like(gamma); }
  fb::gn_elu_bwd(fptr(dout), outp, fptr(y), fptr(mean), fptr(rstd), fptr(gamma), opt_ptr(beta), fptr_mut(part), fptr_mut(ab),
                 fptr_mut(dy), want_dres ? dres.data_ptr<float>() : nullptr, want_affine ? dgamma.data_ptr<float>() : nullptr,
                 want_affine ? dbeta.data_ptr<float>() : nullptr, N, HW, C, G, act ? 1 : 0, cur_stream());
  return {dy, dres, dgamma, dbeta};
}
// fused classifier head: x [N,H,W,C], w [O,C], bias [O] -> (logits [N,O], pooled [N,C])
std::vector<Tensor> head_fwd(Tensor x, Tensor w, c10::optional<Tensor> bias) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_F32_CUDA(w); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 2 && x.size(3) == w.size(1), "head_fwd: x [N,H,W,C], w [O,C]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), HW = (int)(x.size(1) * x.size(2)), C = (int)x.size(3), O = (int)w.size(0);
  auto pooled = torch::empty({NB, C}, x.options());
  auto logits = torch::empty({NB, O}, x.options());
  fb::head_fwd(fptr(x), fptr(w), opt_ptr(bias), fptr_mut(pooled), fptr_mut(logits), NB, HW, C, O, cur_stream());
  return {logits, pooled};
}
Tensor head_bwd(Tensor dlogits, Tensor w, int64_t H, int64_t W) {   // -> dx [N,H,W,C]
  CHECK_F32_CUDA(dlogits); CHECK_CONTIG(dlogits); CHECK_F32_CUDA(w); CHECK_CONTIG(w);
  c10::cuda::CUDAGuard guard(dlogits.device());
  const int NB = (int)dlogits.size(0), O = (int)dlogits.size(1), C = (int)w.size(1);
  auto dx = torch::empty({NB, H, W, C}, dlogits.options());
  fb::head_bwd(fptr(dlogits), fptr(w), fptr_mut(dx), NB, (int)(H * W), C, O, cur_stream());
  return dx;
}
Tensor avgpool_nhwc(Tensor x) {   // [N,H,W,C] -> [N,C]
  CHECK_F32_CUDA(x); CHECK_CONTIG(x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty({x.size(0), x.size(3)}, x.options());
  fb::avgpool_nhwc(fptr(x), fptr_mut(out), (int)x.size(0), (int)(x.size(1) * x.size(2)), (int)x.size(3), cur_stream());
  return out;
}
Tensor avgpool_nhwc_bwd(Tensor dout, int64_t H, int64_t W) {
  CHECK_F32_CUDA(dout); CHECK_CONTIG(dout);
  c10::cuda::CUDAGuard guard(dout.device());
  auto dx = torch::empty({dout.size(0), H, W, dout.size(1)}, dout.options());
  fb::avgpool_nhwc_bwd(fptr(dout), fptr_mut(dx), (int)dout.size(0), (int)(H * W), (int)dout.size(1), cur_stream());
  return dx;
}
Tensor weight_flip(Tensor w) {    // [Co,kh,kw,Ci] -> [Ci,kh,kw,Co], taps rotated
  CHECK_F32_CUDA(w); CHECK_CONTIG(w);
  c10::cuda::CUDAGuard guard(w.device());
  auto out = torch::empty({w.size(3), w.size(1), w.size(2), w.size(0)}, w.options());
  fb::weight_krsc_flip(fptr(w), fptr_mut(out), (int)w.size(0), (int)w.size(3), (int)w.size(1), (int)w.size(2), cur_stream());
  return out;
}

Tensor convT_pack(Tensor w) {    // [Ci, Co, 4, 4] (any strides) -> [4 * Co, 3, 3, Ci]
  CHECK_F32_CUDA(w);
  TORCH_CHECK(w.dim() == 4 && w.size(2) == 4 && w.size(3) == 4, "convT_pack: ConvTranspose2d(k=4) weight expected");
  c10::cuda::CUDAGuard guard(w.device());
  auto out = torch::empty({4 * w.size(1), 3, 3, w.size(0)}, w.options().memory_format(c10::MemoryFormat::Contiguous));
  fb::convT_pack(fptr(w), fptr_mut(out), (int)w.size(0), (int)w.size(1), w.stride(0), w.stride(1), w.stride(2), w.stride(3), cur_stream());
  return out;
}

// ---------------------------------------------------------------------------------------------- tensor cores
Tensor linear_tf32(Tensor x, Tensor w, c10::optional<Tensor> bias, bool act) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "linear_tf32: x [M,K], w [N,K]");
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)x.size(0), K = (int)x.size(1), N = (int)w.size(0);
  auto out = torch::empty({M, N}, x.options());
  fb::linear_tf32(fptr(x), fptr(w), opt_ptr(bias), fptr_mut(out), M, N, K, K, K, N, act ? 1 : 0, cur_stream());
  return out;
}
bool conv_supported(int64_t H_out, int64_t W_out, int64_t C_in, int64_t stride) {
  return fb::conv_geometry_supported((int)H_out, (int)W_out, (int)C_in, (int)stride);
}
// Tile orientation the convolution picks by itself for this output shape (fb::CONV_ORIENT_ROW / _PIXEL)
int64_t conv_orientation(int64_t NB, int64_t H_out, int64_t W_out, int64_t C_out, int64_t stride) {
  return fb::pick_conv_orientation((int)NB, (int)H_out, (int)W_out, (int)C_out, (int)stride);
}
// Whether pixel-major tiles of this shape run the window-reuse main loop (else the per-tap loop)
bool conv_window_reuse(int64_t H_out, int64_t W_out, int64_t C_in, int64_t C_out, int64_t kh, int64_t stride, int64_t dil) {
  return fb::conv_window_reuse((int)H_out, (int)W_out, (int)C_in, (int)C_out, (int)kh, (int)stride, (int)dil);
}
// x: [N,H,W,Ci] contiguous; w: [Co,kh,kw,Ci] contiguous.  Returns y [N,Ho,Wo,Co]; stats (2*Co) accumulated if given.
// orient: -1 = chosen from the shape, 0 = row-major tiles, 1 = pixel-major tiles (C_out 64 / 128; window reuse where
// conv_window_reuse allows it), 2 = pixel-major tiles with the per-tap main loop (A/B comparisons).
Tensor conv2d_nhwc(Tensor x, Tensor w, c10::optional<Tensor> stats, int64_t stride, int64_t pad, int64_t dil, int64_t orient) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  const int Ho = (H + 2 * (int)pad - (int)dil * (kh - 1) - 1) / (int)stride + 1;
  const int Wo = (W + 2 * (int)pad - (int)dil * (kw - 1) - 1) / (int)stride + 1;
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  float* st = (stats.has_value() && stats->defined()) ? stats->data_ptr<float>() : nullptr;
  fb::conv2d_nhwc_tf32(fptr(x), fptr(w), fptr_mut(y), st, NB, H, W, Ci, Co, kh, kw, (int)stride, (int)pad, (int)dil, Ho, Wo, cur_stream(),
                       (int)orient);
  return y;
}

// Same kernel with an explicit output size: the window is anchored at (-pad, -pad) and whatever sticks out on the
// bottom/right is zero-filled by the TMA unit (used by the stride-2 data gradient: 2x2 taps, pad 0, out = in size).
Tensor conv2d_nhwc_sized(Tensor x, Tensor w, c10::optional<Tensor> stats, int64_t stride, int64_t pad, int64_t dil,
                         int64_t Ho, int64_t Wo) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  TORCH_CHECK(Ho > 0 && Wo > 0, "conv2d_nhwc_sized: positive output size");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  float* st = (stats.has_value() && stats->defined()) ? stats->data_ptr<float>() : nullptr;
  fb::conv2d_nhwc_tf32(fptr(x), fptr(w), fptr_mut(y), st, NB, H, W, Ci, Co, kh, kw, (int)stride, (int)pad, (int)dil, (int)Ho,
                       (int)Wo, cur_stream());
  return y;
}

// Weight gradient: dw [Co, kh, kw, Cw] += wgrad(x [N,H,W,Cx], dy [N,Ho,Wo,Co]).  `dw` is accumulated into (zeroed by the
// caller, or the parameter's gradient buffer itself); Cw <= Cx (channel-padded activations).
bool conv_wgrad_supported(int64_t Cx, int64_t Co, int64_t stride, int64_t Wo, int64_t Ho) {
  return fb::conv_wgrad_supported((int)Cx, (int)Co, (int)stride, (int)Wo, (int)Ho);
}
void conv_wgrad(Tensor x, Tensor dy, Tensor dw, int64_t stride, int64_t pad, int64_t dil) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(dy); CHECK_F32_CUDA(dw); CHECK_CONTIG(x); CHECK_CONTIG(dy); CHECK_CONTIG(dw);
  TORCH_CHECK(x.dim() == 4 && dy.dim() == 4 && dw.dim() == 4 && x.size(0) == dy.size(0) && dw.size(0) == dy.size(3) &&
              dw.size(3) <= x.size(3), "conv_wgrad: x [N,H,W,Cx], dy [N,Ho,Wo,Co], dw [Co,kh,kw,Cw<=Cx]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Cx = (int)x.size(3);
  const int Ho = (int)dy.size(1), Wo = (int)dy.size(2), Co = (int)dy.size(3);
  const int kh = (int)dw.size(1), kw = (int)dw.size(2), Cw = (int)dw.size(3);
  fb::conv_wgrad_tf32(fptr(x), fptr(dy), fptr_mut(dw), NB, H, W, Cx, Cw, Co, kh, kw, (int)stride, (int)pad, (int)dil, Ho, Wo,
                      cur_stream());
}

// Phase-packed stride-1 convolution (w: [4*Ci, kh, kw, Cin]) whose output lands pixel-shuffled: returns [N, 2*Ho, 2*Wo, Ci].
bool conv_shuffle_supported(int64_t Ho, int64_t Wo, int64_t Cin, int64_t Ci) {
  return fb::conv_shuffle_supported((int)Ho, (int)Wo, (int)Cin, (int)Ci);
}
Tensor conv2d_nhwc_shuffle(Tensor x, Tensor w, int64_t pad, int64_t Ho, int64_t Wo) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3) && w.size(0) % 4 == 0, "conv2d_nhwc_shuffle: x [N,H,W,Cin], w [4*Ci,kh,kw,Cin]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Cin = (int)x.size(3);
  const int C4 = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  auto out = torch::empty({NB, 2 * Ho, 2 * Wo, C4 / 4}, x.options());
  fb::conv2d_nhwc_shuffle_tf32(fptr(x), fptr(w), fptr_mut(out), NB, H, W, Cin, C4, kh, kw, (int)pad, (int)Ho, (int)Wo, cur_stream());
  return out;
}

// `B` dilated convolutions of the same input in one launch: w [Co_total, B * kh, kw, Ci] block diagonal, y [N, Ho, Wo, Co_total]
bool conv_multidil_supported(int64_t Ho, int64_t Wo, int64_t Ci, int64_t stride, int64_t branches) {
  return fb::conv_multidil_supported((int)Ho, (int)Wo, (int)Ci, (int)stride, (int)branches);
}
Tensor conv2d_nhwc_multidil(Tensor x, Tensor w, c10::optional<Tensor> bias, bool act, int64_t kh, int64_t stride,
                            std::vector<int64_t> dils, std::vector<int64_t> pads, int64_t Ho, int64_t Wo) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc_multidil: x [N,H,W,Ci], w [Co,B*kh,kw,Ci]");
  const int B = (int)dils.size();
  TORCH_CHECK(B >= 1 && B <= 8 && (int)pads.size() == B && w.size(1) == B * kh, "conv2d_nhwc_multidil: branch tables");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kw = (int)w.size(2);
  if (bias.has_value() && bias->defined()) TORCH_CHECK(bias->numel() == Co && bias->is_contiguous(), "bias must be [Co]");
  int d[8], pd[8];
  for (int b = 0; b < B; ++b) { d[b] = (int)dils[b]; pd[b] = (int)pads[b]; }
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  fb::conv2d_nhwc_multidil_tf32(fptr(x), fptr(w), opt_ptr(bias), act ? 1 : 0, fptr_mut(y), NB, H, W, Ci, Co, B, (int)kh, kw,
                                (int)stride, d, pd, (int)Ho, (int)Wo, cur_stream());
  return y;
}

// conv + bias (+ ELU) in one kernel: the bias-carrying convolutions of the VAE / CPC networks (SURVEY G6)
Tensor conv2d_nhwc_bias_act(Tensor x, Tensor w, c10::optional<Tensor> bias, bool act, int64_t stride, int64_t pad, int64_t dil) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  const int Ho = (H + 2 * (int)pad - (int)dil * (kh - 1) - 1) / (int)stride + 1;
  const int Wo = (W + 2 * (int)pad - (int)dil * (kw - 1) - 1) / (int)stride + 1;
  TORCH_CHECK(Ho > 0 && Wo > 0, "conv2d_nhwc_bias_act: empty output");
  if (bias.has_value() && bias->defined()) TORCH_CHECK(bias->numel() == Co && bias->is_contiguous(), "bias must be [Co]");
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  fb::conv2d_nhwc_bias_act_tf32(fptr(x), fptr(w), opt_ptr(bias), act ? 1 : 0, fptr_mut(y), NB, H, W, Ci, Co, kh, kw, (int)stride,
                                (int)pad, (int)dil, Ho, Wo, cur_stream());
  return y;
}

// conv + eval-mode BatchNorm (running statistics) (+ residual) (+ ELU): inference of the ResNet groups.  x [N,H,W,Ci],
// w [Co,kh,kw,Ci], residual [N,Ho,Wo,Co] or None; returns y [N,Ho,Wo,Co].  The running statistics are only read.
Tensor conv2d_nhwc_bn_eval(Tensor x, Tensor w, Tensor gamma, Tensor beta, Tensor running_mean, Tensor running_var, double eps,
                           c10::optional<Tensor> residual, bool act, int64_t stride, int64_t pad) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc_bn_eval: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  const int Ho = (H + 2 * (int)pad - (kh - 1) - 1) / (int)stride + 1;
  const int Wo = (W + 2 * (int)pad - (kw - 1) - 1) / (int)stride + 1;
  TORCH_CHECK(Ho > 0 && Wo > 0, "conv2d_nhwc_bn_eval: empty output");
  for (const Tensor* t : {&gamma, &beta, &running_mean, &running_var}) {
    CHECK_F32_CUDA((*t));
    TORCH_CHECK(t->numel() == Co && t->is_contiguous(), "conv2d_nhwc_bn_eval: BatchNorm parameters and statistics must be [Co]");
  }
  const float* res = nullptr;
  if (residual.has_value() && residual->defined()) {
    CHECK_F32_CUDA((*residual)); CHECK_CONTIG((*residual));
    TORCH_CHECK(residual->dim() == 4 && residual->size(0) == NB && residual->size(1) == Ho && residual->size(2) == Wo &&
                residual->size(3) == Co, "conv2d_nhwc_bn_eval: residual must be [N,Ho,Wo,Co]");
    res = residual->data_ptr<float>();
    TORCH_CHECK((reinterpret_cast<uintptr_t>(res) & 15) == 0, "conv2d_nhwc_bn_eval: residual must be 16-byte aligned");
  }
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  fb::conv2d_nhwc_bn_eval_tf32(fptr(x), fptr(w), fptr(gamma), fptr(beta), fptr(running_mean), fptr(running_var), (float)eps, res,
                               act ? 1 : 0, fptr_mut(y), NB, H, W, Ci, Co, kh, kw, (int)stride, (int)pad, 1, Ho, Wo, cur_stream());
  return y;
}

// ---------------------------------------------------------------------------------------------- losses
std::vector<Tensor> cross_entropy_fwd(Tensor logits, Tensor labels) {
  CHECK_F32_CUDA(logits); CHECK_CONTIG(logits);
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.is_cuda(), "labels must be CUDA int64");
  c10::cuda::CUDAGuard guard(logits.device());
  auto loss = torch::empty({}, logits.options());
  auto probs = torch::empty_like(logits);
  fb::cross_entropy_fwd(fptr(logits), (const long long*)labels.data_ptr<int64_t>(), fptr_mut(loss), fptr_mut(probs),
                        (int)logits.size(0), (int)logits.size(1), cur_stream());
  return {loss, probs};
}
Tensor cross_entropy_bwd(Tensor probs, Tensor labels, Tensor gout) {
  c10::cuda::CUDAGuard guard(probs.device());
  auto d = torch::empty_like(probs);
  auto g = gout.contiguous();
  fb::cross_entropy_bwd(fptr(probs), (const long long*)labels.data_ptr<int64_t>(), fptr(g), fptr_mut(d), (int)probs.size(0),
                        (int)probs.size(1), cur_stream());
  return d;
}
// lam: optional one-float32 device tensor (absent = 1); the target of sample i mixes labels i and B-1-i.
static const float* soft_ce_lam(const c10::optional<Tensor>& lam, const Tensor& like) {
  if (!lam.has_value() || !lam->defined()) return nullptr;
  TORCH_CHECK(lam->is_cuda() && lam->device() == like.device() && lam->scalar_type() == torch::kFloat32 && lam->numel() == 1,
              "soft_ce: lam must be a one-element CUDA float32 tensor on the logits' device");
  return lam->data_ptr<float>();
}
std::vector<Tensor> soft_ce_fwd(Tensor logits, Tensor labels, c10::optional<Tensor> lam, double eps) {
  CHECK_F32_CUDA(logits); CHECK_CONTIG(logits);
  TORCH_CHECK(logits.dim() == 2 && logits.size(0) >= 1 && logits.size(1) >= 1, "soft_ce_fwd: logits must be [B >= 1, C >= 1]");
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.is_cuda() && labels.is_contiguous() &&
                  labels.numel() == logits.size(0), "soft_ce_fwd: labels must be a contiguous CUDA int64 [B] tensor");
  TORCH_CHECK(eps >= 0.0 && eps < 1.0, "soft_ce_fwd: eps must lie in [0, 1)");
  c10::cuda::CUDAGuard guard(logits.device());
  auto loss = torch::empty({}, logits.options());
  auto probs = torch::empty_like(logits);
  fb::soft_ce_fwd(fptr(logits), (const long long*)labels.data_ptr<int64_t>(), soft_ce_lam(lam, logits), (float)eps,
                  fptr_mut(loss), fptr_mut(probs), (int)logits.size(0), (int)logits.size(1), cur_stream());
  return {loss, probs};
}
Tensor soft_ce_bwd(Tensor probs, Tensor labels, c10::optional<Tensor> lam, double eps, Tensor gout) {
  CHECK_F32_CUDA(probs); CHECK_CONTIG(probs);
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && labels.is_cuda() && labels.is_contiguous() &&
                  labels.numel() == probs.size(0), "soft_ce_bwd: labels must be a contiguous CUDA int64 [B] tensor");
  c10::cuda::CUDAGuard guard(probs.device());
  auto d = torch::empty_like(probs);
  auto g = gout.contiguous();
  fb::soft_ce_bwd(fptr(probs), (const long long*)labels.data_ptr<int64_t>(), soft_ce_lam(lam, probs), (float)eps, fptr(g),
                  fptr_mut(d), (int)probs.size(0), (int)probs.size(1), cur_stream());
  return d;
}
Tensor vae_loss_fwd(Tensor recon, Tensor x, Tensor mu, Tensor logvar) {
  CHECK_F32_CUDA(recon); CHECK_CONTIG(recon); CHECK_CONTIG(x); CHECK_CONTIG(mu); CHECK_CONTIG(logvar);
  c10::cuda::CUDAGuard guard(recon.device());
  auto out = torch::empty({}, recon.options());
  fb::vae_loss_fwd(fptr(recon), fptr(x), (int)recon.numel(), fptr(mu), fptr(logvar), (int)mu.numel(), fptr_mut(out), cur_stream());
  return out;
}
std::vector<Tensor> vae_loss_bwd(Tensor recon, Tensor x, Tensor mu, Tensor logvar, Tensor gout) {
  c10::cuda::CUDAGuard guard(recon.device());
  auto dr = torch::empty_like(recon), dm = torch::empty_like(mu), dl = torch::empty_like(logvar);
  auto g = gout.contiguous();
  fb::vae_loss_bwd(fptr(recon), fptr(x), (int)recon.numel(), fptr(mu), fptr(logvar), (int)mu.numel(), fptr(g), fptr_mut(dr),
                   fptr_mut(dm), fptr_mut(dl), cur_stream());
  return {dr, dm, dl};
}

// ---------------------------------------------------------------------------------------------- aux (true fp32)
// out[M,N] (+)= act(x[M,K] w[N,K]^T + b): nn.Linear forward
Tensor linear_f32(Tensor x, Tensor w, c10::optional<Tensor> bias, bool act) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1), "linear_f32: x [M,K], w [N,K]");
  c10::cuda::CUDAGuard guard(x.device());
  const int M = (int)x.size(0), K = (int)x.size(1), N = (int)w.size(0);
  auto out = torch::empty({M, N}, x.options());
  fb::gemm_f32(fptr(x), fptr(w), opt_ptr(bias), fptr_mut(out), M, N, K, K, 1, 1, K, N, act ? 1 : 0, 0, cur_stream());
  return out;
}
// dx[M,K] = dz[M,N] w[N,K]
Tensor linear_f32_dgrad(Tensor dz, Tensor w) {
  CHECK_F32_CUDA(dz); CHECK_F32_CUDA(w); CHECK_CONTIG(dz); CHECK_CONTIG(w);
  c10::cuda::CUDAGuard guard(dz.device());
  const int M = (int)dz.size(0), N = (int)dz.size(1), K = (int)w.size(1);
  auto dx = torch::empty({M, K}, dz.options());
  fb::gemm_f32(fptr(dz), fptr(w), nullptr, fptr_mut(dx), M, K, N, N, 1, K, 1, K, 0, 0, cur_stream());
  return dx;
}
// dw[N,K] (+)= dz[M,N]^T x[M,K]   (accumulate = add into an existing gradient buffer)
void linear_f32_wgrad(Tensor dz, Tensor x, Tensor dw, bool accumulate) {
  CHECK_F32_CUDA(dz); CHECK_F32_CUDA(x); CHECK_F32_CUDA(dw); CHECK_CONTIG(dz); CHECK_CONTIG(x); CHECK_CONTIG(dw);
  c10::cuda::CUDAGuard guard(dz.device());
  const int M = (int)dz.size(0), N = (int)dz.size(1), K = (int)x.size(1);
  TORCH_CHECK(dw.size(0) == N && dw.size(1) == K && x.size(0) == M, "linear_f32_wgrad: shape mismatch");
  fb::gemm_f32(fptr(dz), fptr(x), nullptr, fptr_mut(dw), N, K, M, 1, N, K, 1, K, 0, accumulate ? 1 : 0, cur_stream());
}
// dz = dout * ELU'(z) (act) ; db += column sums of dz.  dz / db optional (pass None).  Tensors are [..., C] contiguous.
void act_bwd_bias(Tensor dout, c10::optional<Tensor> out, c10::optional<Tensor> dz, c10::optional<Tensor> db, bool act) {
  CHECK_F32_CUDA(dout); CHECK_CONTIG(dout);
  c10::cuda::CUDAGuard guard(dout.device());
  const int C = (int)dout.size(-1);
  float* dzp = (dz.has_value() && dz->defined()) ? dz->data_ptr<float>() : nullptr;
  float* dbp = (db.has_value() && db->defined()) ? db->data_ptr<float>() : nullptr;
  TORCH_CHECK(!act || (out.has_value() && out->defined()), "act_bwd_bias: the activation output is needed for ELU'");
  fb::act_bwd_bias(fptr(dout), opt_ptr(out), dzp, dbp, (long long)dout.numel(), C, act ? 1 : 0, cur_stream());
}
// x: logical NCHW, memory either contiguous NCHW or channels_last (NHWC); the output keeps the input's memory format
std::vector<Tensor> maxpool2x2_fwd(Tensor x) {
  CHECK_F32_CUDA(x);
  TORCH_CHECK(x.dim() == 4, "maxpool2x2: 4-D tensor expected");
  const bool nhwc = !x.is_contiguous() && x.is_contiguous(at::MemoryFormat::ChannelsLast);
  TORCH_CHECK(nhwc || x.is_contiguous(), "maxpool2x2: contiguous or channels_last input");
  c10::cuda::CUDAGuard guard(x.device());
  const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
  auto fmt = nhwc ? at::MemoryFormat::ChannelsLast : at::MemoryFormat::Contiguous;
  auto y = torch::empty({N, C, H / 2, W / 2}, x.options().memory_format(fmt));
  auto idx = torch::empty({N, C, H / 2, W / 2}, x.options().dtype(torch::kUInt8).memory_format(fmt));
  fb::maxpool2x2_fwd(fptr(x), fptr_mut(y), idx.data_ptr<uint8_t>(), N, C, H, W, nhwc ? 1 : 0, cur_stream());
  return {y, idx};
}
Tensor maxpool2x2_bwd(Tensor dy, Tensor idx, int64_t H, int64_t W) {
  CHECK_F32_CUDA(dy);
  const bool nhwc = !idx.is_contiguous() && idx.is_contiguous(at::MemoryFormat::ChannelsLast);
  auto fmt = nhwc ? at::MemoryFormat::ChannelsLast : at::MemoryFormat::Contiguous;
  Tensor d = dy.contiguous(fmt);
  c10::cuda::CUDAGuard guard(dy.device());
  const int N = (int)dy.size(0), C = (int)dy.size(1);
  auto dx = torch::empty({N, C, H, W}, dy.options().memory_format(fmt));
  fb::maxpool2x2_bwd(fptr(d), idx.data_ptr<uint8_t>(), fptr_mut(dx), N, C, (int)H, (int)W, nhwc ? 1 : 0, cur_stream());
  return dx;
}
void argmax_count(Tensor logits, Tensor labels, Tensor counter) {
  CHECK_F32_CUDA(logits); CHECK_CONTIG(logits);
  TORCH_CHECK(labels.scalar_type() == torch::kInt64 && counter.scalar_type() == torch::kInt64 && counter.numel() >= 2, "argmax_count: int64 labels / counter[2]");
  c10::cuda::CUDAGuard guard(logits.device());
  fb::argmax_count(fptr(logits), (const long long*)labels.data_ptr<int64_t>(), (long long*)counter.data_ptr<int64_t>(), (int)logits.size(0),
                   (int)logits.size(1), cur_stream());
}
int64_t info_nce_max_p() { return fb::info_nce_max_p(); }
int64_t info_nce_scratch_floats() { return fb::info_nce_scratch_floats(); }
std::vector<Tensor> info_nce_fwd(Tensor Z, Tensor Zh, Tensor scratch) {     // Z, Zh: [R, P]
  CHECK_F32_CUDA(Z); CHECK_F32_CUDA(Zh); CHECK_CONTIG(Z); CHECK_CONTIG(Zh);
  c10::cuda::CUDAGuard guard(Z.device());
  const int R = (int)Z.size(0), P = (int)Z.size(1);
  auto loss = torch::empty({}, Z.options());
  auto coef = torch::empty({(int64_t)P * P + 2 * P}, Z.options());
  fb::info_nce_fwd(fptr(Z), fptr(Zh), R, P, fptr_mut(scratch), fptr_mut(loss), fptr_mut(coef), cur_stream());
  return {loss, coef};
}
std::vector<Tensor> info_nce_bwd(Tensor Z, Tensor Zh, Tensor coef, Tensor gout) {
  CHECK_F32_CUDA(Z); CHECK_CONTIG(Z); CHECK_CONTIG(Zh);
  c10::cuda::CUDAGuard guard(Z.device());
  auto dZ = torch::empty_like(Z), dZh = torch::empty_like(Zh);
  fb::info_nce_bwd(fptr(Z), fptr(Zh), fptr(coef), fptr(gout), fptr_mut(dZ), fptr_mut(dZh), (int)Z.size(0), (int)Z.size(1), cur_stream());
  return {dZ, dZh};
}
Tensor gauss_nll_rows_fwd(Tensor x, Tensor mu, Tensor s2) {     // x [B, D], mu / s2 [rows, D] with rows % B == 0
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(mu); CHECK_F32_CUDA(s2); CHECK_CONTIG(x); CHECK_CONTIG(mu); CHECK_CONTIG(s2);
  c10::cuda::CUDAGuard guard(x.device());
  const int B = (int)x.size(0), D = (int)x.size(1), rows = (int)mu.size(0);
  TORCH_CHECK(mu.size(1) == D && rows % B == 0, "gauss_nll_rows: mu [k*B, D]");
  auto out = torch::empty({rows}, x.options());
  fb::gauss_nll_rows_fwd(fptr(x), fptr(mu), fptr(s2), fptr_mut(out), rows, B, D, cur_stream());
  return out;
}
std::vector<Tensor> gauss_nll_rows_bwd(Tensor x, Tensor mu, Tensor s2, Tensor grow) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_CONTIG(mu); CHECK_CONTIG(s2); CHECK_CONTIG(grow);
  c10::cuda::CUDAGuard guard(x.device());
  auto dmu = torch::empty_like(mu), ds2 = torch::empty_like(s2);
  fb::gauss_nll_rows_bwd(fptr(x), fptr(mu), fptr(s2), fptr(grow), fptr_mut(dmu), fptr_mut(ds2), (int)mu.size(0), (int)x.size(0),
                         (int)x.size(1), cur_stream());
  return {dmu, ds2};
}
// direct small convolutions, NCHW
bool smallconv_supported(int64_t Ci, int64_t Co, int64_t k) { return fb::smallconv_supported((int)Ci, (int)Co, (int)k); }
std::vector<Tensor> smallconv_fwd(Tensor x, Tensor w, c10::optional<Tensor> bias, int64_t pad, bool act, bool pool) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), Ci = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), Co = (int)w.size(0), k = (int)w.size(2);
  const int Ho = H + 2 * (int)pad - k + 1, Wo = W + 2 * (int)pad - k + 1;
  auto y = torch::empty({NB, Co, pool ? Ho / 2 : Ho, pool ? Wo / 2 : Wo}, x.options());
  Tensor idx = pool ? torch::empty(y.sizes(), x.options().dtype(torch::kUInt8)) : torch::empty({0}, x.options().dtype(torch::kUInt8));
  fb::smallconv_fwd(fptr(x), fptr(w), opt_ptr(bias), fptr_mut(y), pool ? idx.data_ptr<uint8_t>() : nullptr, NB, Ci, H, W, Co, k,
                    (int)pad, act ? 1 : 0, pool ? 1 : 0, cur_stream());
  return {y, idx};
}
// gradient of the pooled / activated output -> gradient of the pre-activation conv output [NB, Co, Ho, Wo]
Tensor smallconv_unpool_actbwd(Tensor dy, Tensor yout, Tensor idx, int64_t Ho, int64_t Wo, bool act, bool pool) {
  CHECK_F32_CUDA(dy); CHECK_CONTIG(dy); CHECK_CONTIG(yout);
  c10::cuda::CUDAGuard guard(dy.device());
  auto dz = torch::empty({dy.size(0), dy.size(1), Ho, Wo}, dy.options());
  fb::smallconv_unpool_actbwd(fptr(dy), fptr(yout), pool ? idx.data_ptr<uint8_t>() : nullptr, fptr_mut(dz),
                              (long long)(dy.size(0) * dy.size(1)), (int)Ho, (int)Wo, act ? 1 : 0, pool ? 1 : 0, cur_stream());
  return dz;
}
Tensor smallconv_dgrad(Tensor dz, Tensor w, int64_t H, int64_t W, int64_t pad) {
  CHECK_F32_CUDA(dz); CHECK_CONTIG(dz); CHECK_CONTIG(w);
  c10::cuda::CUDAGuard guard(dz.device());
  const int NB = (int)dz.size(0), Co = (int)w.size(0), Ci = (int)w.size(1), k = (int)w.size(2);
  auto dx = torch::empty({NB, Ci, H, W}, dz.options());
  fb::smallconv_dgrad(fptr(dz), fptr(w), fptr_mut(dx), NB, Ci, (int)H, (int)W, Co, k, (int)pad, cur_stream());
  return dx;
}
void smallconv_wgrad(Tensor dz, Tensor x, Tensor dw, c10::optional<Tensor> db, int64_t pad) {   // dw / db are accumulated into
  CHECK_F32_CUDA(dz); CHECK_CONTIG(dz); CHECK_CONTIG(x); CHECK_CONTIG(dw);
  c10::cuda::CUDAGuard guard(dz.device());
  const int NB = (int)x.size(0), Ci = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3), Co = (int)dw.size(0), k = (int)dw.size(2);
  float* dbp = (db.has_value() && db->defined()) ? db->data_ptr<float>() : nullptr;
  fb::smallconv_wgrad(fptr(dz), fptr(x), fptr_mut(dw), dbp, NB, Ci, H, W, Co, k, (int)pad, cur_stream());
}

// ---------------------------------------------------------------------------------------------- collectives
// Pointers are passed as integers: local tensors' data_ptr() or peer-mapped addresses from symmetric memory.
// agg = AGG_MEAN / AGG_MEDIAN / AGG_TRIMMED picks the aggregation rule (trim_b: values dropped at each end, trimmed mean).
// DP rounds (dp_t given): noise std of the mean, key of the noise stream, the device round counter (int64), the stats
// record of the dp_clip launch that precedes the aggregation and, optionally, the block's parameter layout (dp_valid).
static void set_dp(fb::CommArgs& a, double dp_std, int64_t dp_key, const c10::optional<Tensor>& dp_t,
                   const c10::optional<Tensor>& dp_stats, const c10::optional<Tensor>& dp_valid) {
  if (!dp_t.has_value() || !dp_t->defined()) return;
  TORCH_CHECK(dp_t->is_cuda() && dp_t->scalar_type() == at::kLong && dp_t->numel() >= 1, "DP round counter: int64 CUDA tensor");
  TORCH_CHECK(dp_stats.has_value() && dp_stats->defined() && dp_stats->numel() >= fb::DP_STATS_FLOATS,
              "DP rounds need the dp_clip stats record");
  CHECK_F32_CUDA((*dp_stats));
  a.dp = 1;
  a.dp_std = (float)dp_std;
  a.dp_key = (unsigned long long)dp_key;
  a.dp_t = reinterpret_cast<long long*>(dp_t->data_ptr<int64_t>());
  a.dp_stats = dp_stats->data_ptr<float>() + fb::DP_NORM;
  if (dp_valid.has_value() && dp_valid->defined()) {
    TORCH_CHECK(dp_valid->is_cuda() && dp_valid->scalar_type() == at::kByte && dp_valid->is_contiguous() &&
                    dp_valid->numel() >= (a.n + fb::DP_CHUNK - 1) / fb::DP_CHUNK,
                "DP parameter layout: uint8 CUDA tensor with one count per 32-float chunk of the block");
    a.dp_valid = dp_valid->data_ptr<uint8_t>();
  }
}
// Compressed rounds (q_bits 8 or 4): the group size (must be Q_GROUP), key of the rounding stream, the device round
// counter (int64), the payload pointer tables of ALL K workers (codes, scales; local or peer-mapped), the error-feedback
// slices of the local replicas (empty: off) and the per-CTA statistics buffer.
static void set_q(fb::CommArgs& a, const std::vector<int64_t>& local_idx, int64_t q_bits, int64_t q_group, int64_t q_key,
                  const c10::optional<Tensor>& q_t, const std::vector<int64_t>& q_code_ptrs,
                  const std::vector<int64_t>& q_scale_ptrs, const std::vector<Tensor>& q_ef,
                  const c10::optional<Tensor>& q_part) {
  if (q_bits == 0) return;
  TORCH_CHECK(q_bits == 8 || q_bits == 4, "compressed rounds take 8 or 4 bits, got ", q_bits);
  TORCH_CHECK(q_group == fb::Q_GROUP, "compressed rounds use groups of ", fb::Q_GROUP, " coordinates, got ", q_group);
  TORCH_CHECK(q_t.has_value() && q_t->defined() && q_t->is_cuda() && q_t->scalar_type() == at::kLong && q_t->numel() >= 1,
              "compressed round counter: int64 CUDA tensor");
  TORCH_CHECK(q_part.has_value() && q_part->defined() && q_part->numel() >= fb::Q_PART_FLOATS, "compressed rounds need the statistics buffer");
  CHECK_F32_CUDA((*q_part));
  TORCH_CHECK((int)q_code_ptrs.size() == a.K && (int)q_scale_ptrs.size() == a.K, "compressed rounds need K payload pointers");
  TORCH_CHECK(q_ef.empty() || (int)q_ef.size() == a.n_local, "error feedback: one slice per local replica");
  a.qbits = (int)q_bits;
  a.q_key = (unsigned long long)q_key;
  a.q_t = reinterpret_cast<long long*>(q_t->data_ptr<int64_t>());
  a.q_part = q_part->data_ptr<float>();
  for (int k = 0; k < a.K; ++k) {
    TORCH_CHECK(q_code_ptrs[k] % 16 == 0 && q_scale_ptrs[k] % 4 == 0, "payload slices must be 16-byte aligned");
    a.q_codes[k] = reinterpret_cast<unsigned char*>(q_code_ptrs[k]);
    a.q_scales[k] = reinterpret_cast<float*>(q_scale_ptrs[k]);
  }
  for (int j = 0; j < a.n_local; ++j) {
    a.q_worker[j] = (int)local_idx[j];
    if (!q_ef.empty()) {
      CHECK_F32_CUDA(q_ef[j]); CHECK_CONTIG(q_ef[j]);
      TORCH_CHECK(q_ef[j].numel() == a.n, "error feedback slices must have the block's length");
      a.q_ef[j] = q_ef[j].data_ptr<float>();
    }
  }
}
// Sampled rounds (samp_S > 0): participants per round, key of the sampling stream, the device round counter (int64) and
// the K workers' sample counts (int32, on the device).
static void set_samp(fb::CommArgs& a, int64_t samp_S, int64_t samp_key, const c10::optional<Tensor>& samp_t,
                     const c10::optional<Tensor>& client_n) {
  if (samp_S == 0) return;
  TORCH_CHECK(samp_t.has_value() && samp_t->defined() && samp_t->is_cuda() && samp_t->scalar_type() == at::kLong &&
                  samp_t->numel() >= 1, "sampled round counter: int64 CUDA tensor");
  TORCH_CHECK(client_n.has_value() && client_n->defined() && client_n->is_cuda() && client_n->scalar_type() == at::kInt &&
                  client_n->is_contiguous() && client_n->numel() == a.K, "sample counts: one int32 CUDA value per worker");
  a.samp_S = (int)samp_S;
  a.samp_key = (unsigned long long)samp_key;
  a.samp_t = reinterpret_cast<long long*>(samp_t->data_ptr<int64_t>());
  a.client_n = client_n->data_ptr<int>();
}
// Secure-aggregation rounds (sa_t given): f, the clip R, the pair-key table (int32 [K (K - 1) / 2, 8], on the device),
// the device round counter (int64: the nonce), the payload pointers of ALL K workers (4 bytes per coordinate, local or
// peer-mapped) and the per-CTA statistics buffer.
static void set_sa(fb::CommArgs& a, const std::vector<int64_t>& local_idx, int64_t sa_frac_bits, double sa_clip,
                   const c10::optional<Tensor>& sa_keys, const c10::optional<Tensor>& sa_t,
                   const std::vector<int64_t>& sa_pay_ptrs, const c10::optional<Tensor>& sa_part) {
  if (!sa_t.has_value() || !sa_t->defined()) return;
  TORCH_CHECK(sa_t->is_cuda() && sa_t->scalar_type() == at::kLong && sa_t->numel() >= 1,
              "secure-aggregation round counter: int64 CUDA tensor");
  TORCH_CHECK(sa_keys.has_value() && sa_keys->defined() && sa_keys->is_cuda() && sa_keys->scalar_type() == at::kInt &&
                  sa_keys->is_contiguous() && sa_keys->numel() == (int64_t)a.K * (a.K - 1) / 2 * 8,
              "secure-aggregation pair keys: int32 CUDA tensor [K (K - 1) / 2, 8]");
  TORCH_CHECK(sa_part.has_value() && sa_part->defined() && sa_part->numel() >= fb::Q_PART_FLOATS,
              "secure-aggregation rounds need the statistics buffer");
  CHECK_F32_CUDA((*sa_part));
  TORCH_CHECK((int)sa_pay_ptrs.size() == a.K, "secure-aggregation rounds need K payload pointers");
  a.sa = 1;
  a.sa_frac_bits = (int)sa_frac_bits;
  a.sa_clip = (float)sa_clip;
  a.sa_keys = reinterpret_cast<const uint32_t*>(sa_keys->data_ptr<int>());
  a.q_t = reinterpret_cast<long long*>(sa_t->data_ptr<int64_t>());
  a.q_part = sa_part->data_ptr<float>();
  for (int k = 0; k < a.K; ++k) {
    TORCH_CHECK(sa_pay_ptrs[k] % 16 == 0, "payload slices must be 16-byte aligned");
    a.q_codes[k] = reinterpret_cast<unsigned char*>(sa_pay_ptrs[k]);
  }
  for (int j = 0; j < a.n_local; ++j) a.q_worker[j] = (int)local_idx[j];
}
// Top-k rounds (topk_k > 0): k_sel, the payload pointers of ALL K workers (TopKLayout words, local or peer-mapped) and the
// statistics buffer that topk_select filled.
static void set_topk(fb::CommArgs& a, int64_t topk_k, const std::vector<int64_t>& topk_pay_ptrs,
                     const c10::optional<Tensor>& topk_part) {
  if (topk_k == 0) return;
  TORCH_CHECK(topk_k >= 1 && topk_k <= a.n, "top-k rounds need 1 <= k <= n");
  TORCH_CHECK(topk_part.has_value() && topk_part->defined() && topk_part->numel() >= fb::TOPK_STATS_FLOATS,
              "top-k rounds need the selection statistics buffer");
  CHECK_F32_CUDA((*topk_part));
  TORCH_CHECK((int)topk_pay_ptrs.size() == a.K, "top-k rounds need K payload pointers");
  a.topk_k = (int)topk_k;
  a.q_part = topk_part->data_ptr<float>();
  for (int k = 0; k < a.K; ++k) {
    TORCH_CHECK(topk_pay_ptrs[k] % 16 == 0, "payload slices must be 16-byte aligned");
    a.q_codes[k] = reinterpret_cast<unsigned char*>(topk_pay_ptrs[k]);
  }
}
static void fill_ctrl(uint32_t** dst, const std::vector<int64_t>& ctrl_ptrs, int world) {
  for (int p = 0; p < world && p < (int)ctrl_ptrs.size(); ++p) dst[p] = reinterpret_cast<uint32_t*>(ctrl_ptrs[p]);
}
void block_reduce(int64_t mode, std::vector<int64_t> x_ptrs, std::vector<int64_t> y_ptrs, std::vector<int64_t> local_idx,
                  Tensor z, int64_t n, double rho, c10::optional<Tensor> rho_dev, Tensor out, Tensor scratch,
                  std::vector<int64_t> ctrl_ptrs, Tensor sync, int64_t world, int64_t rank, int64_t mc_x, int64_t mc_y,
                  int64_t mc_z, std::vector<int64_t> xw_ptrs, std::vector<int64_t> zw_ptrs, bool two_shot,
                  int64_t max_blocks, double timeout_s, int64_t agg, int64_t trim_b, double dp_std, int64_t dp_key,
                  c10::optional<Tensor> dp_t, c10::optional<Tensor> dp_stats, c10::optional<Tensor> dp_valid,
                  int64_t q_bits, int64_t q_group, int64_t q_key,
                  c10::optional<Tensor> q_t, std::vector<int64_t> q_code_ptrs, std::vector<int64_t> q_scale_ptrs,
                  std::vector<Tensor> q_ef, c10::optional<Tensor> q_part, int64_t samp_S, int64_t samp_key,
                  c10::optional<Tensor> samp_t, c10::optional<Tensor> client_n, int64_t sa_frac_bits, double sa_clip,
                  c10::optional<Tensor> sa_keys, c10::optional<Tensor> sa_t, std::vector<int64_t> sa_pay_ptrs,
                  c10::optional<Tensor> sa_part, int64_t topk_k, std::vector<int64_t> topk_pay_ptrs,
                  c10::optional<Tensor> topk_part) {
  CHECK_F32_CUDA(z); CHECK_F32_CUDA(out); CHECK_F32_CUDA(scratch);
  TORCH_CHECK(out.numel() >= fb::COMM_OUT_FLOATS && scratch.numel() >= fb::COMM_SCRATCH_FLOATS, "out / scratch too small");
  c10::cuda::CUDAGuard guard(z.device());
  fb::CommArgs a{};
  a.mode = (int)mode; a.K = (int)x_ptrs.size(); a.n_local = (int)local_idx.size(); a.world = (int)world; a.rank = (int)rank;
  a.n = (int)n; a.rho = (float)rho; a.rho_dev = opt_ptr(rho_dev);
  a.two_shot = two_shot ? 1 : 0; a.max_blocks = (int)max_blocks;
  TORCH_CHECK(a.K <= fb::COMM_MAX_K && a.n_local <= fb::COMM_MAX_LOCAL && a.world <= fb::COMM_MAX_WORLD, "block_reduce: limits exceeded");
  for (int k = 0; k < a.K; ++k) {
    a.x[k] = reinterpret_cast<const float*>(x_ptrs[k]);
    a.y[k] = y_ptrs.empty() ? nullptr : reinterpret_cast<const float*>(y_ptrs[k]);
  }
  for (int j = 0; j < a.n_local; ++j) {
    a.xl[j] = reinterpret_cast<float*>(x_ptrs[local_idx[j]]);
    a.yl[j] = y_ptrs.empty() ? nullptr : reinterpret_cast<float*>(y_ptrs[local_idx[j]]);
  }
  for (int p = 0; p < a.world; ++p) {
    a.xw[p] = p < (int)xw_ptrs.size() ? reinterpret_cast<float*>(xw_ptrs[p]) : nullptr;
    a.zw[p] = p < (int)zw_ptrs.size() ? reinterpret_cast<float*>(zw_ptrs[p]) : nullptr;
  }
  if (a.two_shot) {
    if (a.mode == 0) {
      TORCH_CHECK(mc_x != 0 || (int)xw_ptrs.size() == a.world, "two-shot FedAvg needs broadcast targets");
    } else {
      TORCH_CHECK(mc_z != 0 || (int)zw_ptrs.size() == a.world, "two-shot FedProx/ADMM needs peer-mapped z");
    }
  }
  a.mc_x = reinterpret_cast<float*>(mc_x);
  a.mc_y = reinterpret_cast<float*>(mc_y);
  a.mc_z = reinterpret_cast<float*>(mc_z);
  a.z = z.data_ptr<float>();
  a.out = out.data_ptr<float>();
  a.scratch = scratch.data_ptr<float>();
  fill_ctrl(a.ctrl, ctrl_ptrs, a.world);
  a.sync = reinterpret_cast<uint32_t*>(sync.data_ptr<int>());
  a.timeout_cycles = (long long)(timeout_s * 1.9e9);
  a.agg = (int)agg; a.trim_b = (int)trim_b;
  set_dp(a, dp_std, dp_key, dp_t, dp_stats, dp_valid);
  set_q(a, local_idx, q_bits, q_group, q_key, q_t, q_code_ptrs, q_scale_ptrs, q_ef, q_part);
  set_samp(a, samp_S, samp_key, samp_t, client_n);
  set_sa(a, local_idx, sa_frac_bits, sa_clip, sa_keys, sa_t, sa_pay_ptrs, sa_part);
  set_topk(a, topk_k, topk_pay_ptrs, topk_part);
  fb::block_reduce_launch(a, cur_stream());
}

// FedAvg with a server optimizer (FedOpt instantiation of the aggregation kernel): opt = FEDOPT_AVGM .. FEDOPT_YOGI, m / v
// the server state slices (v unused by avgm), mw / vw and mc_m / mc_v their two-shot broadcast targets.
void block_reduce_fedopt(int64_t opt, double lr, double beta1, double beta2, double tau, Tensor m, c10::optional<Tensor> v,
                         std::vector<int64_t> x_ptrs, std::vector<int64_t> local_idx, Tensor z, int64_t n, Tensor out,
                         Tensor scratch, std::vector<int64_t> ctrl_ptrs, Tensor sync, int64_t world, int64_t rank,
                         int64_t mc_x, int64_t mc_m, int64_t mc_v, std::vector<int64_t> xw_ptrs,
                         std::vector<int64_t> mw_ptrs, std::vector<int64_t> vw_ptrs, bool two_shot, int64_t max_blocks,
                         double timeout_s, int64_t agg, int64_t trim_b, double dp_std, int64_t dp_key,
                         c10::optional<Tensor> dp_t, c10::optional<Tensor> dp_stats,
                         c10::optional<Tensor> dp_valid, int64_t q_bits, int64_t q_group, int64_t q_key,
                         c10::optional<Tensor> q_t, std::vector<int64_t> q_code_ptrs, std::vector<int64_t> q_scale_ptrs,
                         std::vector<Tensor> q_ef, c10::optional<Tensor> q_part, int64_t samp_S, int64_t samp_key,
                         c10::optional<Tensor> samp_t, c10::optional<Tensor> client_n, int64_t sa_frac_bits,
                         double sa_clip, c10::optional<Tensor> sa_keys, c10::optional<Tensor> sa_t,
                         std::vector<int64_t> sa_pay_ptrs, c10::optional<Tensor> sa_part, int64_t topk_k,
                         std::vector<int64_t> topk_pay_ptrs, c10::optional<Tensor> topk_part) {
  TORCH_CHECK(opt >= fb::FEDOPT_AVGM && opt <= fb::FEDOPT_YOGI, "block_reduce_fedopt: unknown server optimizer ", opt);
  const bool adaptive = opt != fb::FEDOPT_AVGM;
  CHECK_F32_CUDA(z); CHECK_F32_CUDA(out); CHECK_F32_CUDA(scratch); CHECK_F32_CUDA(m); CHECK_CONTIG(m);
  TORCH_CHECK(out.numel() >= fb::COMM_OUT_FLOATS && scratch.numel() >= fb::COMM_SCRATCH_FLOATS, "out / scratch too small");
  TORCH_CHECK(z.numel() == n && m.numel() == n, "block_reduce_fedopt: z and m must have the block's length");
  if (adaptive) {
    TORCH_CHECK(v.has_value() && v->defined(), "block_reduce_fedopt: adaptive server optimizers need v");
    CHECK_F32_CUDA((*v)); CHECK_CONTIG((*v));
    TORCH_CHECK(v->numel() == n, "block_reduce_fedopt: v must have the block's length");
  }
  c10::cuda::CUDAGuard guard(z.device());
  fb::CommArgs a{};
  a.mode = 0; a.K = (int)x_ptrs.size(); a.n_local = (int)local_idx.size(); a.world = (int)world; a.rank = (int)rank;
  a.n = (int)n; a.two_shot = two_shot ? 1 : 0; a.max_blocks = (int)max_blocks;
  TORCH_CHECK(a.K <= fb::COMM_MAX_K && a.n_local <= fb::COMM_MAX_LOCAL && a.world <= fb::COMM_MAX_WORLD,
              "block_reduce_fedopt: limits exceeded");
  for (int k = 0; k < a.K; ++k) a.x[k] = reinterpret_cast<const float*>(x_ptrs[k]);
  for (int j = 0; j < a.n_local; ++j) a.xl[j] = reinterpret_cast<float*>(x_ptrs[local_idx[j]]);
  for (int p = 0; p < a.world; ++p) {
    a.xw[p] = p < (int)xw_ptrs.size() ? reinterpret_cast<float*>(xw_ptrs[p]) : nullptr;
    a.mw[p] = p < (int)mw_ptrs.size() ? reinterpret_cast<float*>(mw_ptrs[p]) : nullptr;
    a.vw[p] = p < (int)vw_ptrs.size() ? reinterpret_cast<float*>(vw_ptrs[p]) : nullptr;
  }
  if (a.two_shot) {
    TORCH_CHECK(mc_x != 0 || (int)xw_ptrs.size() == a.world, "two-shot FedOpt needs broadcast targets for the weights");
    TORCH_CHECK(mc_m != 0 || (int)mw_ptrs.size() == a.world, "two-shot FedOpt needs peer-mapped m");
    TORCH_CHECK(!adaptive || mc_v != 0 || (int)vw_ptrs.size() == a.world, "two-shot FedOpt needs peer-mapped v");
  }
  a.mc_x = reinterpret_cast<float*>(mc_x);
  a.mc_m = reinterpret_cast<float*>(mc_m);
  a.mc_v = reinterpret_cast<float*>(mc_v);
  a.z = z.data_ptr<float>();
  a.out = out.data_ptr<float>();
  a.scratch = scratch.data_ptr<float>();
  fill_ctrl(a.ctrl, ctrl_ptrs, a.world);
  a.sync = reinterpret_cast<uint32_t*>(sync.data_ptr<int>());
  a.timeout_cycles = (long long)(timeout_s * 1.9e9);
  a.opt = (int)opt;
  a.lr = (float)lr; a.beta1 = (float)beta1; a.beta2 = (float)beta2; a.tau = (float)tau;
  a.m = m.data_ptr<float>();
  a.v = adaptive ? v->data_ptr<float>() : nullptr;
  a.agg = (int)agg; a.trim_b = (int)trim_b;
  set_dp(a, dp_std, dp_key, dp_t, dp_stats, dp_valid);
  set_q(a, local_idx, q_bits, q_group, q_key, q_t, q_code_ptrs, q_scale_ptrs, q_ef, q_part);
  set_samp(a, samp_S, samp_key, samp_t, client_n);
  set_sa(a, local_idx, sa_frac_bits, sa_clip, sa_keys, sa_t, sa_pay_ptrs, sa_part);
  set_topk(a, topk_k, topk_pay_ptrs, topk_part);
  fb::block_reduce_launch(a, cur_stream());
}

// DP-FedAvg update clipping of the local replicas xs against the server model z, bound C; see DPClipArgs.
void dp_clip(std::vector<Tensor> xs, Tensor z, double bound, Tensor stats, int64_t max_blocks) {
  TORCH_CHECK(!xs.empty() && xs.size() <= (size_t)fb::COMM_MAX_LOCAL, "dp_clip: bad replica count");
  CHECK_F32_CUDA(z); CHECK_CONTIG(z); CHECK_F32_CUDA(stats);
  TORCH_CHECK(stats.numel() >= fb::DP_STATS_FLOATS, "dp_clip: stats too small");
  c10::cuda::CUDAGuard guard(z.device());
  fb::DPClipArgs a{};
  a.n = (int)z.numel(); a.n_local = (int)xs.size(); a.max_blocks = (int)max_blocks; a.bound = (float)bound;
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(xs[j]); CHECK_CONTIG(xs[j]);
    TORCH_CHECK(xs[j].numel() == a.n, "dp_clip: block slices must have z's length");
    a.x[j] = fptr_mut(xs[j]);
  }
  a.z = fptr(z);
  a.stats = fptr_mut(stats);
  fb::dp_clip_launch(a, cur_stream());
}

// Top-k selection of the local replicas xs against the server model z, k_sel entries each; see TopKArgs.  pay: the
// replicas' payload slices (int32, at least topk_payload_words(n, k) words, 16-byte aligned); ef: their error-feedback
// slices (empty: off); u: [n_local, >= n] float32 scratch when error feedback is off; ws: int32 workspace of
// topk_ws_ints(n, n_local) words, zero at first use; stats: the aggregation's statistics buffer.
static void check_vec4(const std::vector<Tensor>& ts, const char* name);
int64_t topk_payload_words(int64_t n, int64_t k) { return fb::topk_layout((int)n, (int)k).words; }
int64_t topk_ws_ints(int64_t n, int64_t n_local) { return fb::topk_ws_ints((int)n, (int)n_local); }
void topk_select(std::vector<Tensor> xs, Tensor z, int64_t k, std::vector<Tensor> pay, std::vector<Tensor> ef,
                 c10::optional<Tensor> u, Tensor ws, Tensor stats, int64_t max_blocks) {
  TORCH_CHECK(!xs.empty() && xs.size() <= (size_t)fb::COMM_MAX_LOCAL, "topk_select: 1 to 16 replicas");
  TORCH_CHECK(pay.size() == xs.size() && (ef.empty() || ef.size() == xs.size()),
              "topk_select: one payload (and error-feedback slice) per replica");
  CHECK_F32_CUDA(z); CHECK_CONTIG(z); CHECK_F32_CUDA(stats);
  fb::TopKArgs a{};
  a.n = (int)z.numel(); a.n_local = (int)xs.size(); a.k = (int)k; a.max_blocks = (int)max_blocks;
  TORCH_CHECK(a.n >= 1 && k >= 1 && k <= a.n, "topk_select: needs 1 <= k <= n");
  TORCH_CHECK(stats.numel() >= fb::TOPK_STATS_FLOATS, "topk_select: statistics buffer too small");
  TORCH_CHECK(ws.is_cuda() && ws.scalar_type() == at::kInt && ws.is_contiguous() && ws.numel() >= fb::topk_ws_ints(a.n, a.n_local),
              "topk_select: workspace must be an int32 CUDA tensor of topk_ws_ints(n, n_local) words");
  const int words = fb::topk_layout(a.n, a.k).words;
  if (ef.empty()) {
    TORCH_CHECK(u.has_value() && u->defined(), "topk_select: without error feedback it needs the u scratch");
    CHECK_F32_CUDA((*u)); CHECK_CONTIG((*u));
    TORCH_CHECK(u->dim() == 2 && u->size(0) == a.n_local && u->size(1) >= a.n && u->size(1) % 4 == 0,
                "topk_select: u scratch [n_local, >= n] with rows of a multiple of 4 floats");
  }
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(xs[j]); CHECK_CONTIG(xs[j]);
    TORCH_CHECK(xs[j].numel() == a.n, "topk_select: block slices must have z's length");
    TORCH_CHECK(pay[j].is_cuda() && pay[j].scalar_type() == at::kInt && pay[j].is_contiguous() && pay[j].numel() >= words,
                "topk_select: payload slices must be int32 CUDA tensors of topk_payload_words(n, k) words");
    a.x[j] = fptr(xs[j]);
    a.pay[j] = reinterpret_cast<uint32_t*>(pay[j].data_ptr<int>());
    if (!ef.empty()) {
      CHECK_F32_CUDA(ef[j]); CHECK_CONTIG(ef[j]);
      TORCH_CHECK(ef[j].numel() == a.n, "topk_select: error feedback slices must have the block's length");
      a.ef[j] = fptr_mut(ef[j]);
    } else {
      a.u[j] = fptr_mut(*u) + (int64_t)j * u->size(1);
    }
  }
  a.z = fptr(z);
  a.ws = ws.data_ptr<int>();
  a.stats = fptr_mut(stats);
  check_vec4(xs, "topk_select"); check_vec4(pay, "topk_select"); check_vec4(ef, "topk_select"); check_vec4({z}, "topk_select");
  c10::cuda::CUDAGuard guard(z.device());
  fb::topk_select_launch(a, cur_stream());
}

// SCAFFOLD control variates of the local replicas; see ScaffoldArgs.
static fb::ScaffoldArgs scaffold_args(const std::vector<Tensor>& cs, const Tensor& c, const char* name) {
  TORCH_CHECK(!cs.empty() && cs.size() <= (size_t)fb::COMM_MAX_LOCAL, name, ": 1 to ", fb::COMM_MAX_LOCAL, " replicas");
  CHECK_F32_CUDA(c); CHECK_CONTIG(c);
  fb::ScaffoldArgs a{};
  a.n = (int)c.numel(); a.n_local = (int)cs.size();
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(cs[j]); CHECK_CONTIG(cs[j]);
    TORCH_CHECK(cs[j].numel() == a.n, name, ": every vector must have c's length");
    a.ci[j] = const_cast<float*>(fptr(cs[j]));
  }
  a.c = fptr(c);
  return a;
}
static void check_vec4(const std::vector<Tensor>& ts, const char* name) {
  for (const Tensor& t : ts)
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, name, ": vectors must start at a 16-byte boundary");
}
void scaffold_cv(std::vector<Tensor> cs, std::vector<Tensor> xs, Tensor c, Tensor z, std::vector<double> scales) {
  fb::ScaffoldArgs a = scaffold_args(cs, c, "scaffold_cv");
  TORCH_CHECK(xs.size() == cs.size() && scales.size() == cs.size(), "scaffold_cv: one x and one scale per c_i");
  CHECK_F32_CUDA(z); CHECK_CONTIG(z);
  TORCH_CHECK(z.numel() == a.n, "scaffold_cv: every vector must have c's length");
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(xs[j]); CHECK_CONTIG(xs[j]);
    TORCH_CHECK(xs[j].numel() == a.n, "scaffold_cv: every vector must have c's length");
    a.x[j] = fptr(xs[j]);
    a.scale[j] = (float)scales[j];
  }
  a.z = fptr(z);
  check_vec4(cs, "scaffold_cv"); check_vec4(xs, "scaffold_cv"); check_vec4({c, z}, "scaffold_cv");
  c10::cuda::CUDAGuard guard(c.device());
  fb::scaffold_cv_launch(a, cur_stream());
}
int64_t scaffold_corr_blocks(int64_t n) { return fb::scaffold_corr_blocks((int)n); }
void scaffold_corr(std::vector<Tensor> cs, std::vector<Tensor> ds, Tensor c, Tensor norm_sq, Tensor ws, Tensor tickets) {
  fb::ScaffoldArgs a = scaffold_args(cs, c, "scaffold_corr");
  TORCH_CHECK(ds.size() == cs.size(), "scaffold_corr: one d_i per c_i");
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(ds[j]); CHECK_CONTIG(ds[j]);
    TORCH_CHECK(ds[j].numel() == a.n, "scaffold_corr: every vector must have c's length");
    a.d[j] = fptr_mut(ds[j]);
  }
  CHECK_F32_CUDA(norm_sq); CHECK_F32_CUDA(ws);
  TORCH_CHECK(tickets.is_cuda() && tickets.scalar_type() == torch::kInt32, "scaffold_corr: tickets must be CUDA int32");
  TORCH_CHECK(norm_sq.numel() >= a.n_local && tickets.numel() >= a.n_local &&
                  ws.numel() >= (int64_t)a.n_local * fb::scaffold_corr_blocks(a.n),
              "scaffold_corr: norm_sq / tickets need one entry per replica, ws n_local * scaffold_corr_blocks(n) floats");
  check_vec4(cs, "scaffold_corr"); check_vec4(ds, "scaffold_corr"); check_vec4({c}, "scaffold_corr");
  a.ws = fptr_mut(ws);
  a.tickets = reinterpret_cast<unsigned int*>(tickets.data_ptr<int>());
  a.norm_sq = fptr_mut(norm_sq);
  c10::cuda::CUDAGuard guard(c.device());
  fb::scaffold_corr_launch(a, cur_stream());
}

// Barzilai-Borwein update (consensus_multi.py:242-278) as one kernel; see BBArgs.
void bb_update(std::vector<Tensor> xs, std::vector<Tensor> ys, std::vector<Tensor> yhat0s, std::vector<Tensor> x0s, Tensor z,
               std::vector<int64_t> workers, int64_t K, Tensor rho_dev, Tensor log, Tensor scratch, Tensor out,
               std::vector<int64_t> ctrl_ptrs, Tensor sync, int64_t world, int64_t rank, double epsilon, double alphacorrmin,
               double rhomax, bool seed_only, int64_t max_blocks, double timeout_s) {
  TORCH_CHECK(!xs.empty() && xs.size() == x0s.size() && xs.size() <= (size_t)fb::COMM_MAX_LOCAL, "bb_update: bad replica count");
  CHECK_F32_CUDA(z); CHECK_F32_CUDA(rho_dev); CHECK_F32_CUDA(log); CHECK_F32_CUDA(scratch);
  TORCH_CHECK(log.numel() >= 8 * K && scratch.numel() >= fb::BB_SCRATCH_FLOATS, "bb_update: log / scratch too small");
  c10::cuda::CUDAGuard guard(z.device());
  fb::BBArgs a{};
  a.K = (int)K; a.n_local = (int)xs.size(); a.world = (int)world; a.rank = (int)rank; a.n = (int)xs[0].numel();
  a.seed_only = seed_only ? 1 : 0; a.max_blocks = (int)max_blocks;
  a.epsilon = (float)epsilon; a.alphacorrmin = (float)alphacorrmin; a.rhomax = (float)rhomax;
  for (int j = 0; j < a.n_local; ++j) {
    CHECK_F32_CUDA(xs[j]); CHECK_CONTIG(xs[j]); CHECK_CONTIG(x0s[j]);
    TORCH_CHECK(xs[j].numel() == a.n && x0s[j].numel() == a.n, "bb_update: equal lengths required");
    a.x[j] = fptr(xs[j]);
    a.x0[j] = fptr_mut(x0s[j]);
    if (!seed_only) {
      CHECK_CONTIG(ys[j]); CHECK_CONTIG(yhat0s[j]);
      a.y[j] = fptr(ys[j]);
      a.yhat0[j] = fptr_mut(yhat0s[j]);
    }
    a.worker[j] = (int)workers[j];
  }
  a.z = fptr(z);
  a.rho_dev = fptr_mut(rho_dev);
  a.log = fptr_mut(log);
  a.scratch = fptr_mut(scratch);
  a.out = fptr_mut(out);
  fill_ctrl(a.ctrl, ctrl_ptrs, a.world);
  a.sync = reinterpret_cast<uint32_t*>(sync.data_ptr<int>());
  a.timeout_cycles = (long long)(timeout_s * 1.9e9);
  fb::bb_update_launch(a, cur_stream());
}

// ---------------------------------------------------------------------------------------------- CUDA IPC helpers
// Fallback symmetric-memory transport when torch's symmetric memory is unavailable: plain cudaMalloc'ed arenas
// exported/imported with CUDA IPC handles (exchanged through the torch.distributed store by the Python side).
py::bytes ipc_get_handle(int64_t ptr) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(ptr));
  TORCH_CHECK(e == cudaSuccess, "cudaIpcGetMemHandle: ", cudaGetErrorString(e));
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}
int64_t ipc_open_handle(py::bytes handle) {
  std::string s = handle;
  TORCH_CHECK(s.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  cudaIpcMemHandle_t h;
  memcpy(&h, s.data(), sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  TORCH_CHECK(e == cudaSuccess, "cudaIpcOpenMemHandle: ", cudaGetErrorString(e));
  return reinterpret_cast<int64_t>(p);
}
void ipc_close_handle(int64_t ptr) { cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr)); }

int64_t launch_count() { return (int64_t)fb::launch_count(); }

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "federated_pytorch_test_b200: hand-written sm_90a kernels";
  m.def("launch_count", &launch_count);
  m.def("adam_prox", &adam_prox);
  m.def("sgd_prox", &sgd_prox);
  m.def("grad_norm_blocks", &grad_norm_blocks);
  m.def("grad_norm", &grad_norm);
  m.def("scaffold_cv", &scaffold_cv);
  m.def("scaffold_corr_blocks", &scaffold_corr_blocks);
  m.def("scaffold_corr", &scaffold_corr);
  m.def("bump_step", &bump_step);
  m.def("l1_l2", &l1_l2);
  m.def("make_pair", &make_pair);
  m.def("welford", &welford);
  m.def("penalty_value", &penalty_value);
  m.def("penalty_grad", &penalty_grad);
  m.def("multi_dot", &multi_dot);
  m.def("lbfgs_two_loop", &lbfgs_two_loop);
  m.def("normalize_u8", &normalize_u8);
  m.def("augment_normalize_u8", &augment_normalize_u8, py::arg("u8"), py::arg("rows"), py::arg("key"), py::arg("counter"),
        py::arg("mean"), py::arg("std"), py::arg("to_nchw"));
  m.def("mix_normalize_u8", &mix_normalize_u8, py::arg("u8"), py::arg("rows"), py::arg("augment"), py::arg("key"),
        py::arg("counter"), py::arg("mean"), py::arg("std"), py::arg("to_nchw"), py::arg("cutmix"), py::arg("lam_f"),
        py::arg("mlam_f"), py::arg("y0"), py::arg("y1"), py::arg("x0"), py::arg("x1"), py::arg("lam_eff"));
  m.def("col_stats", &col_stats);
  m.def("head_fwd", &head_fwd);
  m.def("head_bwd", &head_bwd);
  m.def("bn_elu_fwd", &bn_elu_fwd, py::arg("y"), py::arg("stats"), py::arg("gamma"), py::arg("beta"), py::arg("residual"),
        py::arg("running_mean"), py::arg("running_var"), py::arg("eps"), py::arg("momentum"), py::arg("act"),
        py::arg("self_clean"), py::arg("use_running") = false);
  m.def("bn_elu_bwd", &bn_elu_bwd);
  m.def("stem_conv_supported", &stem_conv_supported);
  m.def("stem_conv_bn", &stem_conv_bn, py::arg("x"), py::arg("w"), py::arg("stats"), py::arg("mode"), py::arg("gamma") = py::none(),
        py::arg("beta") = py::none(), py::arg("running_mean") = py::none(), py::arg("running_var") = py::none(),
        py::arg("eps") = 1e-5, py::arg("momentum") = 0.1, py::arg("act") = true, py::arg("self_clean") = false);
  m.def("gn_elu_fwd", &gn_elu_fwd, py::arg("y"), py::arg("gamma"), py::arg("beta"), py::arg("residual"), py::arg("groups"),
        py::arg("eps"), py::arg("act"));
  m.def("gn_elu_bwd", &gn_elu_bwd, py::arg("dout"), py::arg("out"), py::arg("y"), py::arg("mean"), py::arg("rstd"),
        py::arg("gamma"), py::arg("beta"), py::arg("groups"), py::arg("want_dres"), py::arg("act"), py::arg("want_affine"));
  m.def("avgpool_nhwc", &avgpool_nhwc);
  m.def("avgpool_nhwc_bwd", &avgpool_nhwc_bwd);
  m.def("weight_flip", &weight_flip);
  m.def("convT_pack", &convT_pack);
  m.def("linear_tf32", &linear_tf32);
  m.def("conv_supported", &conv_supported);
  m.def("conv_orientation", &conv_orientation);
  m.def("conv_window_reuse", &conv_window_reuse, py::arg("H_out"), py::arg("W_out"), py::arg("C_in"), py::arg("C_out"), py::arg("kh"),
        py::arg("stride") = 1, py::arg("dil") = 1);
  m.def("conv2d_nhwc", &conv2d_nhwc, py::arg("x"), py::arg("w"), py::arg("stats"), py::arg("stride"), py::arg("pad"), py::arg("dil"),
        py::arg("orient") = -1);
  m.def("conv2d_nhwc_sized", &conv2d_nhwc_sized);
  m.def("conv2d_nhwc_bias_act", &conv2d_nhwc_bias_act);
  m.def("conv2d_nhwc_bn_eval", &conv2d_nhwc_bn_eval);
  m.def("conv2d_nhwc_shuffle", &conv2d_nhwc_shuffle);
  m.def("conv_shuffle_supported", &conv_shuffle_supported);
  m.def("conv2d_nhwc_multidil", &conv2d_nhwc_multidil);
  m.def("conv_multidil_supported", &conv_multidil_supported);
  m.def("conv_wgrad", &conv_wgrad);
  m.def("conv_wgrad_supported", &conv_wgrad_supported);
  m.def("cross_entropy_fwd", &cross_entropy_fwd);
  m.def("cross_entropy_bwd", &cross_entropy_bwd);
  m.def("soft_ce_fwd", &soft_ce_fwd, py::arg("logits"), py::arg("labels"), py::arg("lam"), py::arg("eps"));
  m.def("soft_ce_bwd", &soft_ce_bwd, py::arg("probs"), py::arg("labels"), py::arg("lam"), py::arg("eps"), py::arg("gout"));
  m.def("vae_loss_fwd", &vae_loss_fwd);
  m.def("vae_loss_bwd", &vae_loss_bwd);
  m.def("linear_f32", &linear_f32);
  m.def("linear_f32_dgrad", &linear_f32_dgrad);
  m.def("linear_f32_wgrad", &linear_f32_wgrad);
  m.def("act_bwd_bias", &act_bwd_bias);
  m.def("maxpool2x2_fwd", &maxpool2x2_fwd);
  m.def("maxpool2x2_bwd", &maxpool2x2_bwd);
  m.def("argmax_count", &argmax_count);
  m.def("info_nce_max_p", &info_nce_max_p);
  m.def("info_nce_scratch_floats", &info_nce_scratch_floats);
  m.def("info_nce_fwd", &info_nce_fwd);
  m.def("info_nce_bwd", &info_nce_bwd);
  m.def("gauss_nll_rows_fwd", &gauss_nll_rows_fwd);
  m.def("gauss_nll_rows_bwd", &gauss_nll_rows_bwd);
  m.def("smallconv_supported", &smallconv_supported);
  m.def("smallconv_fwd", &smallconv_fwd);
  m.def("smallconv_unpool_actbwd", &smallconv_unpool_actbwd);
  m.def("smallconv_dgrad", &smallconv_dgrad);
  m.def("smallconv_wgrad", &smallconv_wgrad);
  m.def("block_reduce", &block_reduce);
  m.def("block_reduce_fedopt", &block_reduce_fedopt);
  m.def("dp_clip", &dp_clip);
  m.def("topk_select", &topk_select);
  m.def("topk_payload_words", &topk_payload_words);
  m.def("topk_ws_ints", &topk_ws_ints);
  m.def("bb_update", &bb_update);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close_handle", &ipc_close_handle);
}

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
               c10::optional<Tensor> rho_dev) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x); CHECK_CONTIG(g); CHECK_CONTIG(m); CHECK_CONTIG(v);
  c10::cuda::CUDAGuard guard(x.device());
  fb::adam_prox(fptr_mut(x), fptr(g), fptr_mut(m), fptr_mut(v), step.data_ptr<int>(), (int)x.numel(), (float)lr, (float)b1,
                (float)b2, (float)eps, opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, cur_stream(), opt_ptr(rho_dev));
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
std::vector<Tensor> make_pair(Tensor g, Tensor gprev, Tensor d, double t, double trust) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_CONTIG(gprev); CHECK_CONTIG(d);
  c10::cuda::CUDAGuard guard(g.device());
  auto y = torch::empty_like(g), s = torch::empty_like(g);
  auto out = torch::empty({3}, g.options());
  fb::make_pair(fptr(g), fptr(gprev), fptr(d), (float)t, (float)trust, fptr_mut(y), fptr_mut(s), (int)g.numel(), fptr_mut(out), cur_stream());
  return {y, s, out};
}
Tensor welford(Tensor g, Tensor mean, Tensor m2, int64_t n_iter) {
  CHECK_F32_CUDA(g);
  c10::cuda::CUDAGuard guard(g.device());
  auto out = torch::empty({1}, g.options());
  fb::welford(fptr(g), fptr_mut(mean), fptr_mut(m2), (int)g.numel(), 1.0f / (float)n_iter, fptr_mut(out), cur_stream());
  return out;
}
Tensor penalty_value(Tensor x, c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2) {
  CHECK_F32_CUDA(x); CHECK_CONTIG(x);
  c10::cuda::CUDAGuard guard(x.device());
  auto out = torch::empty({1}, x.options());
  fb::penalty_value(fptr(x), opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, (int)x.numel(), fptr_mut(out), cur_stream());
  return out;
}
void penalty_grad(Tensor g, Tensor x, c10::optional<Tensor> z, c10::optional<Tensor> y, double rho, double l1, double l2) {
  CHECK_F32_CUDA(g); CHECK_CONTIG(g); CHECK_CONTIG(x);
  c10::cuda::CUDAGuard guard(g.device());
  fb::penalty_grad(fptr_mut(g), fptr(x), opt_ptr(z), opt_ptr(y), (float)rho, (float)l1, (float)l2, (int)g.numel(), cur_stream());
}
Tensor multi_dot(std::vector<Tensor> a, std::vector<Tensor> b) {
  TORCH_CHECK(a.size() == b.size() && !a.empty() && a.size() <= 8, "multi_dot: 1..8 pairs");
  c10::cuda::CUDAGuard guard(a[0].device());
  std::vector<const float*> pa, pb;
  for (size_t i = 0; i < a.size(); ++i) {
    CHECK_F32_CUDA(a[i]); CHECK_CONTIG(a[i]); CHECK_CONTIG(b[i]);
    TORCH_CHECK(a[i].numel() == a[0].numel() && b[i].numel() == a[0].numel(), "multi_dot: equal lengths required");
    pa.push_back(fptr(a[i])); pb.push_back(fptr(b[i]));
  }
  auto out = torch::empty({(int64_t)a.size()}, a[0].options());
  fb::multi_dot(pa.data(), pb.data(), (int)a.size(), (int)a[0].numel(), fptr_mut(out), cur_stream());
  return out;
}
Tensor lbfgs_two_loop(Tensor Y, Tensor S, Tensor order, Tensor g, double hdiag) {
  CHECK_F32_CUDA(Y); CHECK_CONTIG(Y); CHECK_CONTIG(S); CHECK_CONTIG(g);
  TORCH_CHECK(order.scalar_type() == torch::kInt32 && order.is_cuda(), "order must be a CUDA int32 tensor");
  c10::cuda::CUDAGuard guard(g.device());
  const int k = (int)order.numel(), n = (int)g.numel();
  auto d = torch::empty_like(g);
  auto work = torch::empty({(int64_t)fb::lbfgs_two_loop_work_floats(k)}, g.options());
  fb::lbfgs_two_loop(fptr(Y), fptr(S), order.data_ptr<int>(), k, n, (int)Y.size(1), fptr(g), (float)hdiag, fptr_mut(d), fptr_mut(work), cur_stream());
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
void col_stats(Tensor y, Tensor stats) {
  CHECK_F32_CUDA(y); CHECK_CONTIG(y);
  c10::cuda::CUDAGuard guard(y.device());
  const int C = (int)y.size(-1);
  fb::col_stats(fptr(y), fptr_mut(stats), (int)(y.numel() / C), C, cur_stream());
}
// y, out: [M, C] views of NHWC tensors.  Returns (out, save_mean, save_invstd).
std::vector<Tensor> bn_elu_fwd(Tensor y, Tensor stats, Tensor gamma, Tensor beta, c10::optional<Tensor> residual,
                               c10::optional<Tensor> running_mean, c10::optional<Tensor> running_var, double eps,
                               double momentum, bool act, bool self_clean) {
  CHECK_F32_CUDA(y); CHECK_CONTIG(y);
  c10::cuda::CUDAGuard guard(y.device());
  const int C = (int)y.size(-1);
  const int M = (int)(y.numel() / C);
  auto out = torch::empty_like(y);
  auto sm = torch::empty({C}, y.options()), si = torch::empty({C}, y.options());
  float* rm = (running_mean.has_value() && running_mean->defined()) ? running_mean->data_ptr<float>() : nullptr;
  float* rv = (running_var.has_value() && running_var->defined()) ? running_var->data_ptr<float>() : nullptr;
  TORCH_CHECK(stats.numel() >= 2 * C + (self_clean ? 1 : 0), "stats buffer too small");
  fb::bn_elu_fwd(fptr(y), fptr_mut(stats), fptr(gamma), fptr(beta), opt_ptr(residual), fptr_mut(out), rm, rv, fptr_mut(sm),
                 fptr_mut(si), M, C, (float)eps, (float)momentum, act ? 1 : 0, self_clean ? 1 : 0, cur_stream());
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
  static const bool fused_optin = [] { const char* e = std::getenv("FEDB200_BN_BWD_FUSED"); return e != nullptr && std::atoi(e) != 0; }();
  const bool persistent = !fused_optin && sums_buf.has_value() && sums_buf->defined();   // the opt-in fused kernel zeroes its own scratch
  if (persistent) TORCH_CHECK(sums_buf->numel() == 2 * C + 1 && sums_buf->is_contiguous(), "bn_elu_bwd: sums buffer must be [2C + 1]");
  auto sums = persistent ? *sums_buf : torch::empty({2 * C + 1}, y.options());
  auto dy = torch::empty_like(y);
  Tensor dres;
  if (want_dres) dres = torch::empty_like(y);
  float* dg = (dgamma.has_value() && dgamma->defined()) ? dgamma->data_ptr<float>() : nullptr;
  float* db = (dbeta.has_value() && dbeta->defined()) ? dbeta->data_ptr<float>() : nullptr;
  if (fused_optin && fb::bn_elu_bwd_fused(fptr(dout), outp, fptr(y), fptr(mean), fptr(invstd), fptr(gamma), betap, fptr_mut(sums),
                                          fptr_mut(dy), want_dres ? dres.data_ptr<float>() : nullptr, dg, db, M, C, act ? 1 : 0,
                                          cur_stream()))
    return {dy, dres};
  fb::bn_elu_bwd_reduce(fptr(dout), outp, fptr(y), fptr(mean), fptr(invstd), fptr(gamma), betap, fptr_mut(sums), M, C,
                        act ? 1 : 0, persistent ? 1 : 0, cur_stream());
  fb::bn_elu_bwd_apply(fptr(dout), outp, fptr(y), fptr(mean), fptr(invstd), fptr(gamma), betap, fptr_mut(sums), fptr_mut(dy),
                       want_dres ? dres.data_ptr<float>() : nullptr, dg, db, M, C, act ? 1 : 0, persistent ? 1 : 0, cur_stream());
  return {dy, dres};
}
// fused classifier head (experimental): x [N,H,W,C], w [O,C], bias [O] -> (logits [N,O], pooled [N,C])
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
// x: [N,H,W,Ci] contiguous; w: [Co,kh,kw,Ci] contiguous.  Returns y [N,Ho,Wo,Co]; stats (2*Co) accumulated if given.
Tensor conv2d_nhwc(Tensor x, Tensor w, c10::optional<Tensor> stats, int64_t stride, int64_t pad, int64_t dil) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_CONTIG(x); CHECK_CONTIG(w);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  const int Ho = (H + 2 * (int)pad - (int)dil * (kh - 1) - 1) / (int)stride + 1;
  const int Wo = (W + 2 * (int)pad - (int)dil * (kw - 1) - 1) / (int)stride + 1;
  auto y = torch::empty({NB, Ho, Wo, Co}, x.options());
  float* st = (stats.has_value() && stats->defined()) ? stats->data_ptr<float>() : nullptr;
  fb::conv2d_nhwc_tf32(fptr(x), fptr(w), fptr_mut(y), st, NB, H, W, Ci, Co, kh, kw, (int)stride, (int)pad, (int)dil, Ho, Wo, cur_stream());
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

// y += conv(x, w), in place (experimental)
Tensor conv2d_nhwc_accumulate(Tensor x, Tensor w, Tensor y, int64_t stride, int64_t pad, int64_t dil) {
  CHECK_F32_CUDA(x); CHECK_F32_CUDA(w); CHECK_F32_CUDA(y); CHECK_CONTIG(x); CHECK_CONTIG(w); CHECK_CONTIG(y);
  TORCH_CHECK(x.dim() == 4 && w.dim() == 4 && y.dim() == 4 && x.size(3) == w.size(3), "conv2d_nhwc_accumulate: x [N,H,W,Ci], w [Co,kh,kw,Ci]");
  c10::cuda::CUDAGuard guard(x.device());
  const int NB = (int)x.size(0), H = (int)x.size(1), W = (int)x.size(2), Ci = (int)x.size(3);
  const int Co = (int)w.size(0), kh = (int)w.size(1), kw = (int)w.size(2);
  const int Ho = (H + 2 * (int)pad - (int)dil * (kh - 1) - 1) / (int)stride + 1;
  const int Wo = (W + 2 * (int)pad - (int)dil * (kw - 1) - 1) / (int)stride + 1;
  TORCH_CHECK(y.size(0) == NB && y.size(1) == Ho && y.size(2) == Wo && y.size(3) == Co, "conv2d_nhwc_accumulate: y must be [N,Ho,Wo,Co]");
  fb::conv2d_nhwc_accumulate_tf32(fptr(x), fptr(w), fptr_mut(y), NB, H, W, Ci, Co, kh, kw, (int)stride, (int)pad, (int)dil, Ho, Wo,
                                  cur_stream());
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
static void fill_ctrl(uint32_t** dst, const std::vector<int64_t>& ctrl_ptrs, int world) {
  for (int p = 0; p < world && p < (int)ctrl_ptrs.size(); ++p) dst[p] = reinterpret_cast<uint32_t*>(ctrl_ptrs[p]);
}
void block_reduce(int64_t mode, std::vector<int64_t> x_ptrs, std::vector<int64_t> y_ptrs, std::vector<int64_t> local_idx,
                  Tensor z, int64_t n, double rho, c10::optional<Tensor> rho_dev, Tensor out, Tensor scratch,
                  std::vector<int64_t> ctrl_ptrs, Tensor sync, int64_t world, int64_t rank, int64_t mc_x, int64_t mc_y,
                  int64_t mc_z, std::vector<int64_t> xw_ptrs, std::vector<int64_t> zw_ptrs, bool two_shot,
                  int64_t max_blocks, double timeout_s) {
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
  fb::block_reduce_launch(a, cur_stream());
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
  m.def("bump_step", &bump_step);
  m.def("l1_l2", &l1_l2);
  m.def("make_pair", &make_pair);
  m.def("welford", &welford);
  m.def("penalty_value", &penalty_value);
  m.def("penalty_grad", &penalty_grad);
  m.def("multi_dot", &multi_dot);
  m.def("lbfgs_two_loop", &lbfgs_two_loop);
  m.def("normalize_u8", &normalize_u8);
  m.def("col_stats", &col_stats);
  m.def("head_fwd", &head_fwd);
  m.def("head_bwd", &head_bwd);
  m.def("bn_elu_fwd", &bn_elu_fwd);
  m.def("bn_elu_bwd", &bn_elu_bwd);
  m.def("avgpool_nhwc", &avgpool_nhwc);
  m.def("avgpool_nhwc_bwd", &avgpool_nhwc_bwd);
  m.def("weight_flip", &weight_flip);
  m.def("convT_pack", &convT_pack);
  m.def("linear_tf32", &linear_tf32);
  m.def("conv_supported", &conv_supported);
  m.def("conv2d_nhwc", &conv2d_nhwc);
  m.def("conv2d_nhwc_sized", &conv2d_nhwc_sized);
  m.def("conv2d_nhwc_bias_act", &conv2d_nhwc_bias_act);
  m.def("conv2d_nhwc_accumulate", &conv2d_nhwc_accumulate);
  m.def("conv2d_nhwc_shuffle", &conv2d_nhwc_shuffle);
  m.def("conv_shuffle_supported", &conv_shuffle_supported);
  m.def("conv2d_nhwc_multidil", &conv2d_nhwc_multidil);
  m.def("conv_multidil_supported", &conv_multidil_supported);
  m.def("conv_wgrad", &conv_wgrad);
  m.def("conv_wgrad_supported", &conv_wgrad_supported);
  m.def("cross_entropy_fwd", &cross_entropy_fwd);
  m.def("cross_entropy_bwd", &cross_entropy_bwd);
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
  m.def("bb_update", &bb_update);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close_handle", &ipc_close_handle);
}

// Training extras next to the ray path (SURVEY.md 8(f) row f3), per-element routines shared by the CUDA kernels
// (csrc/nr_losses.cu) and the host build of tests/cpu_harness/loss_cpu_harness.cu:
//   depth_mean_point   NeuralRayGenRenderer.predict_mean_for_depth_loss   reference network/renderer.py:280-316
//                      (interpolate_feature_map + dist_decoder.predict_mean of the coarse and the fine decoder), fwd + bwd
//   render_loss_*      RenderLoss       network/loss.py:46-76
//   depth_loss_*       DepthLoss        network/loss.py:78-132
//   consist_loss_*     ConsistencyLoss  network/loss.py:17-44
#pragma once
#include "nr_train_math.cuh"

namespace nr {
namespace ls {

using tr::atomic_add;
using tr::head_bwd;
using tr::head_fwd;
using tr::softplus_f;
using tr::softplus_g;

// ---- predict_mean_for_depth_loss ----------------------------------------------------------------------------------------
typedef NrDepthMeanParams DepthMeanP;   // include/neuray_b200.h

// point i = (view, coordinate): gather the view's ray_feats, run the mean head (Linear 32 ELU Linear 32 ELU Linear 2 Softplus,
// dist_decoder.py:64-71) of decoder 0 (coarse) and 1 (fine, optional); with d_mean also the backward: weight gradients are
// added to d_w_point[k] in the packed w_point layout, the map gradient to d_map.
NR_HD void depth_mean_point(const DepthMeanP& p, long long i) {
  const int view = int(i / p.pn);
  const int fh = p.fh, fw = p.fw;
  const float* map = p.map + (size_t)view * 32 * fh * fw;
  const Taps t = border_taps(p.coords[2 * i], p.coords[2 * i + 1], p.h, p.w, fh, fw, fh == p.h && fw == p.w);
  float rf[32];
  for (int k = 0; k < 32; ++k) rf[k] = bilinear(map + (size_t)k * fh * fw, fw, t);
  float drf[32];
  for (int k = 0; k < 32; ++k) drf[k] = 0.f;
  bool any_grad = false;
  for (int d = 0; d < 2; ++d) {
    if (p.w_point[d] == nullptr) continue;
    const float* Wh = p.w_point[d] + lay::DD_HEAD;   // head 0 = mean decoder
    float h1[32], h2[32], ho[2], mean[2];
    head_fwd(Wh, rf, h1, h2, ho, nullptr, 0, 0);
    for (int o = 0; o < 2; ++o) {
      mean[o] = softplus_f(ho[o]);
      if (p.mean[d] != nullptr) p.mean[d][2 * i + o] = mean[o];
    }
    if (p.d_mean[d] == nullptr) continue;
    any_grad = true;
    float dho[2];
    for (int o = 0; o < 2; ++o) dho[o] = p.d_mean[d][2 * i + o] * softplus_g(mean[o]);
    head_bwd(Wh, rf, h1, h2, dho, drf, p.d_w_point[d] + lay::DD_HEAD, nullptr, 0, 0);
  }
  if (any_grad && p.d_map != nullptr) {
    const int off[4] = {t.y0 * fw + t.x0, t.y0 * fw + t.x1, t.y1 * fw + t.x0, t.y1 * fw + t.x1};
    float* dm = p.d_map + (size_t)view * 32 * fh * fw;
    for (int k = 0; k < 32; ++k)
      for (int q = 0; q < 4; ++q) atomic_add(dm + (size_t)k * fh * fw + off[q], drf[k] * t.w[q]);
  }
}

// ---- RenderLoss (loss.py:58-66): sum_c (pr - gt)^2 per ray; masked mean with +1e-3 in the denominator, or plain mean --------
NR_HD float render_loss_term(const float* pr, const float* gt, long long r) {
  float s = 0.f;
  for (int c = 0; c < 3; ++c) { const float d = pr[3 * r + c] - gt[3 * r + c]; s += d * d; }
  return s;
}

// ---- DepthLoss (loss.py:92-127) ---------------------------------------------------------------------------------------------
typedef NrDepthLossParams DepthLossP;
// ground-truth depth of coordinate i of a view, in the normalised inverse-depth coordinate the decoder's mean lives in
NR_HD float depth_process(float depth, float near, float far) {
  depth = fmaxf(depth, 1e-5f);
  const float a = -1.f / near, b = -1.f / far;
  depth = (-1.f / depth - a) / (b - a);
  return fminf(fmaxf(depth, 0.f), 1.f);
}
NR_HD float depth_at(const float* map, const float* coords, long long i, int h, int w) {
  return bilinear(map, w, border_taps(coords[2 * i], coords[2 * i + 1], h, w, h, w, true));
}
// loss term and its derivative with respect to the prediction; mask (1 unless the 'gso' consistency mask applies)
NR_HD void depth_loss_term(const DepthLossP& p, long long i, const float* depth_pr, float& term, float& dterm, float& mask) {
  const int view = int(i / p.pn);
  const float near = p.depth_range[2 * view], far = p.depth_range[2 * view + 1];
  const float gt = depth_process(depth_at(p.true_depth + (size_t)view * p.h * p.w, p.coords, i, p.h, p.w), near, far);
  const float pr = depth_pr[i];
  const float d = gt - pr;
  if (p.loss_type == 0) { term = d * d; dterm = -2.f * d; }
  else {        // nn.SmoothL1Loss(beta): |d| < beta ? 0.5 d^2 / beta : |d| - 0.5 beta   (input = gt, target = pr, symmetric)
    const float ad = fabsf(d);
    if (ad < p.beta) { term = 0.5f * d * d / p.beta; dterm = -d / p.beta; }
    else { term = ad - 0.5f * p.beta; dterm = d > 0.f ? -1.f : 1.f; }
  }
  mask = 1.f;
  if (p.aug_depth != nullptr) {
    const float aug = depth_process(depth_at(p.aug_depth + (size_t)view * p.h * p.w, p.coords, i, p.h, p.w), near, far);
    mask = fabsf(aug - gt) < p.correct_thresh ? 1.f : 0.f;
  }
}

// ---- ConsistencyLoss (loss.py:30-43): cross entropy between the rendered (detached) and the decoder's own hit probability ---
NR_HD float consist_term(float p0, float p1) { return -p0 * logf(p1 + 1e-5f) - (1.f - p0) * logf(1.f - p1 + 1e-5f); }
NR_HD float consist_dterm(float p0, float p1) { return -p0 / (p1 + 1e-5f) + (1.f - p0) / (1.f - p1 + 1e-5f); }

}  // namespace ls
}  // namespace nr

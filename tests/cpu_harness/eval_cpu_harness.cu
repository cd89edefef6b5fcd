// Test infrastructure: the per-pixel routines of eval.py's PSNR / SSIM (csrc/nr_metrics_math.cuh) on the HOST, with the
// Gaussian window sums and reductions of csrc/nr_metrics.cu written as plain 2-D loops, so that tests/test_eval_metrics.py
// can check them against the float64 restatement without a GPU.  Not part of the product library.
#include <vector>

#include "../../neuray_b200/csrc/nr_metrics_math.cuh"

using namespace nr::mt;

extern "C" int nr_cpu_unit(const uint8_t* v, long long n, float* out) {
  for (long long i = 0; i < n; ++i) out[i] = unit(v[i]);
  return 0;
}

extern "C" int nr_cpu_gauss_window(double* g) {
  double w[2 * HALF + 1];
  gauss_window(w);
  for (int i = 0; i <= 2 * HALF; ++i) g[i] = w[i];
  return 0;
}

// one pair of uint8 [h,w,3] images: out[2] = {psnr, ssim}, as nr_eval_metrics writes them
extern "C" int nr_cpu_eval_metrics(const uint8_t* gt, const uint8_t* pr, int h, int w, double* out) {
  if (h < 11 || w < 11) return -1;
  double g[2 * HALF + 1];
  gauss_window(g);
  std::vector<double> x((size_t)h * w), y((size_t)h * w);
  double sse = 0.0, ssim = 0.0;
  for (int k = 0; k < 3; ++k) {
    for (long long i = 0; i < (long long)h * w; ++i) {
      x[i] = unit(gt[3 * i + k]);
      y[i] = unit(pr[3 * i + k]);
      sse += (x[i] - y[i]) * (x[i] - y[i]);
    }
    for (int i = HALF; i < h - HALF; ++i)
      for (int j = HALF; j < w - HALF; ++j) {
        double s[4] = {0.0, 0.0, 0.0, 0.0};
        for (int a = -HALF; a <= HALF; ++a)
          for (int b = -HALF; b <= HALF; ++b) {
            const double wt = g[a + HALF] * g[b + HALF];
            const double u = x[(i + a) * w + j + b], v = y[(i + a) * w + j + b];
            s[0] += wt * u; s[1] += wt * v; s[2] += wt * mul_rn(u, v); s[3] += wt * (mul_rn(u, u) + mul_rn(v, v));
          }
        ssim += tf_ssim_term(s[0], s[1], s[2], s[3]);
      }
  }
  const double mse = sse / (3.0 * h * w);
  out[0] = mse == 0.0 ? INFINITY : 10.0 * log10(1.0 / mse);
  out[1] = ssim / (3.0 * (h - 2 * HALF) * (w - 2 * HALF));
  return 0;
}

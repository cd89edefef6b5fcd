// Test infrastructure: the per-pixel routines of csrc/nr_metrics_math.cuh on the HOST, with the window sums and reductions of
// csrc/nr_metrics.cu written as plain loops, so that tests/test_metrics.py can check them against the float64 restatement
// without a GPU.  Not part of the product library.
#include <vector>

#include "../../neuray_b200/csrc/nr_metrics_math.cuh"

using namespace nr::mt;

extern "C" int nr_cpu_quantise(const float* x, long long n, uint8_t* q) {
  for (long long i = 0; i < n; ++i) q[i] = (uint8_t)quantise(x[i]);
  return 0;
}

// one prediction: out[4] = {sse_r, sse_g, sse_b, ssim}, as nr_image_metrics writes them
extern "C" int nr_cpu_image_metrics(const float* gt, const float* pr, int h, int w, int margin_h, int margin_w, double* out) {
  const int ch = h - 2 * margin_h, cw = w - 2 * margin_w;
  if (ch < 11 || cw < 11) return -1;
  std::vector<int> x(ch * cw), y(ch * cw);
  double mean[3];
  for (int k = 0; k < 3; ++k) {
    long long sse = 0;
    for (int i = 0; i < ch; ++i)
      for (int j = 0; j < cw; ++j) {
        const long long o = 3 * ((long long)(margin_h + i) * w + margin_w + j) + k;
        x[i * cw + j] = quantise(gt[o]);
        y[i * cw + j] = quantise(pr[o]);
        sse += (x[i * cw + j] - y[i * cw + j]) * (x[i * cw + j] - y[i * cw + j]);
      }
    double s = 0.0;
    for (int i = HALF; i < ch - HALF; ++i)
      for (int j = HALF; j < cw - HALF; ++j) {
        int sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
        for (int a = -HALF; a <= HALF; ++a)
          for (int b = -HALF; b <= HALF; ++b) {
            const int u = x[(i + a) * cw + j + b], v = y[(i + a) * cw + j + b];
            sx += u; sy += v; sxx += u * u; syy += v * v; sxy += u * v;
          }
        s += ssim_term(sx, sy, sxx, syy, sxy);
      }
    out[k] = double(sse);
    mean[k] = s / (double(ch - 2 * HALF) * (cw - 2 * HALF));
  }
  out[3] = (mean[0] + mean[1] + mean[2]) / 3.0;
  return 0;
}

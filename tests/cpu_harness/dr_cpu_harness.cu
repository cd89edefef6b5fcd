// Test infrastructure: runs the direct-rendering routines of csrc/nr_dr_math.cuh on the HOST (nvcc compiles the same
// __host__ __device__ code for the CPU) so that tests/test_dr_cpu.py can check them against the fp64 oracle without a GPU.
// Not part of the product library.
#include <vector>

#include "../../neuray_b200/csrc/nr_dr_math.cuh"

// nr_direct_render on the host: every point, then every ray, as the two kernels of csrc/nr_dr.cu.
extern "C" int nr_dr_cpu(const NrPassParams* p, const NrDrParams* d) {
  const long long N = (long long)p->rn * p->dn;
  std::vector<float> rows((size_t)p->rfn * nr::dr::ROW);
  for (long long n = 0; n < N; ++n) nr::dr::dr_point(*p, *d, p->w_point, n, rows.data(), 1, d->hit_prob_dr, d->point_colors);
  for (long long r = 0; r < p->rn; ++r) nr::dr::dr_ray(*p, *d, r, d->point_colors);
  return 0;
}

// The SH fit alone: rows [npts][rfn][7] = masked hit, rgb (3), prj_dir (3); hit_sum [npts]; qdir [npts][3] -> color [npts][3].
extern "C" int nr_sh_fit_cpu(int npts, int rfn, const float* rows, const float* hit_sum, const float* regs, const float* qdir, float* color) {
  for (int i = 0; i < npts; ++i)
    nr::dr::sh_fit_color(rows + (size_t)i * rfn * nr::dr::ROW, 1, rfn, hit_sum[i], regs, qdir + 3 * i, color + 3 * i);
  return 0;
}

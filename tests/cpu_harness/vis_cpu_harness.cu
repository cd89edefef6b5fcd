// Test infrastructure: runs the per-view visibility routines of csrc/nr_visibility_math.cuh on the HOST (nvcc compiles the
// same __host__ __device__ code for the CPU) so that tests/test_visibility_cpu.py can check them against the fp64 oracle
// without a GPU.  Not part of the product library.
#include <vector>

#include "../../neuray_b200/csrc/nr_visibility_math.cuh"

// nr_view_visibility on the host: every ray as the kernel of csrc/nr_visibility.cu splits it, each lane's sum, then the
// same tree over the lanes.
extern "C" int nr_vis_cpu(const NrPassParams* p, const NrVisParams* q) {
  const int lanes = nr::vis::ray_lanes(p->dn);
  std::vector<float> acc((size_t)p->rfn * lanes);
  for (long long ray = 0; ray < p->rn; ++ray) {
    for (int lane = 0; lane < lanes; ++lane) nr::vis::lane_sum(*p, p->w_point, q->hit_prob, ray, lane, lanes, acc.data() + lane, lanes);
    for (int half = lanes >> 1; half > 0; half >>= 1)
      for (int lane = 0; lane < half; ++lane) nr::vis::tree_level(acc.data() + lane, lanes, p->rfn, half);
    for (int v = 0; v < p->rfn; ++v) q->visibility[ray * p->rfn + v] = acc[(size_t)v * lanes];
  }
  return 0;
}

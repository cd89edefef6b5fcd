// Training backward of one render_by_depth pass: kernels around the per-point / per-sample / per-ray routines of
// nr_train_math.cuh, and the C-ABI entry points nr_render_pass_bwd / nr_bwd_slot (include/neuray_b200.h).
// One thread per point / sample / ray (the training batch is 512 rays: 32 k points, 262 k rows); weights are read
// through the read-only path (every thread reads the same addresses).  Weight gradients are NOT produced here: each
// Linear's input and pre-activation gradient land on the tapes and the host forms dW = dz · xᵀ with cuBLAS.
#include <string.h>

#include "../../include/neuray_b200.h"
#include "nr_train_math.cuh"

namespace nr {
namespace tr {

#ifndef NR_TRAIN_MINB
#define NR_TRAIN_MINB 2     // 255 registers: the row sweeps spill 2.8 KB per thread at 128; measured 11.0 -> 10.4 ms per training step
#endif
template <int WHICH>
__global__ void __launch_bounds__(128, NR_TRAIN_MINB) train_kernel(const Ctx c, long long count) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x) {
    if (WHICH == 0) row_forward_a(c, i);
    else if (WHICH == 1) point_forward_b(c, i);
    else if (WHICH == 2) row_forward_c(c, i);
    else if (WHICH == 3) { point_forward_d(c, i); }
    else if (WHICH == 4) sample_forward(c, i);
    else if (WHICH == 5) ray_backward(c, i);
    else if (WHICH == 6) sample_backward_q(c, i);
    else if (WHICH == 7) { sample_backward_kv(c, i); point_backward_a(c, i); }
    else if (WHICH == 8) row_backward_b(c, i);
    else if (WHICH == 9) point_backward_c(c, i);
    else row_backward_d(c, i);
  }
}

__global__ void __launch_bounds__(64) self_kernel(const NrSelfParams c) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < c.rn; i += (long long)gridDim.x * blockDim.x) self_hit_prob_ray(c, i);
}

struct SlotName { const char* name; int value; };
static const SlotName kSlots[] = {
    {"R_SLOTS", R_SLOTS}, {"G_SLOTS", G_SLOTS}, {"P_SLOTS", P_SLOTS}, {"GP_SLOTS", GP_SLOTS},
    {"R_RF", R_RF}, {"R_DD", R_DD}, {"R_H1", R_H1}, {"R_H2", R_H2}, {"R_P1", R_P1}, {"R_RGBF", R_RGBF}, {"R_NF", R_NF}, {"R_Q8", R_Q8},
    {"R_R16", R_R16}, {"R_B1", R_B1}, {"R_U", R_U}, {"R_VH", R_VH}, {"R_X2", R_X2}, {"R_U2", R_U2}, {"R_WH", R_WH}, {"R_CH1", R_CH1},
    {"R_CH2", R_CH2}, {"R_MASK", R_MASK}, {"R_HITN", R_HITN}, {"R_VISN", R_VISN}, {"R_BLEND", R_BLEND},
    {"G_DD0", G_DD0}, {"G_DD1", G_DD1}, {"G_DD2", G_DD2}, {"G_PE0", G_PE0}, {"G_PE1", G_PE1}, {"G_NF0", G_NF0}, {"G_NF1", G_NF1},
    {"G_RD0", G_RD0}, {"G_RD1", G_RD1}, {"G_B0", G_B0}, {"G_B1", G_B1}, {"G_V0", G_V0}, {"G_V1", G_V1}, {"G_V20", G_V20}, {"G_V21", G_V21},
    {"G_C0", G_C0}, {"G_C1", G_C1}, {"G_C2", G_C2},
    {"P_GLOB", P_GLOB}, {"P_GIN", P_GIN}, {"P_GH", P_GH}, {"P_G16", P_G16}, {"P_RGBO", P_RGBO}, {"P_AX", P_AX}, {"P_O", P_O}, {"P_XH", P_XH},
    {"P_Y", P_Y}, {"P_T16", P_T16}, {"P_SIG", P_SIG}, {"P_ALPHA", P_ALPHA},
    {"GP_B0SUM", GP_B0SUM}, {"GP_GEO0", GP_GEO0}, {"GP_GEO1", GP_GEO1}, {"GP_DQ", GP_DQ}, {"GP_DK", GP_DK}, {"GP_DV", GP_DV},
    {"GP_DFC", GP_DFC}, {"GP_DLNY", GP_DLNY}, {"GP_OG0", GP_OG0}, {"GP_OG1", GP_OG1},
};

}  // namespace tr
}  // namespace nr

extern "C" {

int nr_bwd_slot(const char* name) {
  if (name == nullptr) return -1;
  for (const auto& s : nr::tr::kSlots)
    if (strcmp(s.name, name) == 0) return s.value;
  return -1;
}

int nr_self_hit_prob(const NrSelfParams* p, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(p != nullptr, "params");
  if (p->rn == 0) return NR_OK;
  NR_CHECK_ARG(p->map && p->coords && p->que_depth && p->w_point && p->hit, "null device pointer");
  NR_CHECK_ARG(p->dn >= 2 && p->fh >= 1 && p->fw >= 1 && p->h > 1 && p->w > 1, "shape");
  NR_CHECK_ARG(p->d_hit == nullptr || p->d_w_point != nullptr, "d_w_point required for the backward");
  tr::self_kernel<<<(p->rn + 63) / 64, 64, 0, (cudaStream_t)stream>>>(*p);
  NR_CHECK_LAUNCH("self_hit_prob");
  return NR_OK;
}

int nr_render_pass_bwd(const NrPassParams* p, const NrBwdParams* b, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(p != nullptr && b != nullptr, "params");
  NR_CHECK_ARG(p->coords && p->que_depth && p->que_cam && p->feat && p->rgb && p->view_params && p->w_point && p->w_ray && p->pos_enc,
               "null device pointer");
  NR_CHECK_ARG(b->tape_row && b->grad_row && b->tape_point && b->grad_point, "tapes");
  NR_CHECK_ARG(p->rfn >= 1 && p->rfn <= NR_MAX_VIEWS && p->dn >= 3 && p->dn <= NR_MAX_SAMPLES, "shape");
  if (p->rn == 0) return NR_OK;
  const long long N = (long long)p->rn * p->dn, R = N * p->rfn;
  tr::Ctx c;
  c.p = *p;
  c.n_heads = p->use_vis ? 4 : 3;
  c.W = p->w_point;
  c.Wr = p->w_ray;
  c.tr = {b->tape_row, R, tr::R_SLOTS};
  c.gr = {b->grad_row, R, tr::G_SLOTS};
  c.tp = {b->tape_point, N, tr::P_SLOTS};
  c.gp = {b->grad_point, N, tr::GP_SLOTS};
  c.d_feat = b->d_feat;
  c.d_pix = b->d_pixel_colors;
  c.d_hit = b->d_hit_prob;
  c.d_depth = b->d_render_depth;
  cudaStream_t s = (cudaStream_t)stream;
  auto blocks = [](long long n) { long long g = (n + 127) / 128; return int(g < 132 * 32 ? g : 132 * 32); };
  tr::train_kernel<0><<<blocks(R), 128, 0, s>>>(c, R);      // rows:   gather .. ray_dir_fc
  tr::train_kernel<1><<<blocks(N), 128, 0, s>>>(c, N);      // points: view pooling #1
  tr::train_kernel<2><<<blocks(R), 128, 0, s>>>(c, R);      // rows:   base_fc .. rgb_fc
  tr::train_kernel<3><<<blocks(N), 128, 0, s>>>(c, N);      // points: view pooling #2, geometry_fc, blend, q/k/v
  tr::train_kernel<4><<<blocks(N), 128, 0, s>>>(c, N);      // samples: attention .. alpha
  tr::train_kernel<5><<<blocks(p->rn), 128, 0, s>>>(c, (long long)p->rn);   // rays: compositing forward + backward
  tr::train_kernel<6><<<blocks(N), 128, 0, s>>>(c, N);      // samples: out_geometry_fc, LayerNorm, attention wrt q
  tr::train_kernel<7><<<blocks(N), 128, 0, s>>>(c, N);      // samples/points: attention wrt k, v; geometry_fc; pooling #2
  tr::train_kernel<8><<<blocks(R), 128, 0, s>>>(c, R);      // rows:   rgb_fc .. base_fc
  tr::train_kernel<9><<<blocks(N), 128, 0, s>>>(c, N);      // points: pooling #1
  tr::train_kernel<10><<<blocks(R), 128, 0, s>>>(c, R);     // rows:   neuray_fc .. dist decoder, scatter
  NR_CHECK_LAUNCH("render_pass_bwd");
  return NR_OK;
}

}  // extern "C"

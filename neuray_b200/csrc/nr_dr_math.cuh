// Direct rendering (DR) of one render_by_depth pass, forward only (reference: network/renderer.py:85-125, 181-185 and
// network/sph_solver.py:34-59), as plain per-point and per-ray routines.  The device kernels of nr_dr.cu run them, and
// tests/cpu_harness/dr_cpu_harness.cu runs the same code on the host.
//
//   dr_point  per point: every view's row through tr::row_front (the gather, dist decoder and compute_prob of the training
//             forward), the masked alpha logits pooled by visibility (predict_alpha_values_dr), the colour either from a
//             degree-3 spherical-harmonics fit to the views' colours (predict_colors_dr) or the NR colour of the point
//             record, and sigmoid(alpha) (the coarse decoder's decode_alpha_value)
//   dr_ray    per ray: alpha_values2hit_prob (cumprod with + 1e-10) and the colour sum
//
// The SH normal matrix M = Aᵀ diag(w) A + diag(regs) is symmetric positive definite (M[0][0] = Σw > 0 after the
// insufficient-weight fix, every other diagonal gets regs > 0), so the solve is an fp32 Cholesky factorisation where
// the reference calls torch.inverse.
#pragma once
#include "nr_train_math.cuh"

namespace nr {
namespace dr {

constexpr int SH = 16;      // degree 3: 1 + 3 + 5 + 7 basis functions
constexpr int ROW = 7;      // per-view scratch floats of dr_point: hit (masked), rgb (3), prj_dir (3)

// The basis of SphericalHarmonicsSolver.get_coefficient_func()[:4], in the reference's order and signs.
NR_HD void sh_basis(float x, float y, float z, float* Y) {
  const float xx = x * x, yy = y * y, zz = z * z;
  Y[0] = 1.f;
  Y[1] = x; Y[2] = y; Y[3] = z;
  Y[4] = x * y; Y[5] = y * z; Y[6] = -xx - yy + 2.f * zz; Y[7] = z * x; Y[8] = xx - yy;
  Y[9] = (3.f * xx - yy) * y; Y[10] = x * y * z; Y[11] = y * (4.f * zz - xx - yy); Y[12] = z * (2.f * zz - 3.f * xx - 3.f * yy);
  Y[13] = x * (4.f * zz - xx - yy); Y[14] = (xx - yy) * z; Y[15] = (xx - 3.f * yy) * x;
}

// Solves M θ = b (3 right-hand sides) for the SPD M, given as its lower triangle packed row by row
// (m[i * (i + 1) / 2 + j], j <= i); m is overwritten by the Cholesky factor L, b by θ.
NR_HD void sh_solve(float* m, float* b) {
#pragma unroll
  for (int i = 0; i < SH; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      float s = m[i * (i + 1) / 2 + j];
#pragma unroll
      for (int k = 0; k < j; ++k) s = fmaf(-m[i * (i + 1) / 2 + k], m[j * (j + 1) / 2 + k], s);
      if (j == i) m[i * (i + 1) / 2 + i] = sqrtf(fmaxf(s, 1e-30f));
      else m[i * (i + 1) / 2 + j] = s / m[j * (j + 1) / 2 + j];
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int i = 0; i < SH; ++i) {          // L y = b
      float s = b[i * 3 + c];
#pragma unroll
      for (int k = 0; k < i; ++k) s = fmaf(-m[i * (i + 1) / 2 + k], b[k * 3 + c], s);
      b[i * 3 + c] = s / m[i * (i + 1) / 2 + i];
    }
#pragma unroll
    for (int i = SH - 1; i >= 0; --i) {     // Lᵀ θ = y
      float s = b[i * 3 + c];
#pragma unroll
      for (int k = i + 1; k < SH; ++k) s = fmaf(-m[k * (k + 1) / 2 + i], b[k * 3 + c], s);
      b[i * 3 + c] = s / m[i * (i + 1) / 2 + i];
    }
  }
}

// predict_colors_dr for one point from its views' rows (scratch element (v, k) at rows[(v * ROW + k) * stride]):
// w_v = hit_v / (Σ hit + 1e-3), every w_v + 1e-4 when Σ w < 1e-4, θ = M⁻¹ Aᵀ diag(w) rgb, colour = Y(que_dir) θ.
NR_HD void sh_fit_color(const float* rows, int stride, int rfn, float hit_sum, const float* regs, const float* qdir, float* color) {
  const float inv = 1.f / (hit_sum + 1e-3f);
  float wsum = 0.f;
  for (int v = 0; v < rfn; ++v) wsum += rows[(v * ROW) * stride] * inv;
  const float wadd = wsum < 1e-4f ? 1e-4f : 0.f;
  float m[SH * (SH + 1) / 2], b[SH * 3];
#pragma unroll
  for (int i = 0; i < SH * (SH + 1) / 2; ++i) m[i] = 0.f;
#pragma unroll
  for (int i = 0; i < SH * 3; ++i) b[i] = 0.f;
  for (int v = 0; v < rfn; ++v) {
    const float* rv = rows + (v * ROW) * stride;
    const float wv = rv[0] * inv + wadd;
    float Y[SH];
    sh_basis(rv[4 * stride], rv[5 * stride], rv[6 * stride], Y);
    const float c0 = rv[stride] * wv, c1 = rv[2 * stride] * wv, c2 = rv[3 * stride] * wv;
#pragma unroll
    for (int i = 0; i < SH; ++i) {
      const float wy = Y[i] * wv;
#pragma unroll
      for (int j = 0; j <= i; ++j) m[i * (i + 1) / 2 + j] = fmaf(wy, Y[j], m[i * (i + 1) / 2 + j]);
      b[i * 3] = fmaf(Y[i], c0, b[i * 3]); b[i * 3 + 1] = fmaf(Y[i], c1, b[i * 3 + 1]); b[i * 3 + 2] = fmaf(Y[i], c2, b[i * 3 + 2]);
    }
  }
#pragma unroll
  for (int i = 0; i < SH; ++i) m[i * (i + 1) / 2 + i] += regs[i];
  sh_solve(m, b);
  float Y[SH];
  sh_basis(qdir[0], qdir[1], qdir[2], Y);
  for (int c = 0; c < 3; ++c) {
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < SH; ++i) a = fmaf(Y[i], b[i * 3 + c], a);
    color[c] = a;
  }
}

// One point n of the pass: writes sigmoid(alpha_dr) to alpha_out[n] and the DR colour to color_out[3n..3n+2].
// `rows` / `stride`: per-view scratch of ROW floats per view (see sh_fit_color); unused with use_nr_color.
NR_HD void dr_point(const NrPassParams& pp, const NrDrParams& d, const float* __restrict__ W, long long n, float* rows, int stride,
                    float* alpha_out, float* color_out) {
  const int n_heads = pp.use_vis ? 4 : 3;
  const PointGeo g = point_geometry(pp.que_cam, pp.coords, pp.que_depth, pp.dn, n);
  float hit_sum = 0.f, vis_sum = 0.f, va_sum = 0.f, mask_sum = 0.f;
  for (int v = 0; v < pp.rfn; ++v) {
    tr::RowFront f;
    tr::row_front(pp, W, n_heads, g, v, f, nullptr, 0);
    // predict_proj_ray_prob (renderer.py:79-82): alpha from the unmasked values, then the mask
    const float alpha = f.mask > 0.f ? logf(f.hit / (f.visb - f.hit + 1e-5f) + 1e-5f) : d.alpha_ground_state;
    const float vis = f.visb * f.mask, hit = f.hit * f.mask;
    hit_sum += hit; vis_sum += vis; va_sum = fmaf(vis, alpha, va_sum); mask_sum += f.mask;
    if (!d.use_nr_color) {
      float* rv = rows + (v * ROW) * stride;
      rv[0] = hit;
      rv[stride] = f.rgb[0]; rv[2 * stride] = f.rgb[1]; rv[3 * stride] = f.rgb[2];     // zero where masked
      rv[4 * stride] = f.dir[0]; rv[5 * stride] = f.dir[1]; rv[6 * stride] = f.dir[2];
    }
  }
  // predict_alpha_values_dr (renderer.py:85-94); a point no view sees gets the ground state
  const float alpha_dr = mask_sum == 0.f ? d.alpha_ground_state : va_sum / (vis_sum + 1e-5f);
  alpha_out[n] = tr::sigm(alpha_dr);
  if (d.use_nr_color) {
    for (int c = 0; c < 3; ++c) color_out[3 * n + c] = pp.point_rec[n * NR_POINT_REC + 16 + c];
  } else {
    const float qdir[3] = {g.qx, g.qy, g.qz};
    sh_fit_color(rows, stride, pp.rfn, hit_sum, d.regs, qdir, color_out + 3 * n);
  }
}

// One ray: alpha_values2hit_prob (render_ops.py:72-80) over the ray's sigmoid(alpha) in place in hit_prob_dr, and
// pixel_colors_dr = Σ_d hit_dr · colour.
NR_HD void dr_ray(const NrPassParams& pp, const NrDrParams& d, long long ray, const float* color) {
  const int dn = pp.dn;
  float* hp = d.hit_prob_dr + ray * dn;
  const float* col = color + ray * dn * 3;
  float t = 1.f, px = 0.f, py = 0.f, pz = 0.f;
  for (int s = 0; s < dn; ++s) {
    const float a = hp[s];
    const float hv = a * t;
    hp[s] = hv;
    t *= 1.f - a + 1e-10f;
    px = fmaf(hv, col[3 * s], px); py = fmaf(hv, col[3 * s + 1], py); pz = fmaf(hv, col[3 * s + 2], pz);
  }
  d.pixel_colors_dr[3 * ray] = px; d.pixel_colors_dr[3 * ray + 1] = py; d.pixel_colors_dr[3 * ray + 2] = pz;
}

}  // namespace dr
}  // namespace nr

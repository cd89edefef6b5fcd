// Backward of one render_by_depth pass (training), as plain per-point / per-sample / per-ray routines.
//
// Structure (reference: network/renderer.py:168-203 with dist_decoder.py, aggregate_net.py, ibrnet.py; the forward
// restated here is the one of oracle/neuray_oracle.py, i.e. of the reference):
//   point_forward   per point: every (point, view) row up to the 20-float record, all activations a backward needs go
//                   to a slot-major "tape" in global memory (row tape [R_SLOTS][rfn*N], point tape [P_SLOTS][N])
//   sample_forward  per sample: attention over the ray's samples, LayerNorm, out_geometry_fc -> alpha
//   ray_backward    per ray: compositing forward + backward -> d sigma, d blended colour
//   sample_backward_q / sample_backward_kv  per sample: out_geometry_fc, LayerNorm, attention (query side / key side)
//   point_backward  per point: everything else in reverse, gradients of the gathered features scattered into the
//                   channel-last map gradient
// Every Linear layer's pre-activation gradient dz is written to a gradient tape next to its input on the forward tape;
// the weight gradients are then plain GEMMs dW = dz · xᵀ over all rows (done by the host with cuBLAS), biases are row
// sums.  One thread runs one point / sample / ray with loops over the views or samples inside: the training batch is
// small (512 rays) and the code is the same on the host, where tests/ compile it with nvcc as host code and check it
// against PyTorch autograd without a GPU.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "nr_common.cuh"

namespace nr {
namespace tr {

// ---- tape slots -------------------------------------------------------------------------------------------------
enum RowSlot {
  R_RF = 0,        // 32 gathered ray_feats (x mask)
  R_HITN = 32,     // (hit - .5) * 2        } contiguous with R_RF: prob_embed.0 input (34)
  R_VISN = 33,     // (visibility - .5) * 2 }
  R_DD = 34,       // 4  ray_diff = [dir - que_dir, dot]: ray_dir_fc.0 input
  R_MASK = 38, R_TLO = 39, R_THI = 40, R_W1 = 41,
  R_H1 = 42,       // 4 heads x 32
  R_H2 = 170,      // 4 heads x 32
  R_MEAN = 298, R_VAR = 300, R_AW = 302, R_VISD = 303,
  R_C0 = 304,      // 2 cdf(lo) per mixture component (before the vis factor)
  R_C1 = 306,      // 2 cdf(hi)
  R_P1 = 308,      // 32 prob_embed hidden (ReLU)
  R_RGBF = 340,    // 35 rgb_feat (after + ray_dir_fc)  } contiguous: per-view part of base_fc.0's input (67)
  R_NF = 375,      // 32 neuray_feat                    }
  R_Q8 = 407, R_SG = 415, R_R16 = 416, R_DF = 432,
  R_B1 = 467,      // 64
  R_X = 531,       // 32
  R_U = 563,       // 32 x * weight
  R_VH = 595,      // 32
  R_XV = 627,      // 33 (post ELU; [32] = visibility logit)
  R_X2 = 660,      // 32  } contiguous: rgb_fc.0 input (37)
  R_VIS2 = 692,    //  1  }
  R_DDC = 693,     //  4  }
  R_VISA = 697,
  R_U2 = 698,      // 32 x2 * visa
  R_WH = 730,      // 32
  R_CH1 = 762,     // 16
  R_CH2 = 778,     // 8
  R_BLEND = 786,
  R_RGB = 787,     // 3 raw rgb taps (x mask)
  R_TCODE = 790,   // feature-map tap code (int bits), -1 if masked
  R_TW = 791,      // 4 tap weights
  R_SLOTS = 795
};
enum RowGrad {
  G_DD0 = 0, G_DD1 = 128, G_DD2 = 256, G_PE0 = 264, G_PE1 = 296, G_NF0 = 328, G_NF1 = 336, G_RD0 = 337, G_RD1 = 353,
  G_B0 = 388, G_B1 = 452, G_V0 = 484, G_V1 = 516, G_V20 = 549, G_V21 = 581, G_C0 = 582, G_C1 = 598, G_C2 = 606, G_SLOTS = 607
};
enum PointSlot {
  P_GLOB = 0,      // 140: mean0, var0, mean1, var1 (35 each)
  P_MSUM = 140, P_VSUM = 141,
  P_GIN = 142,     // 65: mean, var, mean weight
  P_GH = 207,      // 64
  P_G16 = 271,     // 16
  P_RGBO = 287,    // 3
  P_AX = 290,      // 16 geometry feature + pos_enc
  P_Q = 306, P_K = 322, P_V = 338,
  P_O = 354,       // 16 attention output
  P_XH = 370,      // 16 normalised pre-LN activations
  P_RSTD = 386,
  P_Y = 387,       // 16
  P_T16 = 403,     // 16
  P_SIG = 419, P_ALPHA = 420,
  P_AM = 421,      // 4 softmax max per head
  P_AD = 425,      // 4 softmax denominators
  P_HZ = 429,      // 64 view-invariant part of base_fc.0's pre-activation (incl. bias)
  P_SLOTS = 493
};
enum PointGrad {
  GP_B0SUM = 0,    // 64  sum over views of base_fc.0's dz (pairs with P_GLOB)
  GP_GEO0 = 64, GP_GEO1 = 128, GP_DQ = 144, GP_DK = 160, GP_DV = 176,
  GP_DFC = 192,    // 16 dz of attention.fc (= gradient of the pre-LN sum; also the residual branch)
  GP_DLNY = 208,   // 16 gradient of the LayerNorm output
  GP_OG0 = 224, GP_OG1 = 240,
  GP_DG16 = 241,   // 16 (unused by the GEMMs: gradient handed to point_backward)
  GP_DRGB = 257,   // 3
  GP_DELTA = 260,  // 4
  GP_DO = 264,     // 16
  GP_DGIN = 280,   // 65 gradient of geometry_fc.0's input
  GP_DMT = 345,    // 32 total gradient of the pooled means (#2)
  GP_DW2SUM = 377, GP_BSUM = 378,
  GP_DGLOB = 379,  // 140 gradient of the pooled statistics (#1)
  GP_DM0 = 519,    // 35 total gradient of mean0
  GP_DM1 = 554,    // 35 total gradient of mean1
  GP_SLOTS = 589
};

// Tape layout: rows are grouped in tiles of 128; a tile holds all slots of its 128 rows, slot-major:
//   element (slot, i) = p[((i >> 7) * slots + slot) * 128 + (i & 127)].
// A CTA of 128 threads (consecutive rows) therefore works on ONE contiguous piece of memory (slots x 512 bytes) and a
// K-chunk of a Linear's input is one contiguous block of n_in x 512 bytes for the weight-gradient GEMMs (with a plain
// slot-major layout every slot of a row is a megabyte apart).
constexpr int TILE = 128;
#ifndef NR_TAPE_RESTRICT
#define NR_TAPE_RESTRICT 0
#endif
struct Tape {
#if NR_TAPE_RESTRICT
  float* __restrict__ p;
#else
  float* p;
#endif
  long long rows;     // logical rows (the buffer holds ceil(rows / 128) * 128)
  int slots;
  NR_HD float& at(int slot, long long i) const { return p[((i >> 7) * slots + slot) * TILE + (i & (TILE - 1))]; }
};
template <int K>
NR_HD void ldv(const Tape& t, int slot, long long i, float* o) {
#pragma unroll
  for (int k = 0; k < K; ++k) o[k] = t.at(slot + k, i);
}
template <int K>
NR_HD void stv(const Tape& t, int slot, long long i, const float* v) {
#pragma unroll
  for (int k = 0; k < K; ++k) t.at(slot + k, i) = v[k];
}

struct Ctx {
  NrPassParams p;
  int n_heads;
  const float* W;      // w_point (lay:: layout); shared memory on the device
  const float* Wr;     // w_ray
  Tape tr, tp, gr, gp;
  float* d_feat;       // [rfn,fh,fw,64] gradient of the channel-last maps (accumulated)
  const float* d_pix;  // [rn,3] or null
  const float* d_hit;  // [rn,dn] or null
  const float* d_depth;// [rn] or null
};

// ---- small math ---------------------------------------------------------------------------------------------------
NR_HD float elu_f(float x) { return x > 0.f ? x : expf(x) - 1.f; }
NR_HD float elu_g(float a) { return a > 0.f ? 1.f : a + 1.f; }           // derivative from the activation's output
NR_HD float sigm(float x) { return 1.f / (1.f + expf(-x)); }
NR_HD float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
NR_HD float softplus_g(float a) { return 1.f - expf(-a); }               // derivative from the activation's output

// z[OUT] = b + W^T x with W stored [IN][LD].  Weight rows are read with 128-bit loads when the shapes allow (all
// weight blocks start on 16-byte boundaries, nr_common.cuh lay::): every thread reads the same addresses, so the load
// instruction count, not the bandwidth, is what these row loops pay for.
template <int IN, int OUT, int LD = OUT>
NR_HD void lin(const float* __restrict__ W, const float* __restrict__ b, const float* x, float* z) {
#pragma unroll
  for (int j = 0; j < OUT; ++j) z[j] = b ? b[j] : 0.f;
  for (int i = 0; i < IN; ++i) {
    const float xi = x[i];
    if constexpr (OUT % 4 == 0 && LD % 4 == 0) {
      const float4* __restrict__ w4 = reinterpret_cast<const float4*>(W + i * LD);
#pragma unroll
      for (int j = 0; j < OUT / 4; ++j) {
        const float4 w = w4[j];
        z[4 * j] = fmaf(w.x, xi, z[4 * j]); z[4 * j + 1] = fmaf(w.y, xi, z[4 * j + 1]);
        z[4 * j + 2] = fmaf(w.z, xi, z[4 * j + 2]); z[4 * j + 3] = fmaf(w.w, xi, z[4 * j + 3]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < OUT; ++j) z[j] = fmaf(W[i * LD + j], xi, z[j]);
    }
  }
}
// dx[IN] = W dz
template <int IN, int OUT, int LD = OUT>
NR_HD void lin_t(const float* __restrict__ W, const float* dz, float* dx) {
  for (int i = 0; i < IN; ++i) {
    float a = 0.f;
    if constexpr (OUT % 4 == 0 && LD % 4 == 0) {
      const float4* __restrict__ w4 = reinterpret_cast<const float4*>(W + i * LD);
#pragma unroll
      for (int j = 0; j < OUT / 4; ++j) {
        const float4 w = w4[j];
        a = fmaf(w.x, dz[4 * j], a); a = fmaf(w.y, dz[4 * j + 1], a); a = fmaf(w.z, dz[4 * j + 2], a); a = fmaf(w.w, dz[4 * j + 3], a);
      }
    } else {
#pragma unroll
      for (int j = 0; j < OUT; ++j) a = fmaf(W[i * LD + j], dz[j], a);
    }
    dx[i] = a;
  }
}

NR_HD void atomic_add(float* p, float v) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}

// four consecutive floats (16-byte aligned) in one reduction: red.global.add.v4.f32 on the device
NR_HD void atomic_add4(float* p, float a, float b, float c, float d) {
#ifdef __CUDA_ARCH__
  atomicAdd(reinterpret_cast<float4*>(p), make_float4(a, b, c, d));
#else
  p[0] += a; p[1] += b; p[2] += c; p[3] += d;
#endif
}

// ---- one dist-decoder head (dist_decoder.py:64-97): Linear(32,32) ELU Linear(32,32) ELU Linear(32,2) ------------------
// Wh: head hd's block of w_point (lay::DD_*); h1, h2: the two ELU outputs.  With `tape` non-null the forward writes h1 / h2
// to its R_H1 / R_H2 slots of row r, and the backward dz1 / dz0 to its G_DD1 / G_DD0 slots; with `dWh` non-null the
// backward adds the weight gradients to dWh (laid out like Wh) by atomics.  Both happen where the values are made: a
// store after the call would keep 32 more values live and spill in the 255-register training kernels.
NR_HD void head_fwd(const float* __restrict__ Wh, const float* rf, float* h1, float* h2, float* out, const Tape* tape, long long r,
                    int hd) {
  lin<32, 32>(Wh + lay::DD_L0_W, Wh + lay::DD_L0_B, rf, h1);
  for (int k = 0; k < 32; ++k) h1[k] = elu_f(h1[k]);
  lin<32, 32>(Wh + lay::DD_L1_W, Wh + lay::DD_L1_B, h1, h2);
  for (int k = 0; k < 32; ++k) h2[k] = elu_f(h2[k]);
  if (tape) {
    stv<32>(*tape, R_H1 + 32 * hd, r, h1);
    stv<32>(*tape, R_H2 + 32 * hd, r, h2);
  }
  for (int o = 0; o < 2; ++o) {
    float a = Wh[lay::DD_L2_B + o];
    for (int k = 0; k < 32; ++k) a = fmaf(Wh[lay::DD_L2_W + o * 32 + k], h2[k], a);
    out[o] = a;
  }
}
// Backward from the output gradients dho: W0 dz0 is added to drf (rf, the head's input, is read only with dWh).
NR_HD void head_bwd(const float* __restrict__ Wh, const float* rf, const float* h1, const float* h2, const float* dho, float* drf,
                    float* dWh, const Tape* tape, long long r, int hd) {
  if (dWh)
    for (int o = 0; o < 2; ++o) {
      atomic_add(dWh + lay::DD_L2_B + o, dho[o]);
      for (int k = 0; k < 32; ++k) atomic_add(dWh + lay::DD_L2_W + o * 32 + k, dho[o] * h2[k]);
    }
  float dz1[32], dz0[32], t[32];
  for (int k = 0; k < 32; ++k) dz1[k] = (Wh[lay::DD_L2_W + k] * dho[0] + Wh[lay::DD_L2_W + 32 + k] * dho[1]) * elu_g(h2[k]);
  if (tape) stv<32>(*tape, G_DD1 + 32 * hd, r, dz1);
  lin_t<32, 32>(Wh + lay::DD_L1_W, dz1, dz0);
  for (int k = 0; k < 32; ++k) dz0[k] *= elu_g(h1[k]);
  if (tape) stv<32>(*tape, G_DD0 + 32 * hd, r, dz0);
  if (dWh)
    for (int j = 0; j < 32; ++j) {
      atomic_add(dWh + lay::DD_L1_B + j, dz1[j]);
      atomic_add(dWh + lay::DD_L0_B + j, dz0[j]);
      for (int i = 0; i < 32; ++i) {                                // WT[in][out]
        atomic_add(dWh + lay::DD_L1_W + i * 32 + j, h1[i] * dz1[j]);
        atomic_add(dWh + lay::DD_L0_W + i * 32 + j, rf[i] * dz0[j]);
      }
    }
  lin_t<32, 32>(Wh + lay::DD_L0_W, dz0, t);
  for (int k = 0; k < 32; ++k) drf[k] += t[k];
}

// ---- compute_prob (dist_decoder.py:6-51, 109-140) ----------------------------------------------------------------------
// The two-component mixture from the heads' outputs ho (mean, var, aw, vis; ho[3] is read only with use_vis).
struct Mix { float mean[2], var[2], aw, visd; };
NR_HD Mix mix_fwd(const float (&ho)[4][2], float var_bias, bool use_vis) {
  Mix m;
  for (int i = 0; i < 2; ++i) { m.mean[i] = softplus_f(ho[0][i]); m.var[i] = softplus_f(ho[1][i]) + var_bias; }
  m.aw = sigm(ho[2][0]);
  m.visd = use_vis ? sigm(ho[3][0]) : 1.f;
  return m;
}
// Hit and visibility of the bin (lo, hi) in normalised inverse depth, before any projection mask; c0 / c1: each
// component's CDF at lo / hi, before the vis factor.
NR_HD void bin_fwd(const Mix& m, float lo, float hi, float* c0, float* c1, float& hit, float& visb) {
  hit = 0.f; visb = 0.f;
  for (int i = 0; i < 2; ++i) {
    c0[i] = sigm(2.f * (lo - m.mean[i]) * m.var[i]);      // 0.5 + 0.5 tanh(x)
    c1[i] = sigm(2.f * (hi - m.mean[i]) * m.var[i]);
    const float mix = i == 0 ? m.aw : 1.f - m.aw;
    visb += (1.f - c0[i] * m.visd) * mix;
    hit += (c1[i] - c0[i]) * m.visd * mix;
  }
}
// Gradients of the mixture's parameters (mix: of the two component weights aw, 1 - aw).
struct MixGrad { float mean[2], var[2], mix[2], visd; };
// bin_fwd's backward: the gradients of (hit, visb) added to g.
NR_HD void bin_bwd(const Mix& m, float lo, float hi, const float* c0, const float* c1, float dhit, float dvisb, MixGrad& g) {
  for (int i = 0; i < 2; ++i) {
    const float mix = i == 0 ? m.aw : 1.f - m.aw;
    const float dc1 = dhit * mix, dc0 = -(dhit + dvisb) * mix;          // wrt cdf * visd
    g.mix[i] += dhit * (c1[i] - c0[i]) * m.visd + dvisb * (1.f - c0[i] * m.visd);
    g.visd += dc1 * c1[i] + dc0 * c0[i];
    const float dx1 = dc1 * m.visd * 2.f * c1[i] * (1.f - c1[i]), dx0 = dc0 * m.visd * 2.f * c0[i] * (1.f - c0[i]);
    g.mean[i] -= (dx1 + dx0) * m.var[i];
    g.var[i] += dx1 * (hi - m.mean[i]) + dx0 * (lo - m.mean[i]);
  }
}
// mix_fwd's backward: the gradients of the heads' outputs (zero for ho[3] without use_vis).
NR_HD void mix_bwd(const Mix& m, const MixGrad& g, float var_bias, bool use_vis, float (&dho)[4][2]) {
  for (int i = 0; i < 2; ++i) {
    dho[0][i] = g.mean[i] * softplus_g(m.mean[i]);
    dho[1][i] = g.var[i] * softplus_g(m.var[i] - var_bias);
  }
  dho[2][0] = (g.mix[0] - g.mix[1]) * m.aw * (1.f - m.aw);
  dho[2][1] = 0.f;
  dho[3][0] = use_vis ? g.visd * m.visd * (1.f - m.visd) : 0.f;
  dho[3][1] = 0.f;
}

// ---- one (point, view) row up to the dist decoder's probabilities (renderer.py:67-83 with project_points_dict) ------
// Shared by the training forward (row_forward_a) and direct rendering (nr_dr_math.cuh).  `hit` and `visb` are compute_prob's
// values BEFORE the projection mask; `dir` is project_points_directions' unit vector (ref camera -> point, negated).  With
// `tape` non-null the heads' hidden activations go to its R_H1 / R_H2 slots of row r.
struct RowFront {
  float mask, dir[3];
  float rf[32], imf[32], rgb[3], tw[4];
  int tcode;
  Mix m;
  float c0[2], c1[2], lo, hi, hit, visb;
};
NR_HD void row_front(const NrPassParams& pp, const float* __restrict__ W, int n_heads, const PointGeo& g, int v, RowFront& o,
                     const Tape* tape, long long r) {
  const int h = pp.h, w = pp.w, fh = pp.fh, fw = pp.fw;
  const float* vp = pp.view_params + v * 20;
  const Proj pj = project(vp, g.X, g.Y, g.Z, h, w);
  o.mask = pj.valid ? 1.f : 0.f;
  for (int k = 0; k < 3; ++k) o.dir[k] = pj.dir[k];
  for (int k = 0; k < 3; ++k) o.rgb[k] = 0.f;
  for (int k = 0; k < 4; ++k) o.tw[k] = 0.f;
  for (int k = 0; k < 32; ++k) { o.rf[k] = 0.f; o.imf[k] = 0.f; }
  o.tcode = -1;
  if (pj.valid) {
    {
      const Taps t = border_taps(pj.ux, pj.uy, h, w, fh, fw, fh == h && fw == w);
      o.tcode = tap_code(t, v, fh, fw);
      for (int k = 0; k < 4; ++k) o.tw[k] = t.w[k];
      const float* base = pp.feat + (o.tcode & ~63);
      const int dxo = (o.tcode & 1) << 6, dyo = (o.tcode & 2) ? fw * 64 : 0;
      for (int k = 0; k < 32; ++k) {
        o.rf[k] = base[k] * o.tw[0] + base[dxo + k] * o.tw[1] + base[dyo + k] * o.tw[2] + base[dyo + dxo + k] * o.tw[3];
        o.imf[k] = base[32 + k] * o.tw[0] + base[dxo + 32 + k] * o.tw[1] + base[dyo + 32 + k] * o.tw[2] + base[dyo + dxo + 32 + k] * o.tw[3];
      }
    }
    {
      const Taps t = border_taps(pj.ux, pj.uy, h, w, h, w, true);
      const float* b = pp.rgb + (size_t)v * h * w * 4;
      const float* t00 = b + ((size_t)t.y0 * w + t.x0) * 4; const float* t01 = b + ((size_t)t.y0 * w + t.x1) * 4;
      const float* t10 = b + ((size_t)t.y1 * w + t.x0) * 4; const float* t11 = b + ((size_t)t.y1 * w + t.x1) * 4;
      for (int k = 0; k < 3; ++k) o.rgb[k] = t00[k] * t.w[0] + t01[k] * t.w[1] + t10[k] * t.w[2] + t11[k] * t.w[3];
    }
  }

  // dist decoder heads (dist_decoder.py:64-107)
  float ho[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
  for (int hd = 0; hd < n_heads; ++hd) {
    float h1[32], h2[32];
    head_fwd(W + lay::DD_HEAD + hd * lay::DD_HEAD_STRIDE, o.rf, h1, h2, ho[hd], tape, r, hd);
  }
  o.m = mix_fwd(ho, pp.var_bias, pp.use_vis);
  const float zc = fmaxf(pj.zh, 1e-5f);
  const float tz = (-1.f / zc - vp[15]) / (vp[16] - vp[15]);
  o.lo = tz - g.ihp; o.hi = tz + g.ihc;
  bin_fwd(o.m, o.lo, o.hi, o.c0, o.c1, o.hit, o.visb);
}

// ---- forward, phase a, one (point, view) row: gather, dist decoder, probabilities, prob_embed, neuray_fc, ray_dir_fc ----
NR_HD void row_forward_a(const Ctx& c, long long r) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const long long N = (long long)pp.rn * pp.dn;
  const int v = int(r / N);
  const long long n = r - (long long)v * N;
  const PointGeo g = point_geometry(pp.que_cam, pp.coords, pp.que_depth, pp.dn, n);
  {
    RowFront f;
    row_front(pp, W, c.n_heads, g, v, f, &c.tr, r);
    const float mask = f.mask;
    const float* rf = f.rf;
    const float* imf = f.imf;
    const float* rgb = f.rgb;
    float dd[4] = {f.dir[0] - g.qx, f.dir[1] - g.qy, f.dir[2] - g.qz, f.dir[0] * g.qx + f.dir[1] * g.qy + f.dir[2] * g.qz};
    stv<32>(c.tr, R_RF, r, rf);
    stv<4>(c.tr, R_DD, r, dd);
    stv<4>(c.tr, R_DDC, r, dd);
    stv<3>(c.tr, R_RGB, r, rgb);
    stv<4>(c.tr, R_TW, r, f.tw);
    { float tc; memcpy(&tc, &f.tcode, 4); c.tr.at(R_TCODE, r) = tc; }
    c.tr.at(R_MASK, r) = mask;
    const float visb = f.visb * mask, hit = f.hit * mask;
    stv<2>(c.tr, R_MEAN, r, f.m.mean); stv<2>(c.tr, R_VAR, r, f.m.var);
    c.tr.at(R_AW, r) = f.m.aw; c.tr.at(R_VISD, r) = f.m.visd;
    stv<2>(c.tr, R_C0, r, f.c0); stv<2>(c.tr, R_C1, r, f.c1);
    c.tr.at(R_TLO, r) = f.lo; c.tr.at(R_THI, r) = f.hi;
    const float hitn = (hit - 0.5f) * 2.f, visn = (visb - 0.5f) * 2.f;
    c.tr.at(R_HITN, r) = hitn; c.tr.at(R_VISN, r) = visn;

    // prob_embed (aggregate_net.py:28-32, 49-51)
    const float* Wb = W + lay::GRP_B;
    float e[34];
    for (int k = 0; k < 32; ++k) e[k] = rf[k];
    e[32] = hitn; e[33] = visn;
    float p1[32], nf[32];
    lin<34, 32>(Wb + lay::PE0_W, Wb + lay::PE0_B, e, p1);
    for (int k = 0; k < 32; ++k) p1[k] = fmaxf(p1[k], 0.f);
    lin<32, 32>(Wb + lay::PE1_W, Wb + lay::PE1_B, p1, nf);
    stv<32>(c.tr, R_P1, r, p1);
    stv<32>(c.tr, R_NF, r, nf);
    // neuray_fc (ibrnet.py:286-290, 327-329)
    float q8[8];
    lin<32, 8>(Wb + lay::NF0_W, Wb + lay::NF0_B, nf, q8);
    float gate = Wb[lay::NF1_B];
    for (int k = 0; k < 8; ++k) { q8[k] = elu_f(q8[k]); gate = fmaf(Wb[lay::NF1_W + k], q8[k], gate); }
    stv<8>(c.tr, R_Q8, r, q8);
    c.tr.at(R_SG, r) = sigm(gate);
    // ray_dir_fc (ibrnet.py:248-251, 321-323)
    float r16[16], df[36], rgbf[35];
    lin<4, 16>(Wb + lay::RD0_W, Wb + lay::RD0_B, dd, r16);
    for (int k = 0; k < 16; ++k) r16[k] = elu_f(r16[k]);
    lin<16, 36, 36>(Wb + lay::RD1_W, Wb + lay::RD1_B, r16, df);
    for (int k = 0; k < 35; ++k) df[k] = elu_f(df[k]);
    for (int k = 0; k < 3; ++k) rgbf[k] = rgb[k] + df[k];
    for (int k = 0; k < 32; ++k) rgbf[3 + k] = imf[k] + df[3 + k];
    stv<16>(c.tr, R_R16, r, r16);
    stv<35>(c.tr, R_DF, r, df);
    stv<35>(c.tr, R_RGBF, r, rgbf);
  }
}

// ---- forward, phase b, one point: view pooling #1 (ibrnet.py:324-339) and the view-invariant part of base_fc.0 ----------
NR_HD void point_forward_b(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int rfn = pp.rfn;
  const long long N = (long long)pp.rn * pp.dn;
  float msum = 0.f;
  for (int v = 0; v < rfn; ++v) msum += c.tr.at(R_MASK, (long long)v * N + n);
  float glob[140];
  for (int k = 0; k < 140; ++k) glob[k] = 0.f;
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w1 = c.tr.at(R_MASK, r) / (msum + 1e-8f);
    c.tr.at(R_W1, r) = w1;
    const float w0 = c.tr.at(R_SG, r) * w1;
    for (int f = 0; f < 35; ++f) { const float x = c.tr.at(R_RGBF + f, r); glob[f] += x * w0; glob[70 + f] += x * w1; }
  }
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w1 = c.tr.at(R_W1, r), w0 = c.tr.at(R_SG, r) * w1;
    for (int f = 0; f < 35; ++f) {
      const float x = c.tr.at(R_RGBF + f, r);
      const float d0 = x - glob[f], d1 = x - glob[70 + f];
      glob[35 + f] += w0 * d0 * d0; glob[105 + f] += w1 * d1 * d1;
    }
  }
  stv<140>(c.tp, P_GLOB, n, glob);
  c.tp.at(P_MSUM, n) = msum;
  float hz[64];
  lin<140, 64>(W + lay::HOIST_W, W + lay::HOIST_B, glob, hz);
  stv<64>(c.tp, P_HZ, n, hz);
}

// ---- forward, phase c, one row: base_fc, vis_fc, vis_fc2, rgb_fc logit (ibrnet.py:341-350, 362-365) --------------------
NR_HD void row_forward_c(const Ctx& c, long long r) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const long long N = (long long)pp.rn * pp.dn;
  const long long n = r % N;
  const float* Wd = W + lay::GRP_D1;
  float hz[64];
  ldv<64>(c.tp, P_HZ, n, hz);
  {
    const float mask = c.tr.at(R_MASK, r), w1 = c.tr.at(R_W1, r);
    float in67[67], b1[64], x[32];
    ldv<67>(c.tr, R_RGBF, r, in67);
    lin<67, 64>(W + lay::BASE0_W, nullptr, in67, b1);
    for (int k = 0; k < 64; ++k) b1[k] = elu_f(b1[k] + hz[k]);
    lin<64, 32>(W + lay::BASE1_W, W + lay::BASE1_B, b1, x);
    for (int k = 0; k < 32; ++k) x[k] = elu_f(x[k]);
    stv<64>(c.tr, R_B1, r, b1);
    stv<32>(c.tr, R_X, r, x);
    float u[32], vh[32], xv[33], x2[32];
    for (int k = 0; k < 32; ++k) u[k] = x[k] * w1;
    lin<32, 32>(Wd + lay::VIS0_W, Wd + lay::VIS0_B, u, vh);
    for (int k = 0; k < 32; ++k) vh[k] = elu_f(vh[k]);
    lin<32, 32>(Wd + lay::VIS1_W, Wd + lay::VIS1_B, vh, xv);
    float zl = Wd[lay::VIS1L_B];
    for (int k = 0; k < 32; ++k) { xv[k] = elu_f(xv[k]); zl = fmaf(Wd[lay::VIS1L_W + k], vh[k], zl); }
    xv[32] = elu_f(zl);
    const float visa = sigm(xv[32]) * mask;
    for (int k = 0; k < 32; ++k) x2[k] = x[k] + xv[k];
    stv<32>(c.tr, R_U, r, u); stv<32>(c.tr, R_VH, r, vh); stv<33>(c.tr, R_XV, r, xv); stv<32>(c.tr, R_X2, r, x2);
    c.tr.at(R_VISA, r) = visa;
    float u2[32], wh[32];
    for (int k = 0; k < 32; ++k) u2[k] = x2[k] * visa;
    lin<32, 32>(Wd + lay::V20_W, Wd + lay::V20_B, u2, wh);
    float l2 = Wd[lay::V21_B];
    for (int k = 0; k < 32; ++k) { wh[k] = elu_f(wh[k]); l2 = fmaf(Wd[lay::V21_W + k], wh[k], l2); }
    const float vis2 = sigm(l2) * mask;
    stv<32>(c.tr, R_U2, r, u2); stv<32>(c.tr, R_WH, r, wh);
    c.tr.at(R_VIS2, r) = vis2;
    // rgb_fc (the softmax over the views happens in phase d)
    float cin[37], c1[16], c2[8];
    for (int k = 0; k < 32; ++k) cin[k] = x2[k];
    cin[32] = vis2;
    ldv<4>(c.tr, R_DDC, r, cin + 33);
    lin<37, 16>(Wd + lay::RGB0_W, Wd + lay::RGB0_B, cin, c1);
    for (int k = 0; k < 16; ++k) c1[k] = elu_f(c1[k]);
    lin<16, 8>(Wd + lay::RGB1_W, Wd + lay::RGB1_B, c1, c2);
    float lg = Wd[lay::RGB2_B];
    for (int k = 0; k < 8; ++k) { c2[k] = elu_f(c2[k]); lg = fmaf(Wd[lay::RGB2_W + k], c2[k], lg); }
    if (mask == 0.f) lg = -1e9f;
    stv<16>(c.tr, R_CH1, r, c1); stv<8>(c.tr, R_CH2, r, c2);
    c.tr.at(R_BLEND, r) = lg;
  }
}

// ---- forward, phase d, one point: view pooling #2, geometry_fc, colour blend, attention inputs ------------------------
NR_HD void point_forward_d(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int rfn = pp.rfn;
  const long long N = (long long)pp.rn * pp.dn;
  float vsum = 0.f;
  for (int v = 0; v < rfn; ++v) vsum += c.tr.at(R_VIS2, (long long)v * N + n);
  // view pooling #2 + geometry_fc (ibrnet.py:351-354)
  float gin[65];
  for (int k = 0; k < 65; ++k) gin[k] = 0.f;
  float wsum = 0.f;
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w2 = c.tr.at(R_VIS2, r) / (vsum + 1e-8f);
    wsum += w2;
    for (int f = 0; f < 32; ++f) gin[f] += c.tr.at(R_X2 + f, r) * w2;
  }
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w2 = c.tr.at(R_VIS2, r) / (vsum + 1e-8f);
    for (int f = 0; f < 32; ++f) { const float d0 = c.tr.at(R_X2 + f, r) - gin[f]; gin[32 + f] += w2 * d0 * d0; }
  }
  gin[64] = wsum / float(rfn);
  c.tp.at(P_VSUM, n) = vsum;
  stv<65>(c.tp, P_GIN, n, gin);
  const float* We = W + lay::GRP_D2;
  float gh[64], g16[16];
  lin<65, 64>(We + lay::GEO0_W, We + lay::GEO0_B, gin, gh);
  for (int k = 0; k < 64; ++k) gh[k] = elu_f(gh[k]);
  lin<64, 16>(We + lay::GEO1_W, We + lay::GEO1_B, gh, g16);
  for (int k = 0; k < 16; ++k) g16[k] = elu_f(g16[k]);
  stv<64>(c.tp, P_GH, n, gh);
  stv<16>(c.tp, P_G16, n, g16);

  // softmax blend over the views (ibrnet.py:365-367)
  float mx = -3.0e38f;
  for (int v = 0; v < rfn; ++v) mx = fmaxf(mx, c.tr.at(R_BLEND, (long long)v * N + n));
  float den = 0.f, rgbo[3] = {0.f, 0.f, 0.f};
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float e = expf(c.tr.at(R_BLEND, r) - mx);
    c.tr.at(R_BLEND, r) = e;
    den += e;
  }
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float bl = c.tr.at(R_BLEND, r) / den;
    c.tr.at(R_BLEND, r) = bl;
    for (int k = 0; k < 3; ++k) rgbo[k] += bl * c.tr.at(R_RGB + k, r);
  }
  stv<3>(c.tp, P_RGBO, n, rgbo);

  // attention inputs of this sample (ibrnet.py:356-357, 52-75)
  const int s = int(n % pp.dn);
  float ax[16], q[16], k_[16], vv[16];
  for (int k = 0; k < 16; ++k) ax[k] = g16[k] + pp.pos_enc[s * 16 + k];
  lin<16, 16>(c.Wr + lay::WQ, nullptr, ax, q);
  lin<16, 16>(c.Wr + lay::WK, nullptr, ax, k_);
  lin<16, 16>(c.Wr + lay::WV, nullptr, ax, vv);
  stv<16>(c.tp, P_AX, n, ax); stv<16>(c.tp, P_Q, n, q); stv<16>(c.tp, P_K, n, k_); stv<16>(c.tp, P_V, n, vv);
}

// ---- forward of one sample: attention over the ray, LayerNorm, out_geometry_fc -> alpha ---------------------------
NR_HD void sample_forward(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const int dn = pp.dn;
  const long long n0 = (n / dn) * dn;
  const float* Wr = c.Wr;
  const float nvalid = c.tp.at(P_MSUM, n);
  float q[16], o[16];
  ldv<16>(c.tp, P_Q, n, q);
  for (int k = 0; k < 16; ++k) { q[k] *= 0.5f; o[k] = 0.f; }
  float mxh[4] = {0.f, 0.f, 0.f, 0.f}, denh[4] = {1.f, 1.f, 1.f, 1.f};
  if (nvalid > 1.f) {
    for (int hh = 0; hh < 4; ++hh) mxh[hh] = -3.4e38f;
    for (int t = 0; t < dn; ++t)
      for (int hh = 0; hh < 4; ++hh) {
        float l = 0.f;
        for (int d = 0; d < 4; ++d) l = fmaf(q[4 * hh + d], c.tp.at(P_K + 4 * hh + d, n0 + t), l);
        mxh[hh] = fmaxf(mxh[hh], l);
      }
    for (int hh = 0; hh < 4; ++hh) denh[hh] = 0.f;
    for (int t = 0; t < dn; ++t)
      for (int hh = 0; hh < 4; ++hh) {
        float l = 0.f;
        for (int d = 0; d < 4; ++d) l = fmaf(q[4 * hh + d], c.tp.at(P_K + 4 * hh + d, n0 + t), l);
        const float e = expf(l - mxh[hh]);
        denh[hh] += e;
        for (int d = 0; d < 4; ++d) o[4 * hh + d] = fmaf(e, c.tp.at(P_V + 4 * hh + d, n0 + t), o[4 * hh + d]);
      }
    for (int k = 0; k < 16; ++k) o[k] /= denh[k >> 2];
  } else {   // masked query row: uniform attention (ibrnet.py:20)
    for (int t = 0; t < dn; ++t)
      for (int k = 0; k < 16; ++k) o[k] += c.tp.at(P_V + k, n0 + t);
    for (int k = 0; k < 16; ++k) o[k] *= 1.f / float(dn);
  }
  stv<4>(c.tp, P_AM, n, mxh); stv<4>(c.tp, P_AD, n, denh);
  stv<16>(c.tp, P_O, n, o);
  float z[16], ax[16];
  ldv<16>(c.tp, P_AX, n, ax);
  lin<16, 16>(Wr + lay::WFC, nullptr, o, z);
  float mu = 0.f;
  for (int k = 0; k < 16; ++k) { z[k] += ax[k]; mu += z[k]; }
  mu *= 1.f / 16.f;
  float var = 0.f;
  for (int k = 0; k < 16; ++k) var = fmaf(z[k] - mu, z[k] - mu, var);
  const float rstd = 1.f / sqrtf(var * (1.f / 16.f) + 1e-6f);
  float xh[16], y[16];
  for (int k = 0; k < 16; ++k) { xh[k] = (z[k] - mu) * rstd; y[k] = xh[k] * Wr[lay::LN_W + k] + Wr[lay::LN_B + k]; }
  stv<16>(c.tp, P_XH, n, xh); c.tp.at(P_RSTD, n) = rstd; stv<16>(c.tp, P_Y, n, y);
  float t16[16];
  lin<16, 16>(Wr + lay::OG0_W, Wr + lay::OG0_B, y, t16);
  float sg = Wr[lay::OG1_B];
  for (int k = 0; k < 16; ++k) { t16[k] = elu_f(t16[k]); sg = fmaf(Wr[lay::OG1_W + k], t16[k], sg); }
  stv<16>(c.tp, P_T16, n, t16);
  sg = fmaxf(sg, 0.f);
  if (nvalid < 1.f) sg = 0.f;
  c.tp.at(P_SIG, n) = sg;
  c.tp.at(P_ALPHA, n) = 1.f - expf(-sg);
}

// ---- one ray: compositing forward and backward (renderer.py:157-166, 201-202; render_ops.py:72-80) -----------------
NR_HD void ray_backward(const Ctx& c, long long ray) {
  const NrPassParams& pp = c.p;
  const int dn = pp.dn;
  const long long n0 = ray * dn;
  float dpix[3] = {0.f, 0.f, 0.f};
  if (c.d_pix) for (int k = 0; k < 3; ++k) dpix[k] = c.d_pix[ray * 3 + k];
  const float ddep = c.d_depth ? c.d_depth[ray] : 0.f;
  // forward sweep: transmittance T_i in front of every sample, parked in the GP_DELTA slot (free until
  // sample_backward_q writes the attention deltas there); dividing the total transmittance back out would be unstable
  float T = 1.f;
  for (int i = 0; i < dn; ++i) {
    c.gp.at(GP_DELTA, n0 + i) = T;
    T *= 1.f - c.tp.at(P_ALPHA, n0 + i) + 1e-10f;
  }
  float S = 0.f;   // sum over k > i of dH_k * hit_k
  for (int i = dn - 1; i >= 0; --i) {
    const long long n = n0 + i;
    const float a = c.tp.at(P_ALPHA, n), Ti = c.gp.at(GP_DELTA, n);
    const float hit = a * Ti;
    float dH = ddep * pp.que_depth[n];
    if (c.d_hit) dH += c.d_hit[n];
    float drgb[3];
    for (int k = 0; k < 3; ++k) { dH = fmaf(dpix[k], c.tp.at(P_RGBO + k, n), dH); drgb[k] = hit * dpix[k]; }
    stv<3>(c.gp, GP_DRGB, n, drgb);
    const float f = 1.f - a + 1e-10f;
    const float dalpha = dH * Ti - S / f;
    S = fmaf(dH, hit, S);
    const float sg = c.tp.at(P_SIG, n);
    // sigma = relu(raw), zeroed where no view sees the point; alpha = 1 - exp(-sigma)
    float draw = dalpha * (1.f - a);
    if (!(sg > 0.f)) draw = 0.f;
    c.gp.at(GP_OG1, n) = draw;
  }
}

// ---- one sample, query side: out_geometry_fc, LayerNorm, fc, attention wrt q ---------------------------------------
NR_HD void sample_backward_q(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const int dn = pp.dn;
  const long long n0 = (n / dn) * dn;
  const float* Wr = c.Wr;
  const float draw = c.gp.at(GP_OG1, n);
  float t16[16], dz0[16], dy[16];
  ldv<16>(c.tp, P_T16, n, t16);
  for (int k = 0; k < 16; ++k) dz0[k] = draw * Wr[lay::OG1_W + k] * elu_g(t16[k]);
  stv<16>(c.gp, GP_OG0, n, dz0);
  lin_t<16, 16>(Wr + lay::OG0_W, dz0, dy);
  stv<16>(c.gp, GP_DLNY, n, dy);
  float xh[16], dxh[16], m1 = 0.f, m2 = 0.f;
  ldv<16>(c.tp, P_XH, n, xh);
  for (int k = 0; k < 16; ++k) { dxh[k] = dy[k] * Wr[lay::LN_W + k]; m1 += dxh[k]; m2 = fmaf(dxh[k], xh[k], m2); }
  m1 *= 1.f / 16.f; m2 *= 1.f / 16.f;
  const float rstd = c.tp.at(P_RSTD, n);
  float dzl[16], dO[16];
  for (int k = 0; k < 16; ++k) dzl[k] = rstd * (dxh[k] - m1 - xh[k] * m2);
  stv<16>(c.gp, GP_DFC, n, dzl);
  lin_t<16, 16>(Wr + lay::WFC, dzl, dO);
  stv<16>(c.gp, GP_DO, n, dO);
  float dq[16], delta[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < 16; ++k) dq[k] = 0.f;
  if (c.tp.at(P_MSUM, n) > 1.f) {
    float q[16], mxh[4], denh[4];
    ldv<16>(c.tp, P_Q, n, q); ldv<4>(c.tp, P_AM, n, mxh); ldv<4>(c.tp, P_AD, n, denh);
    for (int k = 0; k < 16; ++k) q[k] *= 0.5f;
    for (int t = 0; t < dn; ++t)
      for (int hh = 0; hh < 4; ++hh) {
        float l = 0.f, dP = 0.f;
        for (int d = 0; d < 4; ++d) {
          l = fmaf(q[4 * hh + d], c.tp.at(P_K + 4 * hh + d, n0 + t), l);
          dP = fmaf(dO[4 * hh + d], c.tp.at(P_V + 4 * hh + d, n0 + t), dP);
        }
        delta[hh] = fmaf(expf(l - mxh[hh]) / denh[hh], dP, delta[hh]);
      }
    for (int t = 0; t < dn; ++t)
      for (int hh = 0; hh < 4; ++hh) {
        float l = 0.f, dP = 0.f;
        for (int d = 0; d < 4; ++d) {
          l = fmaf(q[4 * hh + d], c.tp.at(P_K + 4 * hh + d, n0 + t), l);
          dP = fmaf(dO[4 * hh + d], c.tp.at(P_V + 4 * hh + d, n0 + t), dP);
        }
        const float dS = expf(l - mxh[hh]) / denh[hh] * (dP - delta[hh]);
        for (int d = 0; d < 4; ++d) dq[4 * hh + d] = fmaf(dS * 0.5f, c.tp.at(P_K + 4 * hh + d, n0 + t), dq[4 * hh + d]);
      }
  }
  stv<16>(c.gp, GP_DQ, n, dq);
  stv<4>(c.gp, GP_DELTA, n, delta);
}

// ---- one sample, key side (dK, dV over all queries of the ray), then the projections back to the geometry feature ---
NR_HD void sample_backward_kv(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const int dn = pp.dn;
  const long long n0 = (n / dn) * dn;
  const float* Wr = c.Wr;
  float kt[16], vt[16], dK[16], dV[16];
  ldv<16>(c.tp, P_K, n, kt); ldv<16>(c.tp, P_V, n, vt);
  for (int k = 0; k < 16; ++k) { dK[k] = 0.f; dV[k] = 0.f; }
  for (int s = 0; s < dn; ++s) {
    const long long m = n0 + s;
    float dO[16];
    ldv<16>(c.gp, GP_DO, m, dO);
    if (c.tp.at(P_MSUM, m) > 1.f) {
      for (int hh = 0; hh < 4; ++hh) {
        float l = 0.f, dP = 0.f, qh[4];
        for (int d = 0; d < 4; ++d) {
          qh[d] = c.tp.at(P_Q + 4 * hh + d, m) * 0.5f;
          l = fmaf(qh[d], kt[4 * hh + d], l);
          dP = fmaf(dO[4 * hh + d], vt[4 * hh + d], dP);
        }
        const float P = expf(l - c.tp.at(P_AM + hh, m)) / c.tp.at(P_AD + hh, m);
        const float dS = P * (dP - c.gp.at(GP_DELTA + hh, m));
        for (int d = 0; d < 4; ++d) { dK[4 * hh + d] = fmaf(dS, qh[d], dK[4 * hh + d]); dV[4 * hh + d] = fmaf(P, dO[4 * hh + d], dV[4 * hh + d]); }
      }
    } else {
      for (int k = 0; k < 16; ++k) dV[k] += dO[k] * (1.f / float(dn));
    }
  }
  stv<16>(c.gp, GP_DK, n, dK); stv<16>(c.gp, GP_DV, n, dV);
  float dq[16], dax[16], t[16];
  ldv<16>(c.gp, GP_DQ, n, dq);
  ldv<16>(c.gp, GP_DFC, n, dax);                 // residual branch
  lin_t<16, 16>(Wr + lay::WQ, dq, t);
  for (int k = 0; k < 16; ++k) dax[k] += t[k];
  lin_t<16, 16>(Wr + lay::WK, dK, t);
  for (int k = 0; k < 16; ++k) dax[k] += t[k];
  lin_t<16, 16>(Wr + lay::WV, dV, t);
  for (int k = 0; k < 16; ++k) dax[k] += t[k];
  stv<16>(c.gp, GP_DG16, n, dax);
}

// ---- backward, phase a, one point: geometry_fc, what view pooling #2 and the colour blend hand to their rows --------------
NR_HD void point_backward_a(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int rfn = pp.rfn;
  const long long N = (long long)pp.rn * pp.dn;
  const float* We = W + lay::GRP_D2;

  // geometry_fc
  float dgin[65];
  {
    float g16[16], dz1[16], gh[64], dgh[64];
    ldv<16>(c.tp, P_G16, n, g16); ldv<16>(c.gp, GP_DG16, n, dz1);
    for (int k = 0; k < 16; ++k) dz1[k] *= elu_g(g16[k]);
    stv<16>(c.gp, GP_GEO1, n, dz1);
    lin_t<64, 16>(We + lay::GEO1_W, dz1, dgh);
    ldv<64>(c.tp, P_GH, n, gh);
    for (int k = 0; k < 64; ++k) dgh[k] *= elu_g(gh[k]);
    stv<64>(c.gp, GP_GEO0, n, dgh);
    lin_t<65, 64>(We + lay::GEO0_W, dgh, dgin);
  }
  // view pooling #2: gradient of the mean includes the variance's dependence on it
  float gin[65];
  ldv<65>(c.tp, P_GIN, n, gin);
  const float vsum = c.tp.at(P_VSUM, n), vden = vsum + 1e-8f;
  float dmt[32];
  for (int f = 0; f < 32; ++f) dmt[f] = 0.f;
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w2 = c.tr.at(R_VIS2, r) / vden;
    for (int f = 0; f < 32; ++f) dmt[f] += w2 * (c.tr.at(R_X2 + f, r) - gin[f]);
  }
  for (int f = 0; f < 32; ++f) dmt[f] = dgin[f] - 2.f * dgin[32 + f] * dmt[f];
  float dw2sum = 0.f;   // sum_u dw2_u * vis2_u
  float drgbo[3];
  ldv<3>(c.gp, GP_DRGB, n, drgbo);
  float bsum = 0.f;     // sum_u blend_u * dblend_u
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    float dw2 = dgin[64] / float(rfn);
    for (int f = 0; f < 32; ++f) {
      const float x = c.tr.at(R_X2 + f, r), d0 = x - gin[f];
      dw2 += dmt[f] * x + dgin[32 + f] * d0 * d0;
    }
    dw2sum += dw2 * c.tr.at(R_VIS2, r);
    float db = 0.f;
    for (int k = 0; k < 3; ++k) db += drgbo[k] * c.tr.at(R_RGB + k, r);
    bsum += c.tr.at(R_BLEND, r) * db;
  }
  stv<65>(c.gp, GP_DGIN, n, dgin);
  stv<32>(c.gp, GP_DMT, n, dmt);
  c.gp.at(GP_DW2SUM, n) = dw2sum;
  c.gp.at(GP_BSUM, n) = bsum;
}

// ---- backward, phase b, one row: rgb_fc, vis_fc2, vis_fc, base_fc (down to base_fc.0's pre-activation gradient) ---------
NR_HD void row_backward_b(const Ctx& c, long long r) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int rfn = pp.rfn;
  const long long N = (long long)pp.rn * pp.dn;
  const long long n = r % N;
  const float* Wd = W + lay::GRP_D1;
  float dgin[65], gin[65], dmt[32], drgbo[3];
  ldv<65>(c.gp, GP_DGIN, n, dgin); ldv<65>(c.tp, P_GIN, n, gin); ldv<32>(c.gp, GP_DMT, n, dmt); ldv<3>(c.gp, GP_DRGB, n, drgbo);
  const float dw2sum = c.gp.at(GP_DW2SUM, n), bsum = c.gp.at(GP_BSUM, n);
  const float vden = c.tp.at(P_VSUM, n) + 1e-8f;
  {
    const float mask = c.tr.at(R_MASK, r), w1 = c.tr.at(R_W1, r);
    const float vis2 = c.tr.at(R_VIS2, r), w2 = vis2 / vden;
    float dx2[32];
    float dvis2;
    {
      float dw2 = dgin[64] / float(rfn);
      for (int f = 0; f < 32; ++f) {
        const float x = c.tr.at(R_X2 + f, r), d0 = x - gin[f];
        dw2 += dmt[f] * x + dgin[32 + f] * d0 * d0;
        dx2[f] = w2 * (dmt[f] + 2.f * dgin[32 + f] * d0);
      }
      dvis2 = dw2 / vden - dw2sum / (vden * vden);
    }
    // softmax blend -> rgb_fc
    {
      float db = 0.f;
      for (int k = 0; k < 3; ++k) db += drgbo[k] * c.tr.at(R_RGB + k, r);
      const float bl = c.tr.at(R_BLEND, r);
      const float dlogit = mask == 0.f ? 0.f : bl * (db - bsum);
      c.gr.at(G_C2, r) = dlogit;
      float c2[8], dz1[8], c1[16], dc1[16], dcin[37];
      ldv<8>(c.tr, R_CH2, r, c2); ldv<16>(c.tr, R_CH1, r, c1);
      for (int k = 0; k < 8; ++k) dz1[k] = dlogit * Wd[lay::RGB2_W + k] * elu_g(c2[k]);
      stv<8>(c.gr, G_C1, r, dz1);
      lin_t<16, 8>(Wd + lay::RGB1_W, dz1, dc1);
      for (int k = 0; k < 16; ++k) dc1[k] *= elu_g(c1[k]);
      stv<16>(c.gr, G_C0, r, dc1);
      lin_t<37, 16>(Wd + lay::RGB0_W, dc1, dcin);
      for (int k = 0; k < 32; ++k) dx2[k] += dcin[k];
      dvis2 += dcin[32];
    }
    // vis_fc2
    float dvisa = 0.f;
    {
      const float dl2 = dvis2 * vis2 * (1.f - vis2) * mask;
      c.gr.at(G_V21, r) = dl2;
      float wh[32], dz[32], du2[32];
      ldv<32>(c.tr, R_WH, r, wh);
      for (int k = 0; k < 32; ++k) dz[k] = dl2 * Wd[lay::V21_W + k] * elu_g(wh[k]);
      stv<32>(c.gr, G_V20, r, dz);
      lin_t<32, 32>(Wd + lay::V20_W, dz, du2);
      const float visa = c.tr.at(R_VISA, r);
      for (int k = 0; k < 32; ++k) { dvisa = fmaf(du2[k], c.tr.at(R_X2 + k, r), dvisa); dx2[k] = fmaf(du2[k], visa, dx2[k]); }
    }
    // vis_fc (x2 = x + xv[0:32]; visa = sigmoid(xv[32]) * mask)
    float dx[32];
    {
      const float visa = c.tr.at(R_VISA, r);
      float xv[33], dzv[33], vh[32], dvh[32], du[32];
      ldv<33>(c.tr, R_XV, r, xv);
      for (int k = 0; k < 32; ++k) { dx[k] = dx2[k]; dzv[k] = dx2[k] * elu_g(xv[k]); }
      dzv[32] = dvisa * visa * (1.f - visa) * mask * elu_g(xv[32]);
      stv<33>(c.gr, G_V1, r, dzv);
      lin_t<32, 32>(Wd + lay::VIS1_W, dzv, dvh);
      ldv<32>(c.tr, R_VH, r, vh);
      for (int k = 0; k < 32; ++k) dvh[k] = (dvh[k] + Wd[lay::VIS1L_W + k] * dzv[32]) * elu_g(vh[k]);
      stv<32>(c.gr, G_V0, r, dvh);
      lin_t<32, 32>(Wd + lay::VIS0_W, dvh, du);
      for (int k = 0; k < 32; ++k) dx[k] = fmaf(du[k], w1, dx[k]);
    }
    // base_fc
    {
      float x[32], b1[64], db1[64];
      ldv<32>(c.tr, R_X, r, x);
      for (int k = 0; k < 32; ++k) dx[k] *= elu_g(x[k]);
      stv<32>(c.gr, G_B1, r, dx);
      lin_t<64, 32>(W + lay::BASE1_W, dx, db1);
      ldv<64>(c.tr, R_B1, r, b1);
      for (int k = 0; k < 64; ++k) db1[k] *= elu_g(b1[k]);
      stv<64>(c.gr, G_B0, r, db1);
    }
  }
}

// ---- backward, phase c, one point: gradient of the pooled statistics #1 --------------------------------------------------
NR_HD void point_backward_c(const Ctx& c, long long n) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int rfn = pp.rfn;
  const long long N = (long long)pp.rn * pp.dn;
  float dzsum[64];
  for (int k = 0; k < 64; ++k) dzsum[k] = 0.f;
  for (int v = 0; v < rfn; ++v)
    for (int k = 0; k < 64; ++k) dzsum[k] += c.gr.at(G_B0 + k, (long long)v * N + n);
  stv<64>(c.gp, GP_B0SUM, n, dzsum);
  float dglob[140], glob[140];
  lin_t<140, 64>(W + lay::HOIST_W, dzsum, dglob);
  ldv<140>(c.tp, P_GLOB, n, glob);
  // view pooling #1: two weight sets (w0 = sigmoid(gate) * w1, w1 = mask / sum)
  float dm0[35], dm1[35];
  for (int f = 0; f < 35; ++f) { dm0[f] = 0.f; dm1[f] = 0.f; }
  for (int v = 0; v < rfn; ++v) {
    const long long r = (long long)v * N + n;
    const float w1 = c.tr.at(R_W1, r), w0 = c.tr.at(R_SG, r) * w1;
    for (int f = 0; f < 35; ++f) {
      const float x = c.tr.at(R_RGBF + f, r);
      dm0[f] += w0 * (x - glob[f]); dm1[f] += w1 * (x - glob[70 + f]);
    }
  }
  for (int f = 0; f < 35; ++f) { dm0[f] = dglob[f] - 2.f * dglob[35 + f] * dm0[f]; dm1[f] = dglob[70 + f] - 2.f * dglob[105 + f] * dm1[f]; }
  stv<140>(c.gp, GP_DGLOB, n, dglob);
  stv<35>(c.gp, GP_DM0, n, dm0);
  stv<35>(c.gp, GP_DM1, n, dm1);
}

// ---- backward, phase d, one row: view pooling #1, neuray_fc, ray_dir_fc, prob_embed, compute_prob, heads, scatter ----------
NR_HD void row_backward_d(const Ctx& c, long long r) {
  const NrPassParams& pp = c.p;
  const float* __restrict__ W = c.W;
  const int fw = pp.fw;
  const long long N = (long long)pp.rn * pp.dn;
  const long long n = r % N;
  const float* Wb = W + lay::GRP_B;
  float dglob[140], glob[140], dm0[35], dm1[35];
  ldv<140>(c.gp, GP_DGLOB, n, dglob); ldv<140>(c.tp, P_GLOB, n, glob); ldv<35>(c.gp, GP_DM0, n, dm0); ldv<35>(c.gp, GP_DM1, n, dm1);
  {
    const float mask = c.tr.at(R_MASK, r), w1 = c.tr.at(R_W1, r), sg = c.tr.at(R_SG, r), w0 = sg * w1;
    float dz0[64], din[67];
    ldv<64>(c.gr, G_B0, r, dz0);
    lin_t<67, 64>(W + lay::BASE0_W, dz0, din);          // d rgb_feat (35) | d neuray_feat (32)
    float dw0 = 0.f;
    for (int f = 0; f < 35; ++f) {
      const float x = c.tr.at(R_RGBF + f, r), d0 = x - glob[f], d1 = x - glob[70 + f];
      din[f] += w0 * (dm0[f] + 2.f * dglob[35 + f] * d0) + w1 * (dm1[f] + 2.f * dglob[105 + f] * d1);
      dw0 += dm0[f] * x + dglob[35 + f] * d0 * d0;
    }
    // neuray_fc
    float* dnf = din + 35;
    {
      const float dgate = dw0 * w1 * sg * (1.f - sg);
      c.gr.at(G_NF1, r) = dgate;
      float q8[8], dz[8], t[32];
      ldv<8>(c.tr, R_Q8, r, q8);
      for (int k = 0; k < 8; ++k) dz[k] = dgate * Wb[lay::NF1_W + k] * elu_g(q8[k]);
      stv<8>(c.gr, G_NF0, r, dz);
      lin_t<32, 8>(Wb + lay::NF0_W, dz, t);
      for (int k = 0; k < 32; ++k) dnf[k] += t[k];
    }
    // ray_dir_fc (rgb_feat = [rgb, img_feats] + elu(...))
    float dimf[32];
    {
      float df[35], dz[36], r16[16], dr[16];
      ldv<35>(c.tr, R_DF, r, df);
      for (int k = 0; k < 35; ++k) dz[k] = din[k] * elu_g(df[k]);
      dz[35] = 0.f;
      stv<35>(c.gr, G_RD1, r, dz);
      lin_t<16, 36, 36>(Wb + lay::RD1_W, dz, dr);
      ldv<16>(c.tr, R_R16, r, r16);
      for (int k = 0; k < 16; ++k) dr[k] *= elu_g(r16[k]);
      stv<16>(c.gr, G_RD0, r, dr);
      for (int k = 0; k < 32; ++k) dimf[k] = din[3 + k];
    }
    // prob_embed
    float drf[32], dhitn, dvisn;
    {
      stv<32>(c.gr, G_PE1, r, dnf);
      float p1[32], dp1[32], de[34];
      lin_t<32, 32>(Wb + lay::PE1_W, dnf, dp1);
      ldv<32>(c.tr, R_P1, r, p1);
      for (int k = 0; k < 32; ++k) dp1[k] = p1[k] > 0.f ? dp1[k] : 0.f;
      stv<32>(c.gr, G_PE0, r, dp1);
      lin_t<34, 32>(Wb + lay::PE0_W, dp1, de);
      for (int k = 0; k < 32; ++k) drf[k] = de[k];
      dhitn = de[32]; dvisn = de[33];
    }
    // compute_prob
    float dho[4][2];
    {
      Mix m;
      float c0[2], c1[2];
      ldv<2>(c.tr, R_MEAN, r, m.mean); ldv<2>(c.tr, R_VAR, r, m.var); ldv<2>(c.tr, R_C0, r, c0); ldv<2>(c.tr, R_C1, r, c1);
      m.aw = c.tr.at(R_AW, r); m.visd = c.tr.at(R_VISD, r);
      MixGrad dm = {};
      bin_bwd(m, c.tr.at(R_TLO, r), c.tr.at(R_THI, r), c0, c1, 2.f * dhitn * mask, 2.f * dvisn * mask, dm);
      mix_bwd(m, dm, pp.var_bias, pp.use_vis, dho);
    }
    // dist decoder heads
    for (int hd = 0; hd < c.n_heads; ++hd) {
      stv<2>(c.gr, G_DD2 + 2 * hd, r, dho[hd]);
      float h2[32], h1[32];
      ldv<32>(c.tr, R_H2 + 32 * hd, r, h2);
      ldv<32>(c.tr, R_H1 + 32 * hd, r, h1);
      head_bwd(W + lay::DD_HEAD + hd * lay::DD_HEAD_STRIDE, nullptr, h1, h2, dho[hd], drf, nullptr, &c.gr, r, hd);
    }
    for (int hd = c.n_heads; hd < 4; ++hd) {   // unused head: zero rows for the GEMMs
      float z[32];
      for (int k = 0; k < 32; ++k) z[k] = 0.f;
      stv<2>(c.gr, G_DD2 + 2 * hd, r, z); stv<32>(c.gr, G_DD1 + 32 * hd, r, z); stv<32>(c.gr, G_DD0 + 32 * hd, r, z);
    }
    // scatter into the channel-last map gradient (bilinear taps; masked rows carry no gradient)
    int tcode;
    { const float tc = c.tr.at(R_TCODE, r); memcpy(&tcode, &tc, 4); }
    if (tcode >= 0 && c.d_feat != nullptr) {
      float tw[4];
      ldv<4>(c.tr, R_TW, r, tw);
      float* base = c.d_feat + (tcode & ~63);
      const int dxo = (tcode & 1) << 6, dyo = (tcode & 2) ? fw * 64 : 0;
      const int off[4] = {0, dxo, dyo, dyo + dxo};
      for (int t = 0; t < 4; ++t) {
        if (tw[t] == 0.f) continue;
        for (int k = 0; k < 32; k += 4) {          // 16 vector reductions per tap instead of 64 scalar ones
          atomic_add4(base + off[t] + k, drf[k] * tw[t], drf[k + 1] * tw[t], drf[k + 2] * tw[t], drf[k + 3] * tw[t]);
          atomic_add4(base + off[t] + 32 + k, dimf[k] * tw[t], dimf[k + 1] * tw[t], dimf[k + 2] * tw[t], dimf[k + 3] * tw[t]);
        }
      }
    }
  }
}


// ---- predict_self_hit_prob (reference renderer.py:137-155; dist_decoder.py compute_prob with is_ref=False) ---------------
// The query view's own ray_feats (NCHW [32,fh,fw]) sampled at the ray's pixel, decoded by the pass' dist decoder, and
// turned into per-sample hit probabilities along the ray.  One routine does forward and (optionally) backward for one
// ray: d_hit == nullptr -> forward only.  Weight gradients are added to dW in the packed w_point layout (512 rays only:
// plain atomics), the feature-map gradient to d_map (NCHW).
typedef NrSelfParams SelfCtx;   // include/neuray_b200.h

NR_HD void self_hit_prob_ray(const SelfCtx& c, long long ray) {
  const int dn = c.dn, fh = c.fh, fw = c.fw, n_heads = c.use_vis ? 4 : 3;
  const float* __restrict__ W = c.w_point;
  const Taps tap = border_taps(c.coords[2 * ray], c.coords[2 * ray + 1], c.h, c.w, fh, fw, fh == c.h && fw == c.w);
  float rf[32];
  for (int k = 0; k < 32; ++k) rf[k] = bilinear(c.map + (size_t)k * fh * fw, fw, tap);
  float h1[4][32], h2[4][32], ho[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
  for (int hd = 0; hd < n_heads; ++hd) head_fwd(W + lay::DD_HEAD + hd * lay::DD_HEAD_STRIDE, rf, h1[hd], h2[hd], ho[hd], nullptr, 0, 0);
  const Mix m = mix_fwd(ho, c.var_bias, c.use_vis);
  // bin edges in normalised inverse depth (get_near_far_points, is_ref=False: midpoints, half intervals at the ends)
  const float a = -1.f / c.depth_range[0], b = -1.f / c.depth_range[1];
  const float* qd = c.que_depth + ray * dn;
  auto tn = [&](int s) { return (-1.f / fmaxf(qd[s], 1e-5f) - a) / (b - a); };
  MixGrad dm = {};
  for (int s = 0; s < dn; ++s) {
    const float t = tn(s);
    const float lo = s == 0 ? t - (tn(1) - t) * 0.5f : (tn(s - 1) + t) * 0.5f;
    const float hi = s == dn - 1 ? t + 1e6f * 0.5f : (t + tn(s + 1)) * 0.5f;
    float c0[2], c1[2], hit, visb;
    bin_fwd(m, lo, hi, c0, c1, hit, visb);
    c.hit[ray * dn + s] = hit;
    if (c.d_hit != nullptr) bin_bwd(m, lo, hi, c0, c1, c.d_hit[ray * dn + s], 0.f, dm);
  }
  if (c.d_hit == nullptr) return;
  float dho[4][2];
  mix_bwd(m, dm, c.var_bias, c.use_vis, dho);
  float drf[32];
  for (int k = 0; k < 32; ++k) drf[k] = 0.f;
  for (int hd = 0; hd < n_heads; ++hd) {
    const int base = lay::DD_HEAD + hd * lay::DD_HEAD_STRIDE;
    head_bwd(W + base, rf, h1[hd], h2[hd], dho[hd], drf, c.d_w_point + base, nullptr, 0, 0);
  }
  if (c.d_map != nullptr) {
    const int off[4] = {tap.y0 * fw + tap.x0, tap.y0 * fw + tap.x1, tap.y1 * fw + tap.x0, tap.y1 * fw + tap.x1};
    for (int k = 0; k < 32; ++k) {
      float* dmap = c.d_map + (size_t)k * fh * fw;
      for (int q = 0; q < 4; ++q) atomic_add(dmap + off[q], drf[k] * tap.w[q]);
    }
  }
}

}  // namespace tr
}  // namespace nr

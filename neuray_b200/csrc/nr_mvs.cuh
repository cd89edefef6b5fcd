// CostVolumeInitNet's frozen MVSNet (SURVEY.md 8(f) row f4): reference network/mvsnet/mvsnet.py:7-151 (FeatureNet, CostRegNet,
// construct_cost_volume_with_src), network/mvsnet/modules.py:25-70 (homo_warp, depth_regression), network/init_net.py:113-168
// (construct_cost_volume_with_src, get_depth_vals).  Inference only, weights frozen (init_net.py:214-216).
//
// Everything is channel-last: feature maps [N,H,W,C], volumes [D,H,W,C] (one reference view at a time, like the reference's
// eval loop, init_net.py:146: batch_num = 1).  The convolutions here have 3..64 channels on at most 64 x 200 x 200 voxels:
// direct convolutions, one thread per output voxel with all Cout accumulators in registers and warp-uniform (broadcast)
// weight reads; BatchNorm (eval: running statistics, the frozen checkpoint) is folded into a per-channel scale / shift at
// pack time.  The per-voxel routines are __host__ __device__: tests/cpu_harness/mvs_cpu_harness.cu runs the same graph on the
// host against the reference's modules.
#pragma once
#include <math.h>

#include "nr_common.cuh"

#ifndef NR_HD
#define NR_HD __host__ __device__ __forceinline__
#endif

namespace nr {
namespace mvs {

// One direct convolution (2-D when D == 1, kd == 1) or transposed convolution over a channel-last volume.
//   conv:   y[do,ho,wo,:] = sum over taps, cin of x[do*s - pd + kd, ...] w[tap][cin][:]           zero padding
//   deconv: ConvTranspose3d(k 3, stride 2, padding 1, output_padding 1): y[o] gathers x[i] where o = 2 i - 1 + k
// then  y = y * scale + shift  (folded BatchNorm, or bias: scale 1), leaky ReLU (slope, 1 = none), + skip.
struct ConvP {
  const float* x; const float* w; const float* scale; const float* shift; const float* skip; float* y;
  int D, H, W, Cin;              // input volume
  int Do, Ho, Wo, Cout;          // output volume
  int kd, kh, kw, sd, sh, sw, pd, ph, pw;
  int transposed;
  float slope;                   // leaky ReLU slope (1: linear)
  long long y_sd, y_sh, y_sw;    // output strides in floats (element (d,h,w,c) at y[d*y_sd + h*y_sh + w*y_sw + c]); skip uses the same
  const float* in_mean; const float* in_istd;   // first layer: input channels are (x - mean) * istd inside the image, 0 in the padding
};

// output channels per thread: all of them up to 8, groups of 8 beyond
NR_HD int group_size(int Cout) { return Cout <= 8 ? Cout : 8; }

// acc[0..COUT) += xv * w[0..COUT): the weights of one (tap, input channel) are COUT contiguous floats read by every lane of a warp
// from the same address (one broadcast transaction); 128-bit loads keep it at one load instruction per four FMAs
template <int COUT>
NR_HD void axpy_row(float xv, const float* __restrict__ wr, float (&acc)[COUT]) {
  if constexpr (COUT % 4 == 0) {
    const float4* __restrict__ w4 = reinterpret_cast<const float4*>(wr);
#pragma unroll
    for (int j = 0; j < COUT / 4; ++j) {
      const float4 w = w4[j];
      acc[4 * j] = fmaf(xv, w.x, acc[4 * j]); acc[4 * j + 1] = fmaf(xv, w.y, acc[4 * j + 1]);
      acc[4 * j + 2] = fmaf(xv, w.z, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(xv, w.w, acc[4 * j + 3]);
    }
  } else {
#pragma unroll
    for (int o = 0; o < COUT; ++o) acc[o] = fmaf(xv, wr[o], acc[o]);
  }
}

// One thread = one output voxel x one group of COUT consecutive output channels (group g of p.Cout / COUT): the layers with 32 / 64
// outputs sit on 25 600 / 3 200 voxels, far too few threads for the machine if a thread carried all of a voxel's outputs
// (a thread carrying all outputs of a voxel ran ~110 000 serial FMAs on a few dozen CTAs).
template <int COUT>
NR_HD void conv_voxel(const ConvP& p, long long v, int g, float (&acc)[COUT]) {
  const int wo = int(v % p.Wo);
  const long long t = v / p.Wo;
  const int ho = int(t % p.Ho), dz = int(t / p.Ho);
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = 0.f;
  // transposed (stride 2): output o gathers input i through tap k where o + pad - k = 2 i, i.e. only taps of one parity
  const int kd0 = p.transposed ? (dz + p.pd) % p.sd : 0, kdstep = p.transposed ? p.sd : 1;
  const int kh0 = p.transposed ? (ho + p.ph) % p.sh : 0, khstep = p.transposed ? p.sh : 1;
  const int kw0 = p.transposed ? (wo + p.pw) % p.sw : 0, kwstep = p.transposed ? p.sw : 1;
  const bool vec_x = (p.Cin % 4 == 0) && p.in_mean == nullptr;
  for (int kd = kd0; kd < p.kd; kd += kdstep) {
    const int di = p.transposed ? (dz + p.pd - kd) / p.sd : dz * p.sd - p.pd + kd;
    if (di < 0 || di >= p.D) continue;
    for (int kh = kh0; kh < p.kh; kh += khstep) {
      const int hi = p.transposed ? (ho + p.ph - kh) / p.sh : ho * p.sh - p.ph + kh;
      if (hi < 0 || hi >= p.H) continue;
      for (int kw = kw0; kw < p.kw; kw += kwstep) {
        const int wi = p.transposed ? (wo + p.pw - kw) / p.sw : wo * p.sw - p.pw + kw;
        if (wi < 0 || wi >= p.W) continue;
        const float* __restrict__ xin = p.x + (((long long)di * p.H + hi) * p.W + wi) * p.Cin;
        const float* __restrict__ wt = p.w + (long long)((kd * p.kh + kh) * p.kw + kw) * p.Cin * p.Cout + g * COUT;
        if (vec_x) {
          const float4* __restrict__ x4 = reinterpret_cast<const float4*>(xin);
          for (int c4 = 0; c4 < p.Cin / 4; ++c4) {
            const float4 xv = x4[c4];
            const float* wr = wt + 4 * c4 * p.Cout;
            axpy_row<COUT>(xv.x, wr, acc); axpy_row<COUT>(xv.y, wr + p.Cout, acc);
            axpy_row<COUT>(xv.z, wr + 2 * p.Cout, acc); axpy_row<COUT>(xv.w, wr + 3 * p.Cout, acc);
          }
        } else {
          for (int c = 0; c < p.Cin; ++c) {
            float xv = xin[c];
            if (p.in_mean != nullptr) xv = (xv - p.in_mean[c]) * p.in_istd[c];
            axpy_row<COUT>(xv, wt + c * p.Cout, acc);
          }
        }
      }
    }
  }
  const long long yo = (long long)dz * p.y_sd + (long long)ho * p.y_sh + (long long)wo * p.y_sw + g * COUT;
#pragma unroll
  for (int o = 0; o < COUT; ++o) {
    float r = acc[o] * p.scale[g * COUT + o] + p.shift[g * COUT + o];
    r = r >= 0.f ? r : r * p.slope;
    if (p.skip != nullptr) r += p.skip[yo + o];
    p.y[yo + o] = r;
  }
}

// ---- cost volume (mvsnet.py:124-141, modules.py:25-70): variance over {reference feature, warped source features} ------------
struct VolumeP {
  const float* ref_feat;       // [h,w,32] of this reference view
  const float* src_feats;      // [sn,h,w,32]
  const int* nn_ids;           // [nn] source views of this reference view
  const float* transforms;     // [nn][12]: rows of R | T of src_proj @ inv(ref_proj), row-major 3 x 4
  const float* depth_vals;     // [dn]
  float* vol;                  // [dn,h,w,32]
  int nn, dn, h, w;
};
NR_HD void volume_voxel(const VolumeP& p, long long v) {
  const int x = int(v % p.w);
  const long long t = v / p.w;
  const int y = int(t % p.h), d = int(t / p.h);
  const float4* __restrict__ rf = reinterpret_cast<const float4*>(p.ref_feat + ((long long)y * p.w + x) * 32);
  float s[32], q[32];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4 f = rf[c];
    s[4 * c] = f.x; s[4 * c + 1] = f.y; s[4 * c + 2] = f.z; s[4 * c + 3] = f.w;
    q[4 * c] = f.x * f.x; q[4 * c + 1] = f.y * f.y; q[4 * c + 2] = f.z * f.z; q[4 * c + 3] = f.w * f.w;
  }
  const float depth = p.depth_vals[d];
  for (int k = 0; k < p.nn; ++k) {
    const float* T = p.transforms + 12 * k;
    const float gx = float(x) * depth, gy = float(y) * depth, gz = depth;
    const float X = T[0] * gx + T[1] * gy + T[2] * gz + T[3];
    const float Y = T[4] * gx + T[5] * gy + T[6] * gz + T[7];
    float Z = T[8] * gx + T[9] * gy + T[10] * gz + T[11];
    if (Z < 1e-4f) Z = 1e-4f;                                     // modules.py:56-57
    // scale to -1..1 with (W-1)/2 and sample with align_corners=True (modules.py:59-66): pixel coordinates again
    const float gxn = (X / Z) / ((p.w - 1) / 2.f) - 1.f, gyn = (Y / Z) / ((p.h - 1) / 2.f) - 1.f;
    const float fx = (gxn + 1.f) / 2.f * float(p.w - 1), fy = (gyn + 1.f) / 2.f * float(p.h - 1);
    const float x0f = floorf(fx), y0f = floorf(fy);
    const float tx = fx - x0f, ty = fy - y0f;
    const float wgt[4] = {(1.f - tx) * (1.f - ty), tx * (1.f - ty), (1.f - tx) * ty, tx * ty};
    const float* sf = p.src_feats + (long long)p.nn_ids[k] * p.h * p.w * 32;
    float wv[32];
    for (int c = 0; c < 32; ++c) wv[c] = 0.f;
    // out-of-range / non-finite coordinates contribute zero taps (padding_mode='zeros'); the float comparisons reject NaN
    for (int q4 = 0; q4 < 4; ++q4) {
      const float xf = x0f + float(q4 & 1), yf = y0f + float(q4 >> 1);
      if (!(xf >= 0.f && xf <= float(p.w - 1) && yf >= 0.f && yf <= float(p.h - 1))) continue;
      const float4* __restrict__ tap = reinterpret_cast<const float4*>(sf + ((long long)int(yf) * p.w + int(xf)) * 32);
      const float g = wgt[q4];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float4 f = tap[c];
        wv[4 * c] = fmaf(f.x, g, wv[4 * c]); wv[4 * c + 1] = fmaf(f.y, g, wv[4 * c + 1]);
        wv[4 * c + 2] = fmaf(f.z, g, wv[4 * c + 2]); wv[4 * c + 3] = fmaf(f.w, g, wv[4 * c + 3]);
      }
    }
    for (int c = 0; c < 32; ++c) { s[c] += wv[c]; q[c] += wv[c] * wv[c]; }
  }
  const float inv = 1.f / float(p.nn + 1);
  float4* out = reinterpret_cast<float4*>(p.vol + v * 32);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float r[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float m = s[4 * c + e] * inv; r[e] = q[4 * c + e] * inv - m * m; }
    out[c] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// ---- softmax over the depth planes + depth regression (init_net.py:155-159), with the optional bilinear resize of the logits
//      (F.interpolate(cost_reg, (h//4, w//4), mode='bilinear'), align_corners=False) and nan -> 0 (init_net.py:154) -------------
struct SoftmaxP {
  const float* logits;         // [hr,wr,dn] of this view
  const float* depth_vals;     // [dn]
  float* prob;                 // [ho,wo,dn]
  float* depth;                // [ho,wo]
  int hr, wr, ho, wo, dn;
};
NR_HD void resize_taps(int o, int n_in, int n_out, int& i0, int& i1, float& l0, float& l1) {   // align_corners=False
  const float scale = float(n_in) / float(n_out);
  float src = (float(o) + 0.5f) * scale - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = int(src);
  if (i0 > n_in - 1) i0 = n_in - 1;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = src - float(i0);
  l0 = 1.f - l1;
}
NR_HD float nan0(float v) { return v == v ? v : 0.f; }
NR_HD void softmax_pixel(const SoftmaxP& p, int pix, float* tmp /*[dn]*/) {
  const int xo = pix % p.wo, yo = pix / p.wo;
  if (p.hr == p.ho && p.wr == p.wo) {
    const float* l = p.logits + (long long)pix * p.dn;
    for (int d = 0; d < p.dn; ++d) tmp[d] = nan0(l[d]);
  } else {
    int y0, y1, x0, x1;
    float ly0, ly1, lx0, lx1;
    resize_taps(yo, p.hr, p.ho, y0, y1, ly0, ly1);
    resize_taps(xo, p.wr, p.wo, x0, x1, lx0, lx1);
    const float* a = p.logits + ((long long)y0 * p.wr + x0) * p.dn; const float* b = p.logits + ((long long)y0 * p.wr + x1) * p.dn;
    const float* c = p.logits + ((long long)y1 * p.wr + x0) * p.dn; const float* e = p.logits + ((long long)y1 * p.wr + x1) * p.dn;
    for (int d = 0; d < p.dn; ++d) tmp[d] = ly0 * (lx0 * nan0(a[d]) + lx1 * nan0(b[d])) + ly1 * (lx0 * nan0(c[d]) + lx1 * nan0(e[d]));
  }
  float m = tmp[0];
  for (int d = 1; d < p.dn; ++d) m = fmaxf(m, tmp[d]);
  float sum = 0.f;
  for (int d = 0; d < p.dn; ++d) { tmp[d] = expf(tmp[d] - m); sum += tmp[d]; }
  float depth = 0.f;
  float* pr = p.prob + (long long)pix * p.dn;
  for (int d = 0; d < p.dn; ++d) { const float v = tmp[d] / sum; pr[d] = v; depth += v * p.depth_vals[d]; }
  p.depth[pix] = depth;
}

// get_depth_vals (init_net.py:162-168): uniform in inverse depth, the last plane exactly far
NR_HD float depth_val(float near, float far, int j, int dn) {
  if (j == dn - 1) return far;
  const float interval = (1.f / far - 1.f / near) / float(dn - 1);
  return 1.f / (1.f / near + float(j) * interval);
}

// bilinear resize (align_corners=False) of NCHW images into channel-last [N,ho,wo,3] (identity when the sizes agree)
struct ResizeP { const float* img; float* out; int N, H, W, Ho, Wo; };
NR_HD void resize_pixel(const ResizeP& p, long long i) {
  const int xo = int(i % p.Wo);
  const long long t = i / p.Wo;
  const int yo = int(t % p.Ho), n = int(t / p.Ho);
  int y0 = yo, y1 = yo, x0 = xo, x1 = xo;
  float ly0 = 1.f, ly1 = 0.f, lx0 = 1.f, lx1 = 0.f;
  if (p.H != p.Ho || p.W != p.Wo) { resize_taps(yo, p.H, p.Ho, y0, y1, ly0, ly1); resize_taps(xo, p.W, p.Wo, x0, x1, lx0, lx1); }
  for (int c = 0; c < 3; ++c) {
    const float* im = p.img + ((long long)n * 3 + c) * p.H * p.W;
    p.out[i * 3 + c] = ly0 * (lx0 * im[(long long)y0 * p.W + x0] + lx1 * im[(long long)y0 * p.W + x1]) +
                       ly1 * (lx0 * im[(long long)y1 * p.W + x0] + lx1 * im[(long long)y1 * p.W + x1]);
  }
}

// transform of one (reference view, neighbour): rows of R | T of P_src @ inv(P_ref), P = [diag(sx, sy, 1) K pose; 0 0 0 1]
// (init_net.py:103-111 construct_project_matrix, mvsnet.py:120 torch.inverse, modules.py:37-39), in fp64
NR_HD void project_matrix(const float* K, const float* pose, double sx, double sy, double (&P)[16]) {
  const double s[3] = {sx, sy, 1.0};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double a = 0.0;
      for (int k = 0; k < 3; ++k) a += double(K[3 * r + k]) * double(pose[4 * k + c]);
      P[4 * r + c] = s[r] * a;
    }
  P[12] = P[13] = P[14] = 0.0; P[15] = 1.0;
}
NR_HD void affine_inverse(const double (&P)[16], double (&Q)[16]) {     // last row 0 0 0 1
  const double a = P[0], b = P[1], c = P[2], d = P[4], e = P[5], f = P[6], g = P[8], h = P[9], i = P[10];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double r[9] = {(e * i - f * h) / det, (c * h - b * i) / det, (b * f - c * e) / det, (f * g - d * i) / det, (a * i - c * g) / det,
                       (c * d - a * f) / det, (d * h - e * g) / det, (b * g - a * h) / det, (a * e - b * d) / det};
  for (int y = 0; y < 3; ++y) {
    for (int x = 0; x < 3; ++x) Q[4 * y + x] = r[3 * y + x];
    Q[4 * y + 3] = -(r[3 * y] * P[3] + r[3 * y + 1] * P[7] + r[3 * y + 2] * P[11]);
  }
  Q[12] = Q[13] = Q[14] = 0.0; Q[15] = 1.0;
}
NR_HD void pair_transform(const float* Kr, const float* pr, const float* Ks, const float* ps, float ratio, float* out12) {
  double Pr[16], Ps[16], Qi[16];
  project_matrix(Kr, pr, ratio, ratio, Pr);
  project_matrix(Ks, ps, ratio, ratio, Ps);
  affine_inverse(Pr, Qi);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double a = 0.0;
      for (int k = 0; k < 4; ++k) a += Ps[4 * r + k] * Qi[4 * k + c];
      out12[4 * r + c] = float(a);
    }
}

}  // namespace mvs
}  // namespace nr

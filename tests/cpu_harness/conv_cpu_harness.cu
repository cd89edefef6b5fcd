// Test infrastructure: runs the encoder layer graphs of csrc/nr_encoder_graph.cuh on the HOST.  Every building block is
// executed through the same __host__ __device__ routines the CUDA kernels call (csrc/nr_conv.cuh); the tensor-core conv is
// emulated CTA by CTA: the staging loops fill a shared-memory image through a_chunk / b_chunk, every lane gathers its
// fragments through a_frag / b_frag, the m16n8k8 product is formed from the 32 lanes' fragments following the PTX fragment
// layout, and epilogue_thread writes the result.  tests/test_encoders_cpu.py checks this against the reference's torch
// modules without a GPU.  Not part of the product library.
#include <string.h>

#include <vector>

#include "../../neuray_b200/csrc/nr_encoder_graph.cuh"

namespace nr {
void set_error(const char*, ...) {}
}  // namespace nr

using namespace nr;
using namespace nr::cv;

template <int BM, int BN, int KC>
static void host_conv(const ConvP& p) {
  constexpr int MT = mt_of(BM, BN), WN = BN / 32;
  constexpr int A_ST = BM * (KC + 4), B_ST = KC * (BN + 8);
  constexpr int A_ROWS = THREADS / (KC / 4), A_PASSES = BM / A_ROWS;
  const long long M = (long long)p.N * p.Ho * p.Wo;
  const int nk = p.ks * p.ks * (p.Cin / KC);
  std::vector<float> A(A_ST), B(B_ST);
  std::vector<float> acc(size_t(THREADS) * MT * 4 * 4);
  for (long long m0 = 0; m0 < M; m0 += BM) {
    std::fill(acc.begin(), acc.end(), 0.f);
    for (int kt = 0; kt < nk; ++kt) {
      std::fill(A.begin(), A.end(), -777.f);      // poison: a chunk the staging loops miss shows up in the result
      std::fill(B.begin(), B.end(), -777.f);
      for (int tid = 0; tid < THREADS; ++tid) {
        const int a_row = tid / (KC / 4), a_c4 = (tid - a_row * (KC / 4)) * 4;
        for (int j = 0; j < A_PASSES; ++j) {
          const RowInfo ri = row_info(p, m0 + a_row + j * A_ROWS);
          int dst;
          const float* src;
          a_chunk<KC>(p, ri, a_row + j * A_ROWS, a_c4, kt, dst, src);
          for (int e = 0; e < 4; ++e) A[dst + e] = src != nullptr ? src[e] : 0.f;
        }
        for (int idx = tid; idx < KC * BN / 4; idx += THREADS) {
          int dst;
          const float* src;
          b_chunk<BN, KC>(p, idx, kt, dst, src);
          for (int e = 0; e < 4; ++e) B[dst + e] = src[e];
        }
      }
      for (int warp = 0; warp < 8; ++warp) {
        const int warp_m = warp / WN, warp_n = warp - warp_m * WN;
        for (int k8 = 0; k8 < KC / 8; ++k8)
          for (int i = 0; i < MT; ++i)
            for (int j = 0; j < 4; ++j) {
              float At[16][8], Bt[8][8];
              for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t4 = lane & 3;
                int ao[4], bo[2];
                a_frag<KC>(warp_m * (16 * MT) + 16 * i, lane, k8, ao);
                b_frag<BN>(warp_n * 32 + 8 * j, lane, k8, bo);
                At[g][t4] = A[ao[0]]; At[g + 8][t4] = A[ao[1]]; At[g][t4 + 4] = A[ao[2]]; At[g + 8][t4 + 4] = A[ao[3]];
                Bt[t4][g] = B[bo[0]]; Bt[t4 + 4][g] = B[bo[1]];
              }
              for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t4 = lane & 3;
                float* c = &acc[((size_t(warp) * 32 + lane) * MT + i) * 16 + j * 4];
                for (int e = 0; e < 4; ++e) {
                  const int r = g + (e >> 1) * 8, col = 2 * t4 + (e & 1);
                  float sum = 0.f;
                  for (int k = 0; k < 8; ++k) sum += At[r][k] * Bt[k][col];
                  c[e] += sum;
                }
              }
            }
      }
    }
    for (int tid = 0; tid < THREADS; ++tid) {
      const int warp = tid >> 5, lane = tid & 31;
      const int warp_m = warp / WN, warp_n = warp - warp_m * WN;
      float a[MT][4][4];
      memcpy(a, &acc[size_t(tid) * MT * 16], sizeof(a));
      const bool uniform = warp_rows_uniform<BM, BN>(p, m0, warp);
      float s[4][2], q[4][2];
      epilogue_thread<BM, BN>(p, m0, warp, lane, a, uniform, s, q);
      if (p.stats != nullptr && uniform) {
        const long long first = m0 + warp_m * (16 * MT);
        if (first < M) {
          const int n = int(first / ((long long)p.Ho * p.Wo));
          for (int j = 0; j < 4; ++j)
            for (int b = 0; b < 2; ++b) {
              const int col = warp_n * 32 + 8 * j + 2 * (lane & 3) + b;
              double* st = p.stats + ((long long)n * BN + col) * 2;
              st[0] += double(s[j][b]);
              st[1] += double(q[j][b]);
            }
        }
      }
    }
  }
}

struct HostOps {
  template <int BM, int BN>
  static void conv_k(const ConvP& p) { p.Cin % 32 == 0 ? host_conv<BM, BN, 32>(p) : host_conv<BM, BN, 16>(p); }
  void conv(const ConvP& p) {       // the launcher's dispatch (csrc/nr_encoder.cu launch_conv), 132 SMs (H100) assumed for the automatic choice
    const int bm = p.bm != 0 ? p.bm : pick_bm(p.Cout, (long long)p.N * p.Ho * p.Wo, 132);
    switch (p.Cout) {
      case 32: bm == 256 ? conv_k<256, 32>(p) : conv_k<128, 32>(p); break;
      case 64: bm == 64 ? conv_k<64, 64>(p) : conv_k<128, 64>(p); break;
      default: bm == 64 ? conv_k<64, 128>(p) : conv_k<128, 128>(p); break;
    }
  }
  template <int COUT>
  static void conv7_t(const Conv7P& p) {
    for (int n = 0; n < p.N; ++n)
      for (int pix = 0; pix < p.Ho * p.Wo; ++pix) {
        float out[COUT];
        conv7_pixel<COUT>(p, p.w, n, pix, out);
        for (int c = 0; c < COUT; ++c) {
          p.y[((long long)n * p.Ho * p.Wo + pix) * COUT + c] = out[c];
          p.stats[((long long)n * COUT + c) * 2] += out[c];
          p.stats[((long long)n * COUT + c) * 2 + 1] += double(out[c]) * out[c];
        }
      }
  }
  void conv7(const Conv7P& p) { p.Cout == 16 ? conv7_t<16>(p) : conv7_t<32>(p); }
  void norm(const NormP& p) {
    for (int n = 0; n < p.N; ++n)
      for (int c = 0; c < p.C; ++c) {
        float sc = 1.f, sh = 0.f, rsc = 1.f, rsh = 0.f;
        if (p.stats != nullptr) norm_coeffs(p.stats, p.gamma, p.beta, n, c, p.C, p.HW, p.eps, sc, sh);
        if (p.res != nullptr && p.res_stats != nullptr) norm_coeffs(p.res_stats, p.res_gamma, p.res_beta, n, c, p.C, p.HW, p.eps, rsc, rsh);
        for (long long pix = 0; pix < p.HW; ++pix) {
          const long long m = (long long)n * p.HW + pix;
          float o = p.x[m * p.x_stride + p.x_off + c] * sc + sh;
          if (p.res != nullptr) o += p.res[m * p.res_stride + p.res_off + c] * rsc + rsh;
          p.y[m * p.y_stride + p.y_off + c] = act_f(o, p.act);
        }
      }
  }
  void upsample(const UpP& p) {
    for (int n = 0; n < p.N; ++n)
      for (int yo = 0; yo < p.Ho; ++yo)
        for (int xo = 0; xo < p.Wo; ++xo) {
          int y0, y1, x0, x1;
          float ly0, ly1, lx0, lx1;
          up_taps(yo, p.H, p.Ho, y0, y1, ly0, ly1);
          up_taps(xo, p.W, p.Wo, x0, x1, lx0, lx1);
          const float* base = p.x + (long long)n * p.H * p.W * p.x_stride + p.x_off;
          for (int c = 0; c < p.C; ++c) {
            const float a = base[((long long)y0 * p.W + x0) * p.x_stride + c], b = base[((long long)y0 * p.W + x1) * p.x_stride + c];
            const float cc = base[((long long)y1 * p.W + x0) * p.x_stride + c], d = base[((long long)y1 * p.W + x1) * p.x_stride + c];
            p.y[(((long long)n * p.Ho + yo) * p.Wo + xo) * p.y_stride + p.y_off + c] = ly0 * (lx0 * a + lx1 * b) + ly1 * (lx0 * cc + lx1 * d);
          }
        }
  }
  void copy_pad(const enc::CopyP& p) {
    for (int n = 0; n < p.N; ++n)
      for (int yo = 0; yo < p.Ho; ++yo)
        for (int xo = 0; xo < p.Wo; ++xo) {
          const int yi = yo - p.py, xi = xo - p.px;
          const bool in = yi >= 0 && yi < p.H && xi >= 0 && xi < p.W;
          for (int c = 0; c < p.C; ++c)
            p.y[(((long long)n * p.Ho + yo) * p.Wo + xo) * p.y_stride + p.y_off + c] =
                in ? p.x[(((long long)n * p.H + yi) * p.W + xi) * p.x_stride + p.x_off + c] : 0.f;
        }
  }
  void depth_skip(const DepthSkipP& p) {
    for (int n = 0; n < p.N; ++n)
      for (int yo = 0; yo < p.Ho; ++yo)
        for (int xo = 0; xo < p.Wo; ++xo) {
          float out[16];
          depth_skip_pixel(p, n, yo, xo, out);
          for (int c = 0; c < 16; ++c) p.y[(((long long)n * p.Ho + yo) * p.Wo + xo) * p.y_stride + p.y_off + c] = out[c];
        }
  }
  void zero(void* ptr, size_t bytes) { memset(ptr, 0, bytes); }
};

static void host_pack(const enc::NetSpec& spec, const float* const* params, float* packed) {
  memset(packed, 0, size_t(spec.total) * sizeof(float));
  for (int i = 0; i < spec.count; ++i)
    for (long long e = 0; e < spec.t[i].n; ++e) {
      const long long src = enc::pack_source(spec.t[i], e);
      packed[spec.t[i].off + e] = src >= 0 ? params[i][src] : 0.f;
    }
}

extern "C" int nr_cpu_encoder_counts(int* image_tensors, int* vis_tensors) {
  enc::ImageNet in;
  enc::VisNet vn;
  enc::build_image_net(in);
  enc::build_vis_net(vn);
  *image_tensors = in.spec.count;
  *vis_tensors = vn.spec.count;
  return 0;
}
extern "C" int nr_cpu_image_dims(int h, int w, int* fh, int* fw) {
  const enc::ImageDims d = enc::image_dims(h, w);
  *fh = d.u2h; *fw = d.u2w;
  return 0;
}

// imgs [n,3,h,w] -> out [n,fh,fw,out_stride] channels [out_off, out_off + 32)
extern "C" int nr_cpu_image_encoder(const float* const* params, int n_params, const float* imgs, int n, int h, int w, float* out, int out_stride,
                                    int out_off) {
  enc::ImageNet* net = new enc::ImageNet;
  enc::build_image_net(*net);
  if (n_params != net->spec.count) return -1;
  std::vector<float> packed(net->spec.total);
  host_pack(net->spec, params, packed.data());
  const size_t bytes = enc::image_workspace_bytes(*net, n, h, w);
  std::vector<char> ws(bytes + 256);
  char* base = (char*)((uintptr_t(ws.data()) + 255) & ~uintptr_t(255));
  enc::Arena ar{base, bytes, 0, true};
  HostOps ops;
  const long long stats = enc::image_stats_doubles(*net, n, h, w);
  const bool ok = stats > 0 && enc::image_encoder_graph(ops, ar, *net, packed.data(), imgs, n, h, w, out, out_stride, out_off, stats, nullptr);
  delete net;
  return ok ? 0 : -2;
}

extern "C" int nr_cpu_vis_encoder(const float* const* params, int n_params, float* feat, int n, int fh, int fw) {
  enc::VisNet* net = new enc::VisNet;
  enc::build_vis_net(*net);
  if (n_params != net->spec.count) return -1;
  std::vector<float> packed(net->spec.total);
  host_pack(net->spec, params, packed.data());
  const size_t bytes = enc::vis_workspace_bytes(*net, n, fh, fw);
  std::vector<char> ws(bytes + 256);
  char* base = (char*)((uintptr_t(ws.data()) + 255) & ~uintptr_t(255));
  enc::Arena ar{base, bytes, 0, true};
  HostOps ops;
  const bool ok = enc::vis_encoder_graph(ops, ar, *net, packed.data(), feat, n, fh, fw, enc::vis_stats_doubles(*net, n, fh, fw), nullptr);
  delete net;
  return ok ? 0 : -2;
}

// DepthInitNet after extract_depth / get_diff_feats: imgs [n,3,h,w], depth_norm [n,1,h,w], diff_feats [n,8,h,w] (NCHW) -> out slot
extern "C" int nr_cpu_depth_init(const float* const* params, int n_params, const float* imgs, const float* depth_norm, const float* diff_feats, int n,
                                 int h, int w, float* out, int out_stride, int out_off) {
  enc::DepthInitNet* net = new enc::DepthInitNet;
  enc::build_depth_init_net(*net);
  if (n_params != net->res.spec.count) return -1;
  std::vector<float> packed(net->res.spec.total);
  host_pack(net->res.spec, params, packed.data());
  const long long hw = (long long)h * w;
  std::vector<float> x16(size_t(n) * hw * 16, 0.f);
  for (int i = 0; i < n; ++i)
    for (long long p = 0; p < hw; ++p) {
      float* px = &x16[(size_t(i) * hw + p) * 16];
      for (int c = 0; c < 3; ++c) px[c] = imgs[(size_t(i) * 3 + c) * hw + p];
      px[3] = depth_norm[size_t(i) * hw + p];
      for (int c = 0; c < 8; ++c) px[4 + c] = diff_feats[(size_t(i) * 8 + c) * hw + p];
    }
  const long long stats = enc::depth_init_stats_doubles(*net, n, h, w);
  const size_t bytes = enc::depth_init_workspace_bytes(*net, n, h, w);
  std::vector<char> ws(bytes + 256);
  char* base = (char*)((uintptr_t(ws.data()) + 255) & ~uintptr_t(255));
  enc::Arena ar{base, bytes, 0, true};
  HostOps ops;
  const bool ok = stats > 0 && enc::depth_init_graph(ops, ar, *net, packed.data(), x16.data(), depth_norm, n, h, w, out, out_stride, out_off, stats, nullptr);
  delete net;
  return ok ? 0 : -2;
}
extern "C" int nr_cpu_depth_init_dims(int h, int w, int* fh, int* fw, int* tensors) {
  const enc::ImageDims d = enc::depth_init_dims(h, w);
  *fh = d.u2h; *fw = d.u2w;
  enc::DepthInitNet* net = new enc::DepthInitNet;
  enc::build_depth_init_net(*net);
  *tensors = net->res.spec.count;
  delete net;
  return 0;
}

// CostVolumeInitNet's head: imgs [n,3,h,w] NCHW, prob [n,fh,fw,sn] channel-last, depth_norm [n,fh,fw] -> out slot
extern "C" int nr_cpu_cost_volume_head(int sn, const float* const* params, int n_params, const float* imgs, const float* prob, const float* depth_norm,
                                       int n, int h, int w, float* out, int out_stride, int out_off) {
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, sn);
  if (n_params != net->res.spec.count) return -1;
  std::vector<float> packed(net->res.spec.total);
  host_pack(net->res.spec, params, packed.data());
  const enc::ImageDims d = enc::image_dims(h, w);
  const long long hw = (long long)d.u2h * d.u2w;
  std::vector<float> d16(size_t(n) * hw * 16, 0.f);
  for (long long i = 0; i < (long long)n * hw; ++i) d16[i * 16] = depth_norm[i];
  const long long stats = enc::cv_head_stats_doubles(*net, n, h, w, d.u2h, d.u2w);
  const size_t bytes = enc::cv_head_workspace_bytes(*net, n, h, w, d.u2h, d.u2w);
  std::vector<char> ws(bytes + 256);
  char* base = (char*)((uintptr_t(ws.data()) + 255) & ~uintptr_t(255));
  enc::Arena ar{base, bytes, 0, true};
  HostOps ops;
  const bool ok = stats > 0 && enc::cost_volume_head_graph(ops, ar, *net, packed.data(), imgs, prob, sn, d16.data(), n, h, w, d.u2h, d.u2w, out, out_stride,
                                                          out_off, stats, nullptr);
  const int count = net->res.spec.count;
  delete net;
  (void)count;
  return ok ? 0 : -2;
}
extern "C" int nr_cpu_cost_volume_head_tensors(int sn) {
  enc::CostVolumeHead* net = new enc::CostVolumeHead;
  enc::build_cost_volume_head(*net, sn);
  const int c = net->res.spec.count;
  delete net;
  return c;
}

// one convolution: w [cout][cin][ks][ks] (PyTorch layout, packed here), x / y / res channel-last
extern "C" int nr_cpu_conv2d(const float* x, const float* w, const float* bias, const float* res, float* y, double* stats, int n, int h, int wd,
                             int cin, int cout, int ks, int stride, int reflect, int cin_rot, int x_stride, int x_off, int y_stride, int y_off, int pad,
                             int cin_ref, int bm) {
  enc::NetSpec* spec = new enc::NetSpec;
  spec->count = 0; spec->total = 0;
  spec->conv(cout, cin, ks, cin_rot, 0, cin_ref);
  std::vector<float> packed(spec->total);
  const float* params[1] = {w};
  host_pack(*spec, params, packed.data());
  delete spec;
  ConvP p;
  p.x = x; p.w = packed.data(); p.bias = bias; p.res = res; p.y = y; p.stats = stats;
  p.N = n; p.H = h; p.W = wd; p.Cin = cin; p.Cout = cout; p.ks = ks; p.stride = stride; p.reflect = reflect;
  p.pad = pad >= 0 ? pad : (ks - 1) / 2;
  p.Ho = enc::conv_out(h, ks, stride, p.pad); p.Wo = enc::conv_out(wd, ks, stride, p.pad);
  p.x_stride = x_stride; p.x_off = x_off; p.y_stride = y_stride; p.y_off = y_off; p.res_stride = cout; p.res_off = 0;
  p.tf32x1 = 0; p.bm = bm;
  HostOps ops;
  ops.conv(p);
  return 0;
}

// Stand-alone kernels behind the render_ops drop-in functions (reference network/render_ops.py) and the
// per-frame NCHW -> channel-last repack.  These are the cold, un-fused entry points: the renderer itself goes
// through the fused point/ray kernels; these exist so that every public function of network/render_ops.py has a
// CUDA implementation with the reference's semantics (e.g. network/init_net.py:10 imports project_points_ref_views).
#include <stdarg.h>

#include "nr_common.cuh"
#include "nr_resample.cuh"

namespace nr {
namespace ops {

constexpr int TPB = 256;
inline int blocks_for(long long n) { return int((n + TPB - 1) / TPB); }

// ---- per-frame repack --------------------------------------------------------------------------------------
__global__ void pack_feat_kernel(const float* __restrict__ rf, const float* __restrict__ imf, int rfn, int fh, int fw,
                                 float* __restrict__ out) {
  // one thread per (view, texel, 4-channel group): reads 4 strided channels, writes one float4
  const long long total = (long long)rfn * fh * fw * 16;
  const long long hw = (long long)fh * fw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = int(i & 15);
    const long long t = i >> 4;            // view*hw + texel
    const long long v = t / hw, px = t - v * hw;
    const float* __restrict__ src = (g < 8 ? rf : imf) + (v * 32 + (g & 7) * 4) * hw + px;
    float4 o;
    o.x = __ldg(src); o.y = __ldg(src + hw); o.z = __ldg(src + 2 * hw); o.w = __ldg(src + 3 * hw);
    reinterpret_cast<float4*>(out)[i] = o;
  }
}

__global__ void pack_rgb_kernel(const float* __restrict__ imgs, int rfn, int h, int w, float* __restrict__ out) {
  const long long hw = (long long)h * w, total = (long long)rfn * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / hw, px = i - v * hw;
    const float* __restrict__ src = imgs + v * 3 * hw + px;
    reinterpret_cast<float4*>(out)[i] = make_float4(__ldg(src), __ldg(src + hw), __ldg(src + 2 * hw), 0.f);
  }
}

// ---- sampling / ray geometry -------------------------------------------------------------------------------
__global__ void sample_depth_kernel(const float* __restrict__ range, int rn, int dn, const float* __restrict__ jitter,
                                    float* __restrict__ depth, float* __restrict__ dists) {
  const long long total = (long long)rn * dn;
  const float near = __ldg(range), far = __ldg(range + 1);
  const float span = 1.f / far - 1.f / near;
  const float step = span / float(dn - 1);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int s = int(i % dn);
    const long long ray = i / dn;
    auto tick = [&](int k) -> float {
      if (k == 0) return 0.f;
      if (k == dn - 1) return span;
      float val = float(k);
      if (jitter) val = val + (jitter[ray * (dn - 2) + (k - 1)] - 0.5f) * 0.999f;
      return step * val;
    };
    const float d = 1.f / (1.f / near + tick(s));
    depth[i] = d;
    if (dists) dists[i] = (s + 1 < dn ? 1.f / (1.f / near + tick(s + 1)) : 1e6f) - d;
  }
}

__device__ __forceinline__ void ray_of(const float* __restrict__ cam, float cx, float cy, float* d) {
  float cm[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) cm[i] = fmaf(cam[12 + 3 * i + 1], cy, cam[12 + 3 * i] * cx) + cam[12 + 3 * i + 2];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float wld = fmaf(cam[3 * i + 2], cm[2], fmaf(cam[3 * i + 1], cm[1], cam[3 * i] * cm[0])) + cam[9 + i];
    d[i] = wld - cam[9 + i];
  }
}

__global__ void coords2rays_kernel(const float* __restrict__ coords, const float* __restrict__ cam, int rn,
                                   float* __restrict__ centers, float* __restrict__ dirs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rn) return;
  float d[3];
  ray_of(cam, coords[2 * i], coords[2 * i + 1], d);
#pragma unroll
  for (int k = 0; k < 3; ++k) { centers[3 * i + k] = cam[9 + k]; dirs[3 * i + k] = d[k]; }
}

__global__ void depth2points_kernel(const float* __restrict__ coords, const float* __restrict__ cam,
                                    const float* __restrict__ depth, int rn, int dn, float* __restrict__ pts,
                                    float* __restrict__ dirs) {
  const long long total = (long long)rn * dn;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long ray = i / dn;
    float d[3];
    ray_of(cam, coords[2 * ray], coords[2 * ray + 1], d);
    const float z = depth[i];
    const float nrm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k) { pts[3 * i + k] = fmaf(d[k], z, cam[9 + k]); dirs[3 * i + k] = -d[k] / nrm; }
  }
}

__global__ void depth2dists_kernel(const float* __restrict__ depth, long long rows, int dn, const float* __restrict__ range,
                                   float* __restrict__ dists) {
  const long long total = rows * dn;
  const bool inv = range != nullptr;
  const float a = inv ? -1.f / __ldg(range) : 0.f, b = inv ? -1.f / __ldg(range + 1) : 1.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int s = int(i % dn);
    auto val = [&](long long j) -> float { return inv ? (-1.f / depth[j] - a) / (b - a) : depth[j]; };
    dists[i] = s + 1 < dn ? val(i + 1) - val(i) : 1e6f;
  }
}

__global__ void alpha2hit_kernel(const float* __restrict__ alpha, long long rows, int dn, float* __restrict__ hit) {
  // one thread per row: the product is sequential exactly like torch.cumprod on one row
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float T = 1.f;
  for (int s = 0; s < dn; ++s) {
    const float a = alpha[r * dn + s];
    hit[r * dn + s] = a * T;
    T *= (1.f - a + 1e-10f);
  }
}

// ---- projection --------------------------------------------------------------------------------------------
__global__ void project_kernel(const float* __restrict__ pts, long long pn, const float* __restrict__ vps, int rfn, int h,
                               int w, float* __restrict__ dir, float* __restrict__ pix, float* __restrict__ depth,
                               float* __restrict__ mask, float* __restrict__ valid_z) {
  const long long total = pn * rfn;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long v = i / pn, n = i - v * pn;
    const Proj pj = project(vps + v * 20, pts[3 * n], pts[3 * n + 1], pts[3 * n + 2], h, w);
    if (pix) { pix[2 * i] = pj.ux; pix[2 * i + 1] = pj.uy; }
    if (depth) depth[i] = pj.zh;
    if (mask) mask[i] = pj.valid ? 1.f : 0.f;
    if (valid_z) valid_z[i] = pj.valid_z ? 1.f : 0.f;
    if (dir) { dir[3 * i] = pj.dir[0]; dir[3 * i + 1] = pj.dir[1]; dir[3 * i + 2] = pj.dir[2]; }
  }
}

// ---- bilinear sampling on an NCHW map (F.grid_sample semantics through ops.py:14-34) --------------------------
// Taps at pixel (x, y) of an h x w image on an fh x fw map: the texel columns xa, xb and rows ya, yb, clamped into the map,
// and the weights of (ya,xa), (ya,xb), (yb,xa), (yb,xb) times `scale`.  A texel outside the map (zeros padding) or a
// non-finite coordinate contributes nothing: its weight is 0.
struct InterpTaps {
  int xa, xb, ya, yb;
  float w00, w01, w10, w11;
};
__device__ __forceinline__ InterpTaps interp_taps(float x, float y, float h, float w, int fh, int fw, int border, int align,
                                                  float scale) {
  const float gx = x / (w - 1.f) * 2.f - 1.f, gy = y / (h - 1.f) * 2.f - 1.f;
  float ix = align ? (gx + 1.f) / 2.f * float(fw - 1) : ((gx + 1.f) * float(fw) - 1.f) / 2.f;
  float iy = align ? (gy + 1.f) / 2.f * float(fh - 1) : ((gy + 1.f) * float(fh) - 1.f) / 2.f;
  if (border) {
    ix = fminf(fmaxf(ix, 0.f), float(fw - 1));
    iy = fminf(fmaxf(iy, 0.f), float(fh - 1));
  }
  const float x0f = floorf(ix), y0f = floorf(iy);
  const float we = ix - x0f, ww = (x0f + 1.f) - ix, ws = iy - y0f, wn = (y0f + 1.f) - iy;
  const bool finite = fabsf(x0f) < 1e9f && fabsf(y0f) < 1e9f;
  const int x0 = finite ? int(x0f) : -10, y0 = finite ? int(y0f) : -10;
  const bool vx0 = x0 >= 0 && x0 < fw, vx1 = x0 + 1 >= 0 && x0 + 1 < fw;
  const bool vy0 = y0 >= 0 && y0 < fh, vy1 = y0 + 1 >= 0 && y0 + 1 < fh;
  InterpTaps t;
  t.w00 = (vx0 && vy0) ? ww * wn * scale : 0.f; t.w01 = (vx1 && vy0) ? we * wn * scale : 0.f;
  t.w10 = (vx0 && vy1) ? ww * ws * scale : 0.f; t.w11 = (vx1 && vy1) ? we * ws * scale : 0.f;
  t.xa = min(max(x0, 0), fw - 1); t.xb = min(max(x0 + 1, 0), fw - 1);
  t.ya = min(max(y0, 0), fh - 1); t.yb = min(max(y0 + 1, 0), fh - 1);
  return t;
}

__global__ void interp_kernel(const float* __restrict__ feats, const float* __restrict__ pts, const float* __restrict__ mask,
                              int b, int c, int fh, int fw, long long n, float h, float w, int border, int align,
                              float* __restrict__ out) {
  const long long total = (long long)b * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long bi = i / n;
    const InterpTaps t = interp_taps(pts[2 * i], pts[2 * i + 1], h, w, fh, fw, border, align, 1.f);
    const float m = mask ? mask[i] : 1.f;
    const float* __restrict__ base = feats + bi * c * fh * fw;
    for (int ch = 0; ch < c; ++ch) {
      const float* __restrict__ pl = base + (long long)ch * fh * fw;
      const float val = pl[t.ya * fw + t.xa] * t.w00 + pl[t.ya * fw + t.xb] * t.w01 + pl[t.yb * fw + t.xa] * t.w10 +
                        pl[t.yb * fw + t.xb] * t.w11;
      out[i * c + ch] = val * m;
    }
  }
}

// gradient of interp_kernel with respect to the map (the points carry no gradient on any path of the reference that
// reaches this function: coordinates come from projections of detached geometry): d_feats[b,c,fh,fw] += taps * d_out
__global__ void interp_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ pts, const float* __restrict__ mask,
                                  int b, int c, int fh, int fw, long long n, float h, float w, int border, int align,
                                  float* __restrict__ d_feats) {
  const long long total = (long long)b * n;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long bi = i / n;
    const InterpTaps t = interp_taps(pts[2 * i], pts[2 * i + 1], h, w, fh, fw, border, align, mask ? mask[i] : 1.f);
    float* __restrict__ base = d_feats + bi * c * fh * fw;
    for (int ch = 0; ch < c; ++ch) {
      float* __restrict__ pl = base + (long long)ch * fh * fw;
      const float g = d_out[i * c + ch];
      if (t.w00 != 0.f) atomicAdd(pl + t.ya * fw + t.xa, g * t.w00);
      if (t.w01 != 0.f) atomicAdd(pl + t.ya * fw + t.xb, g * t.w01);
      if (t.w10 != 0.f) atomicAdd(pl + t.yb * fw + t.xa, g * t.w10);
      if (t.w11 != 0.f) atomicAdd(pl + t.yb * fw + t.xb, g * t.w11);
    }
  }
}

// ---- stand-alone sample_fine_depth: one warp per ray ------------------------------------------------------------
__global__ void fine_depth_kernel(const float* __restrict__ depth, const float* __restrict__ hit, const float* __restrict__ range, int rn,
                                  int dn, int fdn, const float* __restrict__ u, int u_stride, int use_all, int do_sort, int sort_n,
                                  int per_warp, float* __restrict__ out) {
  extern __shared__ __align__(16) float fsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  float* sT = fsm + size_t(warp) * per_warp;
  float* sCdf = sT + dn;
  float* sSort = sCdf + dn + 4;
  const int M = fdn + (use_all ? dn : 0);
  const bool inv = range != nullptr;
  const float near = inv ? __ldg(range) : 1.f, far = inv ? __ldg(range + 1) : 2.f;
  for (int ray = blockIdx.x * warps + warp; ray < rn; ray += gridDim.x * warps) {
    resample_ray(hit + size_t(ray) * dn, depth + size_t(ray) * dn, dn, inv, near, far, u + size_t(ray) * u_stride, fdn, use_all,
                 do_sort, sort_n, sT, sCdf, sSort, out + size_t(ray) * M, lane);
    __syncwarp();
  }
}

}  // namespace ops

// implemented in nr_point_kernel.cu / nr_ray_kernel.cu / nr_blend.cu
int launch_point_kernel(const NrPassParams* p, float* dbg, long long* timing, float* row_blend, bool tf32, cudaStream_t stream);
int launch_ray_kernel(const NrPassParams* p, cudaStream_t stream);
int launch_blend_weights(const NrPassParams* p, const NrBlendParams* b, cudaStream_t stream);

// One render pass: the point kernel (3xTF32 or TF32 mode; row_blend: optional export of its colour-blend weights), then
// the ray kernel.  Every nr_render_pass_fwd* entry point is this sequence.
static int render_pass_fwd(const NrPassParams* p, float* row_blend, bool tf32, cudaStream_t stream) {
  const int rc = launch_point_kernel(p, nullptr, nullptr, row_blend, tf32, stream);
  if (rc != NR_OK) return rc;
  return launch_ray_kernel(p, stream);
}

// The pass with the blend-weight export on, then the reduction over its hit_prob.
static int render_pass_fwd_blend(const NrPassParams* p, const NrBlendParams* b, bool tf32, cudaStream_t stream) {
  NR_CHECK_ARG(p != nullptr && b != nullptr, "params");
  if (p->rn > 0) NR_CHECK_ARG(b->row_blend && b->blend_weights && p->hit_prob, "null blend workspace, blend_weights or hit_prob");
  const int rc = render_pass_fwd(p, b->row_blend, tf32, stream);
  if (rc != NR_OK) return rc;
  return launch_blend_weights(p, b, stream);
}

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// A failed query is not sticky: cudaGetLastError() clears it, so that the next launch check does not report it again.
int sm_count(int* sms, const char* who) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) return NR_OK;
  cudaGetLastError();
  set_error("%s: cannot query the SM count: %s", who, cudaGetErrorString(e));
  return NR_E_CUDA;
}

int opt_in_smem(const void* fn, size_t bytes, const char* who) {
  if (bytes <= 48 * 1024) return NR_OK;
  const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
  if (e == cudaSuccess) return NR_OK;
  cudaGetLastError();
  set_error("%s: cannot opt in to %zu bytes of dynamic shared memory: %s", who, bytes, cudaGetErrorString(e));
  return NR_E_CUDA;
}

}  // namespace nr

using namespace nr;
using namespace nr::ops;

extern "C" {

int nr_abi_version(void) { return NR_ABI_VERSION; }
const char* nr_last_error(void) { return g_err; }

int nr_weight_layout(NrWeightLayout* o) {
  NR_CHECK_ARG(o != nullptr, "out");
  o->total_point = lay::TOTAL_POINT; o->total_ray = lay::TOTAL_RAY;
  o->dd_head = lay::DD_HEAD; o->dd_head_stride = lay::DD_HEAD_STRIDE;
  o->dd_l0_w = lay::DD_L0_W; o->dd_l0_b = lay::DD_L0_B; o->dd_l1_w = lay::DD_L1_W; o->dd_l1_b = lay::DD_L1_B;
  o->dd_l2_w = lay::DD_L2_W; o->dd_l2_b = lay::DD_L2_B;
  o->grp_b = lay::GRP_B; o->pe0_w = lay::PE0_W; o->pe0_b = lay::PE0_B; o->pe1_w = lay::PE1_W; o->pe1_b = lay::PE1_B;
  o->rd0_w = lay::RD0_W; o->rd0_b = lay::RD0_B; o->rd1_w = lay::RD1_W; o->rd1_b = lay::RD1_B;
  o->nf0_w = lay::NF0_W; o->nf0_b = lay::NF0_B; o->nf1_w = lay::NF1_W; o->nf1_b = lay::NF1_B; o->grp_b_size = lay::GRP_B_SIZE;
  o->hoist_w = lay::HOIST_W; o->hoist_b = lay::HOIST_B; o->base0_w = lay::BASE0_W; o->base1_w = lay::BASE1_W; o->base1_b = lay::BASE1_B;
  o->grp_d1 = lay::GRP_D1; o->vis0_w = lay::VIS0_W; o->vis0_b = lay::VIS0_B; o->vis1_w = lay::VIS1_W; o->vis1_b = lay::VIS1_B;
  o->vis1l_w = lay::VIS1L_W; o->vis1l_b = lay::VIS1L_B; o->v20_w = lay::V20_W; o->v20_b = lay::V20_B; o->v21_w = lay::V21_W;
  o->v21_b = lay::V21_B; o->rgb0_w = lay::RGB0_W; o->rgb0_b = lay::RGB0_B; o->rgb1_w = lay::RGB1_W; o->rgb1_b = lay::RGB1_B;
  o->rgb2_w = lay::RGB2_W; o->rgb2_b = lay::RGB2_B; o->grp_d1_size = lay::GRP_D1_SIZE;
  o->grp_d2 = lay::GRP_D2; o->geo0_w = lay::GEO0_W; o->geo0_b = lay::GEO0_B; o->geo1_w = lay::GEO1_W; o->geo1_b = lay::GEO1_B;
  o->grp_d2_size = lay::GRP_D2_SIZE;
  o->wq = lay::WQ; o->wk = lay::WK; o->wv = lay::WV; o->wfc = lay::WFC; o->ln_w = lay::LN_W; o->ln_b = lay::LN_B;
  o->og0_w = lay::OG0_W; o->og0_b = lay::OG0_B; o->og1_w = lay::OG1_W; o->og1_b = lay::OG1_B;
  return NR_OK;
}

int nr_tc_layout(NrTcLayout* o) {
  NR_CHECK_ARG(o != nullptr, "out");
  o->total = tcl::TOTAL; o->stage = tcl::STAGE; o->head0 = tcl::HEAD0; o->pe0 = tcl::PE0; o->pe1 = tcl::PE1; o->b0 = tcl::B0;
  o->b1 = tcl::B1; o->v01 = tcl::V01; o->v2r = tcl::V2R; o->rd1 = tcl::RD1; o->hst = tcl::HST; o->g0 = tcl::G0;
  return NR_OK;
}

int nr_pack_feature_maps(const float* ray_feats, const float* img_feats, const float* imgs, int rfn, int h, int w, int fh,
                         int fw, float* out_feat, float* out_rgb, void* stream) {
  // ray_feats == img_feats == NULL: the frame pack was written in place by the native encoders (nr_image_encoder_fwd /
  // nr_vis_encoder_fwd), only the rgb pack is produced
  const bool maps = ray_feats != nullptr || img_feats != nullptr;
  NR_CHECK_ARG(imgs && out_rgb && (!maps || (ray_feats && img_feats && out_feat)), "null device pointer");
  NR_CHECK_ARG(rfn >= 1 && rfn <= NR_MAX_VIEWS && h > 1 && w > 1 && fh > 0 && fw > 0, "shape");
  cudaStream_t s = (cudaStream_t)stream;
  const long long nf = (long long)rfn * fh * fw * 16, nr_ = (long long)rfn * h * w;
  if (maps) pack_feat_kernel<<<min(blocks_for(nf), 132 * 16), TPB, 0, s>>>(ray_feats, img_feats, rfn, fh, fw, out_feat);
  pack_rgb_kernel<<<min(blocks_for(nr_), 132 * 16), TPB, 0, s>>>(imgs, rfn, h, w, out_rgb);
  NR_CHECK_LAUNCH("pack_feature_maps");
  return NR_OK;
}

int nr_point_kernel(const NrPassParams* p, void* stream) { return launch_point_kernel(p, nullptr, nullptr, nullptr, false, (cudaStream_t)stream); }
int nr_point_kernel_tf32(const NrPassParams* p, void* stream) { return launch_point_kernel(p, nullptr, nullptr, nullptr, true, (cudaStream_t)stream); }
int nr_point_kernel_debug(const NrPassParams* p, float* dbg, void* stream) {
  NR_CHECK_ARG(dbg != nullptr, "dbg");
  return launch_point_kernel(p, dbg, nullptr, nullptr, false, (cudaStream_t)stream);
}
int nr_point_kernel_timing(const NrPassParams* p, long long* timing, void* stream) {
  NR_CHECK_ARG(timing != nullptr && p != nullptr && p->w_tc != nullptr, "timing buffer / tensor-core weights required");
  return launch_point_kernel(p, nullptr, timing, nullptr, false, (cudaStream_t)stream);
}
int nr_ray_kernel(const NrPassParams* p, void* stream) { return launch_ray_kernel(p, (cudaStream_t)stream); }
int nr_render_pass_fwd(const NrPassParams* p, void* stream) { return render_pass_fwd(p, nullptr, false, (cudaStream_t)stream); }
int nr_render_pass_fwd_tf32(const NrPassParams* p, void* stream) { return render_pass_fwd(p, nullptr, true, (cudaStream_t)stream); }
int nr_render_pass_fwd_blend(const NrPassParams* p, const NrBlendParams* b, void* stream) {
  return render_pass_fwd_blend(p, b, false, (cudaStream_t)stream);
}
int nr_render_pass_fwd_tf32_blend(const NrPassParams* p, const NrBlendParams* b, void* stream) {
  return render_pass_fwd_blend(p, b, true, (cudaStream_t)stream);
}

int nr_sample_depth(const float* depth_range, int rn, int dn, const float* jitter, float* depth, float* dists, void* stream) {
  if (rn == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(dn > 2 && rn >= 0, "sample_depth arguments (dn must be > 2, render_ops.py:157)");
  NR_CHECK_ARG(depth != nullptr && depth_range != nullptr, "sample_depth: null pointer");
  sample_depth_kernel<<<blocks_for((long long)rn * dn), TPB, 0, (cudaStream_t)stream>>>(depth_range, rn, dn, jitter, depth, dists);
  NR_CHECK_LAUNCH("sample_depth");
  return NR_OK;
}

int nr_coords2rays(const float* coords, const float* cam, int rn, float* centers, float* directions, void* stream) {
  if (rn == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(coords && cam && centers && directions && rn >= 0, "coords2rays arguments");
  coords2rays_kernel<<<blocks_for(rn), TPB, 0, (cudaStream_t)stream>>>(coords, cam, rn, centers, directions);
  NR_CHECK_LAUNCH("coords2rays");
  return NR_OK;
}

int nr_depth2points(const float* coords, const float* cam, const float* depth, int rn, int dn, float* pts, float* dirs,
                    void* stream) {
  if (rn == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(coords && cam && depth && pts && dirs && rn >= 0 && dn > 0, "depth2points arguments");
  depth2points_kernel<<<blocks_for((long long)rn * dn), TPB, 0, (cudaStream_t)stream>>>(coords, cam, depth, rn, dn, pts, dirs);
  NR_CHECK_LAUNCH("depth2points");
  return NR_OK;
}

int nr_depth2dists(const float* depth, int rows, int dn, float* dists, void* stream) {
  if (rows == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(depth && dists && rows >= 0 && dn > 0, "depth2dists arguments");
  depth2dists_kernel<<<blocks_for((long long)rows * dn), TPB, 0, (cudaStream_t)stream>>>(depth, rows, dn, nullptr, dists);
  NR_CHECK_LAUNCH("depth2dists");
  return NR_OK;
}

int nr_depth2inv_dists(const float* depth, const float* depth_range, int rows, int dn, float* dists, void* stream) {
  if (rows == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(depth && dists && depth_range && rows >= 0 && dn > 0, "depth2inv_dists arguments");
  depth2dists_kernel<<<blocks_for((long long)rows * dn), TPB, 0, (cudaStream_t)stream>>>(depth, rows, dn, depth_range, dists);
  NR_CHECK_LAUNCH("depth2inv_dists");
  return NR_OK;
}

int nr_alpha_values2hit_prob(const float* alpha, int rows, int dn, float* hit, void* stream) {
  if (rows == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(alpha && hit && rows >= 0 && dn > 0, "alpha_values2hit_prob arguments");
  alpha2hit_kernel<<<blocks_for(rows), TPB, 0, (cudaStream_t)stream>>>(alpha, rows, dn, hit);
  NR_CHECK_LAUNCH("alpha_values2hit_prob");
  return NR_OK;
}

int nr_project_points(const float* pts, int pn, const float* view_params, int rfn, int h, int w, float* dir, float* pix,
                      float* depth, float* mask, float* valid_z, void* stream) {
  if (pn == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(pts && view_params && pn >= 0 && rfn >= 1, "project_points arguments");
  project_kernel<<<min(blocks_for((long long)pn * rfn), 132 * 32), TPB, 0, (cudaStream_t)stream>>>(pts, pn, view_params, rfn, h, w,
                                                                                                  dir, pix, depth, mask, valid_z);
  NR_CHECK_LAUNCH("project_points");
  return NR_OK;
}

int nr_interpolate_feats(const float* feats, const float* pts, const float* mask, int b, int c, int fh, int fw, int n, float h,
                         float w, int border, int align_corners, float* out, void* stream) {
  if (n == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(feats && pts && out && b >= 1 && c >= 1 && fh >= 1 && fw >= 1 && n >= 0, "interpolate_feats arguments");
  interp_kernel<<<min(blocks_for((long long)b * n), 132 * 32), TPB, 0, (cudaStream_t)stream>>>(feats, pts, mask, b, c, fh, fw, n, h, w,
                                                                                              border, align_corners, out);
  NR_CHECK_LAUNCH("interpolate_feats");
  return NR_OK;
}

int nr_interpolate_feats_bwd(const float* d_out, const float* pts, const float* mask, int b, int c, int fh, int fw, int n, float h,
                             float w, int border, int align_corners, float* d_feats, void* stream) {
  if (n == 0) return NR_OK;
  NR_CHECK_ARG(d_out && pts && d_feats && b >= 1 && c >= 1 && fh >= 1 && fw >= 1 && n >= 0, "interpolate_feats_bwd arguments");
  interp_bwd_kernel<<<min(blocks_for((long long)b * n), 132 * 32), TPB, 0, (cudaStream_t)stream>>>(d_out, pts, mask, b, c, fh, fw, n, h,
                                                                                                  w, border, align_corners, d_feats);
  NR_CHECK_LAUNCH("interpolate_feats_bwd");
  return NR_OK;
}

int nr_sample_fine_depth(const float* depth, const float* hit_prob, const float* depth_range, int rn, int dn, int fine_dn,
                         const float* u, int u_stride, int use_all, int do_sort, float* out, void* stream) {
  if (rn == 0) return NR_OK;   // empty input: nothing to do (pointers of empty tensors are null)
  NR_CHECK_ARG(depth && hit_prob && u && out && rn >= 0 && dn >= 2 && fine_dn >= 1, "sample_fine_depth arguments");
  NR_CHECK_ARG(dn <= 4096 && fine_dn <= 4096, "sample_fine_depth: dn / fine_dn too large");
  const int M = fine_dn + (use_all ? dn : 0);
  const int sort_n = sort_size_for(M);
  const int per_warp = (2 * dn + 8 + sort_n + 3) & ~3;
  int warps = 8;
  while (warps > 1 && size_t(warps) * per_warp * 4 > 160 * 1024) warps >>= 1;
  const size_t smem = size_t(warps) * per_warp * 4;
  NR_CHECK_ARG(smem <= 200 * 1024, "sample_fine_depth shared memory");
  if (opt_in_smem((const void*)fine_depth_kernel, smem, "sample_fine_depth") != NR_OK) return NR_E_CUDA;
  const int grid = min((rn + warps - 1) / warps, 132 * 8);
  fine_depth_kernel<<<grid, warps * 32, smem, (cudaStream_t)stream>>>(depth, hit_prob, depth_range, rn, dn, fine_dn, u, u_stride,
                                                                      use_all, do_sort, sort_n, per_warp, out);
  NR_CHECK_LAUNCH("sample_fine_depth");
  return NR_OK;
}

}  // extern "C"

// ---- DepthInitNet.get_diff_feats (reference network/init_net.py:14-61) ---------------------------------------------
// For every pixel of every reference view: back-project with the view's (normalised inverse) depth, re-project into all
// rfn views, sample their depth maps and images there (bilinear, border clamp, align_corners), and pool the absolute
// colour / inverse-depth differences over the views that see the point: masked mean and variance -> 8 channels.
// One thread per (view, pixel); the rfn re-projections are a loop in registers, so none of the reference's
// [rfn, rfn*h*w, *] intermediates exists.  vp: view_params [rfn,20] (K@Rt | centre | -1/near, -1/far | pad), kinv [rfn,9].
namespace nr {
namespace ops {

__global__ void diff_feats_kernel(const float* __restrict__ imgs, const float* __restrict__ depth_in, const float* __restrict__ poses,
                                  const float* __restrict__ Ks, const float* __restrict__ vps, int rfn, int h, int w,
                                  float* __restrict__ out) {
  __shared__ float kinv[NR_MAX_VIEWS * 9];     // K^-1 per view (closed form in fp64, rounded once; reference: torch.inverse)
  for (int t = threadIdx.x; t < rfn; t += blockDim.x) {
    double k[9], inv[9];
    for (int e = 0; e < 9; ++e) k[e] = double(Ks[9 * t + e]);
    const double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6]);
    inv[0] = (k[4] * k[8] - k[5] * k[7]) / det; inv[1] = (k[2] * k[7] - k[1] * k[8]) / det; inv[2] = (k[1] * k[5] - k[2] * k[4]) / det;
    inv[3] = (k[5] * k[6] - k[3] * k[8]) / det; inv[4] = (k[0] * k[8] - k[2] * k[6]) / det; inv[5] = (k[2] * k[3] - k[0] * k[5]) / det;
    inv[6] = (k[3] * k[7] - k[4] * k[6]) / det; inv[7] = (k[1] * k[6] - k[0] * k[7]) / det; inv[8] = (k[0] * k[4] - k[1] * k[3]) / det;
    for (int e = 0; e < 9; ++e) kinv[9 * t + e] = float(inv[e]);
  }
  __syncthreads();
  const long long hw = (long long)h * w, total = (long long)rfn * hw;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int i = int(idx / hw);
    const long long px = idx - (long long)i * hw;
    const int y = int(px / w), x = int(px - (long long)y * w);
    // depth_in in [0,1] -> metric depth of view i (init_net.py:34-35)
    const float* __restrict__ vi = vps + i * 20;
    const float near_inv = vi[15], far_inv = vi[16];
    const float z = -1.f / (__ldg(depth_in + idx) * (far_inv - near_inv) + near_inv);
    // pts3d = R^T (K^-1 [x z, y z, z]) + (-R^T t)   (depth2pts3d, init_net.py:14-27; t = centre of view i)
    const float* ki = kinv + i * 9;
    const float* __restrict__ P = poses + i * 12;
    const float cx = float(x) * z, cy = float(y) * z;
    float c[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) c[r] = ki[3 * r] * cx + ki[3 * r + 1] * cy + ki[3 * r + 2] * z;
    float X[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) X[r] = (P[r] * c[0] + P[4 + r] * c[1] + P[8 + r] * c[2]) + vi[12 + r];
    const float r0 = __ldg(imgs + ((long long)i * 3 + 0) * hw + px), g0 = __ldg(imgs + ((long long)i * 3 + 1) * hw + px),
                b0 = __ldg(imgs + ((long long)i * 3 + 2) * hw + px);
    float n = 0.f, s[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < rfn; ++j) {
      const float* __restrict__ vp = vps + j * 20;
      const Proj pj = project(vp, X[0], X[1], X[2], h, w);
      if (!pj.valid) continue;
      // bilinear, border clamp, align_corners (interpolate_feats(..., padding_mode='border', align_corners=True))
      const Taps t = border_taps(pj.ux, pj.uy, h, w, h, w, true);
      const float* __restrict__ img = imgs + (long long)j * 3 * hw;
      const float dr = fabsf(bilinear(img, w, t) - r0);
      const float dg = fabsf(bilinear(img + hw, w, t) - g0);
      const float db = fabsf(bilinear(img + 2 * hw, w, t) - b0);
      // depth map of view j: the reference samples the METRIC depth of view j (depth = -1/depth_in with view j's range)
      const float* __restrict__ dj = depth_in + (long long)j * hw;
      const float nj = vp[15], fj = vp[16];
      auto metric = [&](float t) { return -1.f / (t * (fj - nj) + nj); };
      const float dint = metric(dj[t.y0 * w + t.x0]) * t.w[0] + metric(dj[t.y0 * w + t.x1]) * t.w[1] + metric(dj[t.y1 * w + t.x0]) * t.w[2] +
                         metric(dj[t.y1 * w + t.x1]) * t.w[3];
      // normalised by the range of the view projected INTO (init_net.py:49-50: near/far broadcast over the first axis = j)
      const float dd = fminf(fabsf(-1.f / fmaxf(dint, 1e-5f) + 1.f / fmaxf(pj.zh, 1e-5f)) / (fj - nj), 1.5f);
      n += 1.f;
      s[0] += dr; s[1] += dg; s[2] += db; s[3] += dd;
      s2[0] = fmaf(dr, dr, s2[0]); s2[1] = fmaf(dg, dg, s2[1]); s2[2] = fmaf(db, db, s2[2]); s2[3] = fmaf(dd, dd, s2[3]);
    }
    // masked_mean_var (ops.py:36-41): mean = sum / max(n, 1e-4); var = sum((x - mean)^2 mask) / max(n, 1e-4)
    const float inv_n = 1.f / fmaxf(n, 1e-4f);
    float* __restrict__ o = out + (long long)i * 8 * hw + px;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float mean = s[k] * inv_n;
      const float var = fmaxf((s2[k] - 2.f * mean * s[k] + mean * mean * n) * inv_n, 0.f);
      // channel order: rgb_mean (3), rgb_var (3), dpt_mean, dpt_var
      if (k < 3) { o[k * hw] = mean; o[(3 + k) * hw] = var; }
      else { o[6 * hw] = mean; o[7 * hw] = var; }
    }
  }
}

}  // namespace ops
}  // namespace nr

extern "C" int nr_diff_feats(const float* imgs, const float* depth_in, const float* poses, const float* Ks, const float* view_params,
                             int rfn, int h, int w, float* out, void* stream) {
  using namespace nr;
  NR_CHECK_ARG(imgs && depth_in && poses && Ks && view_params && out, "null device pointer");
  NR_CHECK_ARG(rfn >= 1 && rfn <= NR_MAX_VIEWS && h > 1 && w > 1, "shape");
  const long long total = (long long)rfn * h * w;
  ops::diff_feats_kernel<<<min(ops::blocks_for(total), 132 * 16), ops::TPB, 0, (cudaStream_t)stream>>>(imgs, depth_in, poses, Ks, view_params,
                                                                                                    rfn, h, w, out);
  NR_CHECK_LAUNCH("diff_feats");
  return NR_OK;
}

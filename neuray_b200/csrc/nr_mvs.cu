// CostVolumeInitNet's frozen MVSNet on the GPU (SURVEY.md 8(f) row f4): kernels over the per-voxel routines of nr_mvs.cuh, the
// stream backend of nr_mvs_graph.cuh and the C-ABI entry points (include/neuray_b200.h).
#include "nr_mvs_graph.cuh"

namespace nr {
namespace mvs {

template <int CG>
__global__ void __launch_bounds__(128) conv_kernel(const __grid_constant__ ConvP p) {
  const int groups = p.Cout / CG;
  const long long total = (long long)p.Do * p.Ho * p.Wo * groups;
  for (long long i = (long long)blockIdx.x * 128 + threadIdx.x; i < total; i += (long long)gridDim.x * 128) {
    float acc[CG];
    conv_voxel<CG>(p, i / groups, int(i % groups), acc);       // the groups of a voxel sit in neighbouring lanes: its x loads coalesce
  }
}
__global__ void __launch_bounds__(128) volume_kernel(const __grid_constant__ VolumeP p) {
  const long long total = (long long)p.dn * p.h * p.w;
  for (long long v = (long long)blockIdx.x * 128 + threadIdx.x; v < total; v += (long long)gridDim.x * 128) volume_voxel(p, v);
}
__global__ void __launch_bounds__(128) softmax_kernel(const __grid_constant__ SoftmaxP p) {
  const int pix = blockIdx.x * 128 + threadIdx.x;
  if (pix >= p.ho * p.wo) return;
  float tmp[128];                      // dn <= 128 (checked by the launcher); cost_volume_sn is 64 in every shipped config
  softmax_pixel(p, pix, tmp);
}
__global__ void __launch_bounds__(256) resize_kernel(const __grid_constant__ ResizeP p) {
  const long long total = (long long)p.N * p.Ho * p.Wo;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) resize_pixel(p, i);
}
__global__ void transforms_kernel(const __grid_constant__ TransformsP p) {
  const int i = blockIdx.x;            // reference view
  for (int k = threadIdx.x; k < p.in.nn; k += blockDim.x) {
    const int s = p.in.nn_ids[i * p.in.nn + k];
    pair_transform(p.in.ref_Ks + 9 * i, p.in.ref_poses + 12 * i, p.in.src_Ks + 9 * s, p.in.src_poses + 12 * s, p.ratio, p.transforms + (i * p.in.nn + k) * 12);
  }
  for (int j = threadIdx.x; j < p.in.dn; j += blockDim.x)
    p.depth_vals[i * p.in.dn + j] = depth_val(p.in.depth_range[2 * i], p.in.depth_range[2 * i + 1], j, p.in.dn);
}

struct PackArgs {
  LayerSpec L[N_LAYERS];
  const float* w[N_LAYERS]; const float* g[N_LAYERS]; const float* b[N_LAYERS]; const float* m[N_LAYERS]; const float* v[N_LAYERS];
  float* out;
};
__global__ void __launch_bounds__(256) pack_kernel(const __grid_constant__ PackArgs a) {
  const LayerSpec& l = a.L[blockIdx.y];
  const int li = blockIdx.y;
  const long long taps = l.dims == 3 ? (long long)l.k * l.k * l.k : (long long)l.k * l.k;
  const long long n = taps * l.cin * l.cout;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < n; e += (long long)gridDim.x * 256)
    a.out[l.w_off + e] = a.w[li][weight_source(l, e)];
  if (blockIdx.x == 0)
    for (int o = threadIdx.x; o < l.cout; o += 256) {
      float sc = 1.f, sh = 0.f;
      if (l.has_bn) fold_bn(a.g[li][o], a.b[li][o], a.m[li][o], a.v[li][o], sc, sh);
      else if (l.has_bias) sh = a.b[li][o];
      a.out[l.scale_off + o] = sc;
      a.out[l.shift_off + o] = sh;
    }
}

inline unsigned grid_of(long long items, int per, int cap) {
  long long g = (items + per - 1) / per;
  if (g > cap) g = cap;
  return unsigned(g < 1 ? 1 : g);
}

struct StreamOps {
  cudaStream_t st;
  int sms, rc;
  void mvs_conv(const ConvP& p) {
    if (rc != NR_OK) return;
    const int cg = group_size(p.Cout);
    const unsigned g = grid_of((long long)p.Do * p.Ho * p.Wo * (p.Cout / cg), 128, 32 * sms);
    if (cg == 1) conv_kernel<1><<<g, 128, 0, st>>>(p);
    else if (cg == 8 && p.Cout % 8 == 0) conv_kernel<8><<<g, 128, 0, st>>>(p);
    else rc = NR_E_UNSUPPORTED;
  }
  void mvs_volume(const VolumeP& p) { if (rc == NR_OK) volume_kernel<<<grid_of((long long)p.dn * p.h * p.w, 128, 32 * sms), 128, 0, st>>>(p); }
  void mvs_softmax(const SoftmaxP& p) { if (rc == NR_OK) softmax_kernel<<<(p.ho * p.wo + 127) / 128, 128, 0, st>>>(p); }
  void mvs_resize(const ResizeP& p) { if (rc == NR_OK) resize_kernel<<<grid_of((long long)p.N * p.Ho * p.Wo, 256, 16 * sms), 256, 0, st>>>(p); }
  void mvs_transforms(const TransformsP& p) { if (rc == NR_OK) transforms_kernel<<<p.in.rfn, 64, 0, st>>>(p); }
};

struct NullOps {
  void mvs_conv(const ConvP&) {}
  void mvs_volume(const VolumeP&) {}
  void mvs_softmax(const SoftmaxP&) {}
  void mvs_resize(const ResizeP&) {}
  void mvs_transforms(const TransformsP&) {}
};

inline size_t workspace_bytes(const MvsNet& net, const MvsIn& in) {
  NullOps ops;
  enc::Arena ar{enc::DRY_BASE, ~size_t(0) / 2, 0, true};
  if (!mvsnet_graph(ops, ar, net, nullptr, nullptr, in, (float*)enc::DRY_BASE, (float*)enc::DRY_BASE)) return 0;
  // feature_net / cost_reg_net release their intermediates: the high-water mark is what counts
  return ar.peak + 256;
}

}  // namespace mvs
}  // namespace nr

using namespace nr;

static mvs::MvsIn to_in(const NrMvsIn* a) {
  mvs::MvsIn in;
  in.ref_imgs = a->ref_imgs; in.src_imgs = a->src_imgs; in.ref_Ks = a->ref_Ks; in.ref_poses = a->ref_poses; in.src_Ks = a->src_Ks;
  in.src_poses = a->src_poses; in.depth_range = a->depth_range; in.nn_ids = a->nn_ids;
  in.rfn = a->rfn; in.sn = a->sn; in.nn = a->nn; in.h = a->h; in.w = a->w; in.dn = a->dn; in.is_train = a->is_train;
  return in;
}

extern "C" int nr_mvsnet_layout(int* n_tensors, long long* packed_floats) {
  NR_CHECK_ARG(n_tensors != nullptr && packed_floats != nullptr, "mvsnet_layout");
  mvs::MvsNet net;
  mvs::build_mvsnet(net);
  *n_tensors = net.n_tensors;
  *packed_floats = net.total + 8;          // + ImageNet mean[3] | 1/std[3]
  return NR_OK;
}

extern "C" int nr_mvsnet_pack(const float* const* params, int n_params, float* packed, void* stream) {
  NR_CHECK_ARG(params != nullptr && packed != nullptr, "mvsnet_pack: null pointer");
  mvs::MvsNet net;
  mvs::build_mvsnet(net);
  NR_CHECK_ARG(n_params == net.n_tensors, "mvsnet_pack: wrong number of tensors (state_dict order of MVSNet: conv weight, then the "
                                          "norm's weight, bias, running_mean, running_var; conv bias where the layer has one)");
  mvs::PackArgs a;
  int t = 0;
  for (int i = 0; i < mvs::N_LAYERS; ++i) {
    a.L[i] = net.L[i];
    a.w[i] = params[t++];
    a.g[i] = a.b[i] = a.m[i] = a.v[i] = nullptr;
    if (net.L[i].has_bn) { a.g[i] = params[t++]; a.b[i] = params[t++]; a.m[i] = params[t++]; a.v[i] = params[t++]; }
    else if (net.L[i].has_bias) a.b[i] = params[t++];
  }
  for (int i = 0; i < t; ++i) NR_CHECK_ARG(params[i] != nullptr, "mvsnet_pack: null tensor");
  a.out = packed;
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(packed, 0, size_t(net.total + 8) * sizeof(float), st);
  mvs::pack_kernel<<<dim3(64, mvs::N_LAYERS), 256, 0, st>>>(a);
  // init_net.py:222-225: ImageNet statistics
  const float consts[8] = {0.485f, 0.456f, 0.406f, 1.f / 0.229f, 1.f / 0.224f, 1.f / 0.225f, 0.f, 0.f};
  cudaMemcpyAsync(packed + net.total, consts, sizeof(consts), cudaMemcpyHostToDevice, st);
  NR_CHECK_LAUNCH("mvsnet_pack");
  return NR_OK;
}

static int check_in(const NrMvsIn* a) {
  NR_CHECK_ARG(a != nullptr, "mvsnet: null input");
  NR_CHECK_ARG(a->rfn >= 1 && a->sn >= 1 && a->nn >= 1 && a->h >= 32 && a->w >= 32 && a->dn >= 8 && a->dn <= 128, "mvsnet: shape");
  return NR_OK;
}

extern "C" int nr_mvsnet_dims(int h, int w, int is_train, int* ho, int* wo) {
  NR_CHECK_ARG(ho != nullptr && wo != nullptr && h >= 32 && w >= 32, "mvsnet_dims");
  const mvs::MvsDims d = mvs::mvs_dims(h, w, is_train);
  const bool resized = d.hr != h || d.wr != w;
  *ho = resized ? h / 4 : d.h4;
  *wo = resized ? w / 4 : d.w4;
  return NR_OK;
}

extern "C" long long nr_mvsnet_workspace(const NrMvsIn* a) {
  if (check_in(a) != NR_OK) return 0;
  mvs::MvsNet net;
  mvs::build_mvsnet(net);
  return (long long)mvs::workspace_bytes(net, to_in(a));
}

extern "C" int nr_mvsnet_fwd(const float* packed, const NrMvsIn* a, float* prob, float* depth, void* workspace, long long workspace_bytes, void* stream) {
  const int rc0 = check_in(a);
  if (rc0 != NR_OK) return rc0;
  NR_CHECK_ARG(packed && prob && depth && workspace, "mvsnet: null pointer");
  NR_CHECK_ARG(a->ref_imgs && a->src_imgs && a->ref_Ks && a->ref_poses && a->src_Ks && a->src_poses && a->depth_range && a->nn_ids, "mvsnet: null input pointer");
  mvs::MvsNet net;
  mvs::build_mvsnet(net);
  enc::Arena ar{(char*)workspace, size_t(workspace_bytes), 0, true};
  int sms;
  if (sm_count(&sms, "mvsnet") != NR_OK) return NR_E_CUDA;
  mvs::StreamOps ops{(cudaStream_t)stream, sms, NR_OK};
  const bool ok = mvs::mvsnet_graph(ops, ar, net, packed, packed + net.total, to_in(a), prob, depth);
  if (ops.rc != NR_OK) return ops.rc;
  NR_CHECK_ARG(ok, "mvsnet: workspace too small (nr_mvsnet_workspace), or a size the regulariser cannot take (depth planes and h/4, w/4 "
                   "multiples of 8, as the reference's skip additions require)");
  NR_CHECK_LAUNCH("mvsnet");
  return NR_OK;
}

/*
 * neuray_b200 C-ABI  (libneuray_b200.so)
 *
 * The reference (liuyuan-pal/NeuRay) is pure Python/PyTorch: it has no FFI or operator-plugin layer, so there is
 * no existing binding to replace.  The drop-in boundary is therefore the reference's Python API for the per-ray
 * rendering path (network/render_ops.py, NeuralRayBaseRenderer.render_by_depth / render_impl / render) and THIS
 * header is the native interface a maintainer binds underneath it (ctypes stub in INTEGRATION.md; the in-tree
 * binding is neuray_b200/_lib.py).  Each entry point cites the reference code it replaces.
 *
 * Conventions
 *   - plain C, no torch types; every pointer is a DEVICE pointer to contiguous fp32 unless stated otherwise
 *   - the caller allocates every output and workspace; nothing is allocated or freed across the ABI
 *   - every call is enqueued on `stream` (a cudaStream_t passed as void*) and never synchronises the host
 *   - returns 0 on success, a negative NR_E_* code on failure; nr_last_error() gives a thread-local message
 *   - one query view per call (qn == 1), exactly like every call site in the reference
 *   - sm_90a (H100) only; there is no CPU fallback
 */
#ifndef NEURAY_B200_H
#define NEURAY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NR_ABI_VERSION 13

#define NR_OK 0
#define NR_E_INVALID (-1)   /* bad argument (null pointer, unsupported shape) */
#define NR_E_CUDA (-2)      /* a CUDA runtime call / launch failed */
#define NR_E_UNSUPPORTED (-3)

#define NR_MAX_VIEWS 32     /* reference views per call */
#define NR_MAX_SAMPLES 256  /* depth samples per ray per pass */
#define NR_POINT_REC 20     /* floats per point in the point-kernel -> ray-kernel record */

int nr_abi_version(void);
const char* nr_last_error(void);

/* ---- weight layout --------------------------------------------------------------------------------------
 * Host code packs one flat fp32 buffer per pass (coarse / fine) in the order the kernels stage it.  The
 * offsets (in floats) come from the library so that host and device cannot disagree. */
typedef struct NrWeightLayout {
  int32_t total_point;      /* floats in the point-kernel weight buffer */
  int32_t total_ray;        /* floats in the ray-kernel weight buffer (without pos_encoding) */
  /* point kernel, dist-decoder heads (mean, var, aw, vis): block h at dd_head + h*dd_head_stride */
  int32_t dd_head, dd_head_stride;
  int32_t dd_l0_w, dd_l0_b, dd_l1_w, dd_l1_b, dd_l2_w, dd_l2_b;   /* offsets inside a head block */
  /* group B */
  int32_t grp_b, pe0_w, pe0_b, pe1_w, pe1_b, rd0_w, rd0_b, rd1_w, rd1_b, nf0_w, nf0_b, nf1_w, nf1_b, grp_b_size;
  /* group C */
  int32_t hoist_w, hoist_b, base0_w, base1_w, base1_b;
  /* group D1 */
  int32_t grp_d1, vis0_w, vis0_b, vis1_w, vis1_b, vis1l_w, vis1l_b, v20_w, v20_b, v21_w, v21_b,
          rgb0_w, rgb0_b, rgb1_w, rgb1_b, rgb2_w, rgb2_b, grp_d1_size;
  /* group D2 */
  int32_t grp_d2, geo0_w, geo0_b, geo1_w, geo1_b, grp_d2_size;
  /* ray kernel */
  int32_t wq, wk, wv, wfc, ln_w, ln_b, og0_w, og0_b, og1_w, og1_b;
} NrWeightLayout;

int nr_weight_layout(NrWeightLayout* out);

/* Layout of the tensor-core weight buffer (floats; details in csrc/nr_common.cuh namespace tcl). */
typedef struct NrTcLayout {
  int32_t total, stage, head0, pe0, pe1, b0, b1, v01, v2r, rd1, hst, g0;
} NrTcLayout;
int nr_tc_layout(NrTcLayout* out);

/* ---- weight packing ------------------------------------------------------------------------------------- */

/* One nn.Linear of the reference: weight [out][in] row-major (PyTorch layout), bias [out]; device pointers. */
typedef struct NrLinear {
  const float* w;
  const float* b;
} NrLinear;

/* The parameters of ONE pass (coarse: dist_decoder + agg_net; fine: fine_dist_decoder + fine_agg_net), by the reference's
 * module structure (dist_decoder.py:64-97, aggregate_net.py:28-32, ibrnet.py:246-290, 52-102):
 *   dist_decoder[h][l]  head h = mean, var, aw, vis (all-NULL vis head when the decoder has none); l = layers .0 .2 .4
 *   prob_embed[l]       agg_net.prob_embed.{0,2}
 *   the rest            agg_net.agg_impl.<name>.{0,2(,4)}; ray attention: w_qs / w_ks / w_vs / fc weights (no bias),
 *                       layer_norm weight + bias */
typedef struct NrPassWeights {
  NrLinear dist_decoder[4][3];
  NrLinear prob_embed[2];
  NrLinear ray_dir_fc[2], neuray_fc[2], base_fc[2], vis_fc[2], vis_fc2[2], rgb_fc[3], geometry_fc[2], out_geometry_fc[2];
  const float *w_qs, *w_ks, *w_vs, *attn_fc, *layer_norm_w, *layer_norm_b;
} NrPassWeights;

/* Packs the three weight buffers of a pass (once per checkpoint load; in training once per optimizer step):
 * w_point [NrWeightLayout.total_point], w_ray [NrWeightLayout.total_ray], w_tc [NrTcLayout.total].  One memset + one
 * kernel per buffer set on `stream`; `w` is a HOST struct of device pointers. */
int nr_pack_weights(const NrPassWeights* w, float* w_point, float* w_ray, float* w_tc, void* stream);

/* The tensor-core buffer of the point kernel's TF32 mode (nr_render_pass_fwd_tf32, nr_point_kernel_tf32): w_tc
 * [NrTcLayout.total] in the same layout, each weight rounded to the nearest tf32 value (ties away from zero) in its hi
 * slot, the lo slots zero.  The TF32 mode reads w_point and w_ray from nr_pack_weights as usual. */
int nr_pack_weights_tf32(const NrPassWeights* w, float* w_tc, void* stream);

/* ---- per-frame packing ---------------------------------------------------------------------------------- */

/* que_cam [24] (NrPassParams.que_cam) and view_params [rfn,20] (NrPassParams.view_params) from the reference's camera
 * tensors (device pointers): que_pose [3,4] world->camera, que_K [3,3], que_range [2]; ref_poses [rfn,3,4], ref_Ks
 * [rfn,3,3], ref_range [rfn,2] (NULL: the -1/near, -1/far entries are zero).  Replaces the torch expressions of
 * render_ops.py:14-20, 95, 112 (K^-1, K@Rt, -R^T t), evaluated in fp64 and rounded once.  Either output may be NULL. */
int nr_camera_blocks(const float* que_pose, const float* que_K, const float* que_range, const float* ref_poses,
                     const float* ref_Ks, const float* ref_range, int rfn, float* que_cam, float* view_params, void* stream);

/* NCHW -> channel-last repack of the reference views' maps, once per frame.
 *   ray_feats, img_feats : [rfn,32,fh,fw]   (reference: ref_imgs_info['ray_feats'|'img_feats'], renderer.py:229-231)
 *   imgs                 : [rfn,3,h,w]
 *   out_feat             : [rfn,fh,fw,64]   ray_feats in channels 0..31, img_feats in 32..63 (256 B per texel)
 *   out_rgb              : [rfn,h,w,4]      rgb + zero pad (16 B per texel)
 * ray_feats == img_feats == NULL: only out_rgb is written (out_feat was filled in place by nr_image_encoder_fwd /
 * nr_vis_encoder_fwd).                                                                                             */
int nr_pack_feature_maps(const float* ray_feats, const float* img_feats, const float* imgs, int rfn, int h, int w,
                         int fh, int fw, float* out_feat, float* out_rgb, void* stream);

/* ---- fused render pass ---------------------------------------------------------------------------------- */

typedef struct NrPassParams {
  /* query rays */
  const float* coords;       /* [rn,2] pixel (x,y) */
  const float* que_depth;    /* [rn,dn] sample depths of this pass (sorted along dn) */
  const float* que_cam;      /* [24]: R^T row-major (9) | camera centre (3) | K^-1 row-major (9) | near, far, 0 */
  int32_t rn, dn;
  /* reference views */
  const float* feat;         /* [rfn,fh,fw,64]  from nr_pack_feature_maps */
  const float* rgb;          /* [rfn,h,w,4] */
  const float* view_params;  /* [rfn,20]: K@Rt row-major (12) | camera centre (3) | -1/near, -1/far | pad(3) */
  int32_t rfn, h, w, fh, fw;
  /* weights of this pass */
  const float* w_point;      /* NrWeightLayout.total_point floats */
  const float* w_ray;        /* NrWeightLayout.total_ray floats */
  const float* pos_enc;      /* [dn,16] sinusoid table (reference ibrnet.py:305-313) */
  int32_t use_vis;           /* 1: compute_prob multiplies the CDFs by the decoder's vis head (dist_decoder.py:127) */
  float var_bias;            /* AddBias value of the variance head (dist_decoder.py:78, ops.py:78-84) */
  /* ray_mask thresholds (renderer.py:195-198) */
  int32_t ray_mask_view_num, ray_mask_point_num;
  /* workspace: rn*dn*NR_POINT_REC floats */
  float* point_rec;
  /* outputs (any may be NULL to skip) */
  float* pixel_colors;       /* [rn,3]   pixel_colors_nr */
  float* hit_prob;           /* [rn,dn]  hit_prob_nr */
  float* render_depth;       /* [rn] */
  uint8_t* ray_mask;         /* [rn] bool */
  /* optional fused hierarchical resampling (sample_fine_depth + sort, render_ops.py:172-229, renderer.py:205-213) */
  int32_t fine_dn;           /* 0: off */
  int32_t fine_use_all;      /* 1: merge the coarse depths in (fine_depth_use_all) -> dn + fine_dn samples */
  const float* fine_u;       /* quantiles: [fine_dn] if fine_u_stride == 0, else [rn,fine_dn] with that row stride */
  int32_t fine_u_stride;
  float* fine_depth;         /* [rn, fine_dn (+dn)] sorted */
  /* tensor-core weights of this pass (NrTcLayout.total floats: hi/lo tf32 parts, pre-swizzled; nr_pack_weights) */
  const float* w_tc;
} NrPassParams;

/* One render_by_depth (reference renderer.py:168-203): depth2inv_dists + depth2points + project_points_dict +
 * predict_proj_ray_prob + get_img_feats + network_rendering (+ ray_mask, render_depth), and optionally the
 * following sample_fine_depth.  Two kernels: point kernel (per point x view) and ray kernel (per ray). */
int nr_render_pass_fwd(const NrPassParams* p, void* stream);

/* The same pass with the point kernel in TF32 mode: one tensor-core pass per product (3xTF32 issues three) on operands
 * rounded to nearest, p->w_tc from nr_pack_weights_tf32 -- the arithmetic torch 1.7 - 1.11 used for nn.Linear on
 * Ampere and later GPUs by default (~1e-3 relative per layer).  The ray kernel is the same as in nr_render_pass_fwd.
 * nr_render_pass_bwd recomputes a pass in fp32, so a pass whose gradient is wanted runs nr_render_pass_fwd. */
int nr_render_pass_fwd_tf32(const NrPassParams* p, void* stream);

/* Direct rendering of the same pass (reference renderer.py:85-125, 181-185 and sph_solver.py, cfg use_dr_prediction),
 * forward only.  Enqueue it after nr_render_pass_fwd of the same NrPassParams: it reads the pass' inputs and, with
 * use_nr_color, the NR colours of its point record.  Per point: the per-view alpha logits of the active pass' dist decoder
 * (ground state where the view misses the point) pooled by visibility, and the colour of a degree-3 spherical-harmonics fit
 * to the views' colours weighted by hit probability (regs on the normal matrix's diagonal; sph_fitter.regs of the
 * reference) or, with use_nr_color (use_nr_color_for_dr), the NR colour; per ray: sigmoid, alpha_values2hit_prob and the
 * colour sum.  Two kernels, no host synchronisation. */
typedef struct NrDrParams {
  float regs[16];            /* SphericalHarmonicsSolver(3).regs: 0, 0.001 x3, 0.005 x5, 0.05 x7 by default */
  float alpha_ground_state;  /* cfg alpha_value_ground_state */
  int32_t use_nr_color;      /* cfg use_nr_color_for_dr */
  float* point_colors;       /* workspace [rn,dn,3] */
  float* pixel_colors_dr;    /* [rn,3] */
  float* hit_prob_dr;        /* [rn,dn] */
} NrDrParams;
int nr_direct_render(const NrPassParams* p, const NrDrParams* d, void* stream);

/* Per-view visibility of each rendered pixel (cfg render_visibility): visibility[r, v] = Σ_d hit_prob[r, d] · vis_v[r, d],
 * where vis_v is the reference's masked prj_dict['vis'] of the same pass (renderer.py:79-82: compute_prob's visibility
 * of the active pass' dist decoder, times the projection mask), recomputed per (point, view) in fp32, and hit_prob the
 * pass' compositing weight (hit_prob_nr).  Views in view_params order; unnormalised, like render_depth.  Enqueue it after
 * nr_render_pass_fwd (or _tf32) of the same NrPassParams: it reads the pass' inputs and its hit_prob.  Each ray's sum
 * runs in an order fixed by dn alone, so a ray's result does not depend on the chunk or launch that renders it.
 * One kernel, no host synchronisation, no workspace. */
typedef struct NrVisParams {
  const float* hit_prob;     /* [rn,dn]: the pass' hit_prob output */
  float* visibility;         /* [rn,rfn] */
} NrVisParams;
int nr_view_visibility(const NrPassParams* p, const NrVisParams* v, void* stream);

/* Per-view colour-blend weight of each rendered pixel (cfg render_blend_weights): nr_render_pass_fwd (or _tf32) with the
 * point kernel also exporting each (view, point) row's blend weight w, then one reduction kernel:
 *   blend_weights[r, v] = Σ_d hit_prob[r, d] · w[v, r, d]
 * w is the reference's blending_weights_valid of the same pass (ibrnet.py:362-366: softmax over the views of rgb_fc's
 * logit, set to -1e9 where the projection mask is 0; a point no view sees gets 1/rfn from every view), hit_prob the pass'
 * compositing weight (hit_prob_nr, so p->hit_prob is required).  Views in view_params order; unnormalised, like
 * render_depth: Σ_v blend_weights[r, v] = Σ_d hit_prob[r, d].  Each ray's sum runs in an order fixed by dn alone, so a ray's
 * result does not depend on the chunk or launch that renders it.  Every other output equals the one of the twin without
 * _blend bit for bit.  Three kernels, no host synchronisation.  blend_weights may be NULL (accepted within NR_ABI_VERSION
 * 13): the pass still fills row_blend, for nr_view_colors, and the reduction is skipped (two kernels). */
typedef struct NrBlendParams {
  float* row_blend;          /* workspace [rfn, rn*dn] */
  float* blend_weights;      /* [rn,rfn], or NULL */
} NrBlendParams;
int nr_render_pass_fwd_blend(const NrPassParams* p, const NrBlendParams* b, void* stream);
int nr_render_pass_fwd_tf32_blend(const NrPassParams* p, const NrBlendParams* b, void* stream);   /* TF32 mode */

/* Per-view weights of each rendered pixel inside the aggregation net (cfg render_agg_weights): nr_render_pass_fwd (or
 * _tf32) with the point kernel also exporting each (view, point) row's two pooling weights and its blend weight, then one
 * reduction kernel per output, the one of nr_render_pass_fwd_blend:
 *   neuray_weights[r, v]   = Σ_d hit_prob[r, d] · weight0[v, r, d]
 *   geometry_weights[r, v] = Σ_d hit_prob[r, d] · weight[v, r, d]
 *   blend_weights[r, v]    as in nr_render_pass_fwd_blend (skipped when blend_weights is NULL)
 * weight0 is the reference's NeuRay weight of the same pass (ibrnet.py:334-337: sigmoid(neuray_fc) · mask / (Σ_v mask +
 * 1e-8), the weight of the first pooled mean/variance), weight its geometry weight (ibrnet.py:349-350: vis / (Σ_v vis +
 * 1e-8) with vis = vis_fc2(x · vis) · mask, the weight of the pooling in front of geometry_fc); hit_prob is the pass'
 * compositing weight (p->hit_prob is required).  Σ_v weight = Σ_v vis / (Σ_v vis + 1e-8), weight0 <= mask / (Σ_v mask +
 * 1e-8), and a point that no view sees has 0 in both.  Views in view_params order; unnormalised, like render_depth.  The
 * sums run in an order fixed by dn alone, so a ray's result does not depend on the chunk or launch that renders it.  Every
 * other output equals the one of nr_render_pass_fwd (or _blend) bit for bit.  Four or five kernels, no host
 * synchronisation. */
typedef struct NrAggParams {
  float* rows;               /* workspace [3, rfn, rn*dn]: blend weight, weight0, weight */
  float* neuray_weights;     /* [rn,rfn] */
  float* geometry_weights;   /* [rn,rfn] */
  float* blend_weights;      /* [rn,rfn], or NULL */
} NrAggParams;
int nr_render_pass_fwd_agg(const NrPassParams* p, const NrAggParams* a, void* stream);
int nr_render_pass_fwd_tf32_agg(const NrPassParams* p, const NrAggParams* a, void* stream);   /* TF32 mode */

/* Where each working view puts the surface along each rendered pixel's ray (cfg render_view_depth): nr_render_pass_fwd
 * (or _tf32) with the point kernel also exporting each (view, point) row's masked hit probability, next to the blend and
 * pooling weights of nr_render_pass_fwd_agg, then one reduction kernel per output, the one of nr_render_pass_fwd_blend:
 *   view_hit[r, v]   = Σ_d hit_v[r, d]
 *   view_depth[r, v] = Σ_d hit_v[r, d] · que_depth[r, d]
 *   blend_weights, neuray_weights, geometry_weights   as in nr_render_pass_fwd_agg (each skipped when NULL)
 * hit_v is the reference's masked prj_dict['hit_prob'] of the same pass (renderer.py:75-82: compute_prob(is_ref=True) of
 * the pass' dist decoder, times the projection mask).  Both sums are unnormalised, like render_depth: view_depth / view_hit
 * is view v's expected surface depth along the ray, comparable with render_depth / Σ_d hit_prob.  Σ_d hit_v is not bounded
 * by 1: each bin is centred on the sample's inverse depth in view v's range but is as wide as the query's interval, and the
 * last interval is 1e6, so the last sample carries all of the view's mass beyond it (a view whose surface lies past far
 * reads as far).  A view that sees none of a ray's samples has exactly 0 in both.  Views in view_params order.  The sums
 * run in an order fixed by dn alone, so a ray's result does not depend on the chunk or launch that renders it.  Every
 * other output equals the one of nr_render_pass_fwd (or _blend, _agg) bit for bit.  p->hit_prob is required only with the
 * blend or agg outputs.  Four to seven kernels, no host synchronisation.  This struct and the two entry points were added
 * within NR_ABI_VERSION 13: nothing existing changed, so a host built against the earlier version-13 header still works. */
typedef struct NrViewParams {
  float* rows;               /* workspace [4, rfn, rn*dn]: blend weight, weight0, weight, hit */
  float* view_hit;           /* [rn,rfn] */
  float* view_depth;         /* [rn,rfn] */
  float* blend_weights;      /* [rn,rfn], or NULL */
  float* neuray_weights;     /* [rn,rfn], or NULL (together with geometry_weights) */
  float* geometry_weights;   /* [rn,rfn], or NULL (together with neuray_weights) */
} NrViewParams;
int nr_render_pass_fwd_view(const NrPassParams* p, const NrViewParams* w, void* stream);
int nr_render_pass_fwd_tf32_view(const NrPassParams* p, const NrViewParams* w, void* stream);   /* TF32 mode */

/* What colour each working view puts into each rendered pixel (cfg render_view_colors): one reduction kernel, enqueued
 * after nr_render_pass_fwd_blend, _agg or _view (or their _tf32 twins) of the same NrPassParams, on plane 0 of that
 * call's workspace (the blend row; blend_weights may be NULL) and the pass' hit_prob:
 *   view_colors[r, v, c] = Σ_d hit_prob[r, d] · w[v, r, d] · rgb_v[r, d, c]
 * w is the reference's blending_weights_valid (ibrnet.py:362-366) and rgb_v its masked prj_dict['rgb'] (render_ops.py:
 * 132-139: the view's image at the sample's projection, 0 where the projection mask is 0), the colour the aggregation net
 * blends: rgb_out = Σ_v rgb_in · blending_weights_valid (ibrnet.py:366-367).  So Σ_v view_colors[r, v] = pixel_colors[r]
 * up to fp32 rounding, and a view that sees none of a ray's samples has exactly 0.  Views in view_params order;
 * unnormalised (view_colors / blend_weights is the colour the view showed, averaged over the surface).  Each ray's sums
 * run in an order fixed by dn alone, with no atomics, so a ray's result does not depend on the chunk or launch that
 * renders it.  One kernel, no host synchronisation, no workspace of its own.  This struct and the entry point were added
 * within NR_ABI_VERSION 13: nothing existing changed, so a host built against the earlier version-13 header still works. */
typedef struct NrColorParams {
  const float* row_blend;    /* [rfn, rn*dn]: plane 0 of the workspace of the pass' _blend, _agg or _view call */
  const float* hit_prob;     /* [rn,dn]: the pass' hit_prob output */
  float* view_colors;        /* [rn,rfn,3] */
} NrColorParams;
int nr_view_colors(const NrPassParams* p, const NrColorParams* c, void* stream);

/* Only the point kernel / only the ray kernel (profiling and stage-level tests). */
int nr_point_kernel(const NrPassParams* p, void* stream);
int nr_point_kernel_tf32(const NrPassParams* p, void* stream);   /* TF32 mode, as in nr_render_pass_fwd_tf32 */
int nr_ray_kernel(const NrPassParams* p, void* stream);

/* Stage-level debug tap of the point kernel: per (view, point) rows of
 * [mask, z, hit, vis, pix_x, pix_y, dir(3), rgb(3), ray_feats(32), img_feats(32)] = 76 floats.  dbg: [rfn,rn*dn,76] */
int nr_point_kernel_debug(const NrPassParams* p, float* dbg, void* stream);

/* Diagnostics: the tensor-core point kernel with clock64() stamps at its phase boundaries (CTA 0, the lead thread of
 * each 128-row block): timing[tile < 64][2][32] device buffer of int64. */
int nr_point_kernel_timing(const NrPassParams* p, long long* timing, void* stream);

/* ---- stand-alone render_ops (reference network/render_ops.py; same names in neuray_b200/render_ops.py) ------- */

/* Depth ranges are DEVICE pointers to [near, far] (one query view): the reference keeps depth_range on the device and no
 * entry point forces a device->host read of it.
 * sample_depth (render_ops.py:146-170).  jitter: NULL or [rn,dn-2] uniforms in [0,1). */
int nr_sample_depth(const float* depth_range, int rn, int dn, const float* jitter, float* depth, float* dists, void* stream);
/* coords2rays (render_ops.py:4-25), one camera.  cam as NrPassParams.que_cam. */
int nr_coords2rays(const float* coords, const float* cam, int rn, float* centers, float* directions, void* stream);
/* depth2points (render_ops.py:27-39) */
int nr_depth2points(const float* coords, const float* cam, const float* depth, int rn, int dn, float* pts, float* dirs, void* stream);
/* depth2dists (render_ops.py:41-44) over rows of length dn */
int nr_depth2dists(const float* depth, int rows, int dn, float* dists, void* stream);
/* depth2inv_dists (render_ops.py:46-52) */
int nr_depth2inv_dists(const float* depth, const float* depth_range, int rows, int dn, float* dists, void* stream);
/* alpha_values2hit_prob (render_ops.py:72-80) */
int nr_alpha_values2hit_prob(const float* alpha, int rows, int dn, float* hit, void* stream);
/* project_points_ref_views (render_ops.py:82-130): pts [pn,3] -> dir [rfn,pn,3], pix [rfn,pn,2], depth [rfn,pn],
 * mask [rfn,pn] (1.0/0.0); valid_z (may be NULL) = project_points_coords' own validity flag. */
int nr_project_points(const float* pts, int pn, const float* view_params, int rfn, int h, int w, float* dir, float* pix,
                      float* depth, float* mask, float* valid_z, void* stream);
/* interpolate_feats (ops.py:14-34) on an NCHW map: feats [b,c,fh,fw], pts [b,n,2] -> out [b,n,c];
 * border: 1 = 'border', 0 = 'zeros'; mask (may be NULL) [b,n] multiplies the result (interpolate_feature_map). */
int nr_interpolate_feats(const float* feats, const float* pts, const float* mask, int b, int c, int fh, int fw, int n,
                         float h, float w, int border, int align_corners, float* out, void* stream);
/* Gradient of nr_interpolate_feats with respect to the map: d_feats [b,c,fh,fw] += bilinear taps * mask * d_out [b,n,c]
 * (reference: autograd through interpolate_feature_map in predict_mean_for_depth_loss, renderer.py:293, and
 * predict_self_hit_prob, renderer.py:151).  d_feats must be zero-initialised or hold a running sum. */
int nr_interpolate_feats_bwd(const float* d_out, const float* pts, const float* mask, int b, int c, int fh, int fw, int n,
                             float h, float w, int border, int align_corners, float* d_feats, void* stream);
/* sample_fine_depth (render_ops.py:172-229) followed by the caller-visible sort (renderer.py:210-213).  depth_range
 * non-NULL: inv_mode=True (resampling in normalised inverse depth, the renderer's mode); NULL: inv_mode=False. */
int nr_sample_fine_depth(const float* depth, const float* hit_prob, const float* depth_range, int rn, int dn, int fine_dn,
                         const float* u, int u_stride, int use_all, int do_sort, float* out, void* stream);

/* ---- DepthInitNet.get_diff_feats (reference network/init_net.py:29-61; SURVEY.md 8f row 2) -----------------------------
 * imgs [rfn,3,h,w], depth_in [rfn,1,h,w] (normalised inverse depth in [0,1], extract_depth_for_init), poses [rfn,3,4],
 * Ks [rfn,3,3], view_params [rfn,20] (nr_camera_blocks with the views' depth ranges) -> out [rfn,8,h,w] =
 * rgb_mean (3) | rgb_var (3) | dpt_mean | dpt_var of the reprojection differences, pooled over the views that see the pixel.
 * One fused launch: rfn^2 * h * w reprojections + gathers in registers, none of the reference's intermediates. */
int nr_diff_feats(const float* imgs, const float* depth_in, const float* poses, const float* Ks, const float* view_params,
                  int rfn, int h, int w, float* out, void* stream);

/* ---- training: backward of one pass -------------------------------------------------------------------------- */

/* Backward of nr_render_pass_fwd for the same NrPassParams (reference: loss.backward() through renderer.py:168-203;
 * SURVEY.md 8b nr_render_pass_bwd).  The call recomputes the pass in fp32, keeps every Linear layer's input on a
 * "tape" and writes every Linear layer's pre-activation gradient next to it; the caller forms the weight gradients as
 * plain GEMMs dW = dz * x^T over all rows (bias = row sums; nr_tape_gemms below does all of them in one launch).
 * Tape layout: tiles of 128 rows, slot-major inside a tile: element (slot, i) of a tape with S slots is
 * tape[((i / 128) * S + slot) * 128 + i % 128], so a tape over M rows holds S * 128 * ceil(M / 128) floats; row i of
 * the row tapes is view * (rn*dn) + point.  Slot numbers come from
 * nr_bwd_slot("R_RF"), ... (names: csrc/nr_train_math.cuh; "R_SLOTS", "G_SLOTS", "P_SLOTS", "GP_SLOTS" = sizes).
 * d_feat [rfn,fh,fw,64] must be zero-initialised (or hold a running sum): gradients of the gathered ray_feats
 * (channels 0..31) and img_feats (32..63) are atomically added to it.  Any upstream gradient may be NULL (= zero). */
typedef struct NrBwdParams {
  const float* d_pixel_colors;   /* [rn,3]  */
  const float* d_hit_prob;       /* [rn,dn] */
  const float* d_render_depth;   /* [rn]    */
  float* tape_row;               /* R_SLOTS  slots over rfn*rn*dn rows */
  float* grad_row;               /* G_SLOTS  slots over rfn*rn*dn rows */
  float* tape_point;             /* P_SLOTS  slots over rn*dn rows     */
  float* grad_point;             /* GP_SLOTS slots over rn*dn rows     */
  float* d_feat;                 /* [rfn,fh,fw,64] accumulated; NULL: feature-map gradients not wanted */
} NrBwdParams;
int nr_render_pass_bwd(const NrPassParams* p, const NrBwdParams* b, void* stream);
int nr_bwd_slot(const char* name);   /* -1: unknown name */

/* All weight gradients of a pass in one launch.  Layer i: dz = n_out slots starting at g_slot of tape g_tape, x = n_in
 * slots starting at x_slot of tape x_tape (tapes: 0 = tape_row, 1 = grad_row, 2 = tape_point, 3 = grad_point; the two
 * tapes of a layer must have the same row count).  out + out_off receives [n_out][n_in + 1], ADDED to what is there:
 * columns 0..n_in-1 = dW, column n_in = the bias gradient.  `descs` is a host array of at most 48 entries. */
typedef struct NrGemmDesc {
  int32_t g_tape, g_slot, n_out, x_tape, x_slot, n_in, out_off, reserved;
} NrGemmDesc;
int nr_tape_gemms(const NrGemmDesc* descs, int n_desc, const float* tape_row, const float* grad_row, long long rows,
                  const float* tape_point, const float* grad_point, long long points, float* out, void* stream);

/* predict_self_hit_prob (reference renderer.py:137-155, fine-tuning configs): the query view's own ray_feats sampled at
 * each ray's pixel, decoded by the pass' dist decoder, hit probability per sample (compute_prob, is_ref=False).
 * d_hit == NULL: forward only (writes hit).  Otherwise also the backward: weight gradients are ADDED to d_w_point in the
 * packed w_point layout (NrWeightLayout), the map gradient to d_map (may be NULL). */
typedef struct NrSelfParams {
  const float* map;          /* [32,fh,fw] query ray_feats */
  const float* coords;       /* [rn,2] */
  const float* que_depth;    /* [rn,dn] */
  const float* w_point;
  int32_t rn, dn, h, w, fh, fw, use_vis;
  const float* depth_range;  /* device [2]: near, far of the query view */
  float var_bias;
  float* hit;                /* [rn,dn] */
  const float* d_hit;        /* [rn,dn] or NULL */
  float* d_w_point;          /* [NrWeightLayout.total_point] accumulated */
  float* d_map;              /* [32,fh,fw] accumulated, or NULL */
} NrSelfParams;
int nr_self_hit_prob(const NrSelfParams* p, void* stream);

/* ---- encoders upstream of the ray path (SURVEY.md 8(f) row f1) ------------------------------------------------
 * image_encoder = ResUNetLight(3, [1,2,6,4], 32, inplanes=16)  (reference network/ops.py:150-230, built at renderer.py:59,
 * called at renderer.py:229,233) and vis_encoder = DefaultVisEncoder (network/vis_encoder.py:6-21, called at
 * renderer.py:231,234), forward only (inference; training keeps the torch modules upstream of the boundary).
 * Everything runs channel-last; the last layer of each encoder writes straight into the [rfn,fh,fw,64] frame pack of
 * NrPassParams.feat (ray_feats in channels 0..31, img_feats in 32..63), so a frame needs no NCHW->NHWC repack.
 *
 * Parameters: `params` is a HOST array of DEVICE pointers to the module's tensors in state_dict() order (conv weights
 * [cout][cin][kh][kw], InstanceNorm weight / bias, conv bias; image encoder: 84 tensors, vis encoder: 14).  nr_*_pack
 * re-lays them once per checkpoint into one flat buffer (conv weights as [tap][cin][cout]). */
typedef struct NrEncoderLayout {
  int32_t image_tensors, vis_tensors;
  int64_t image_packed_floats, vis_packed_floats;
  int32_t depth_init_tensors, reserved;
  int64_t depth_init_packed_floats;
} NrEncoderLayout;
int nr_encoder_layout(NrEncoderLayout* out);
int nr_image_encoder_pack(const float* const* params, int n_params, float* packed, void* stream);
int nr_vis_encoder_pack(const float* const* params, int n_params, float* packed, void* stream);
/* output map size for h x w images (h/4 x w/4 when h, w are multiples of 16; the decoder's skip connections pad otherwise,
 * ops.py:199-208) */
int nr_image_encoder_dims(int h, int w, int* fh, int* fw);
long long nr_image_encoder_workspace(int n, int h, int w);     /* bytes */
long long nr_vis_encoder_workspace(int n, int fh, int fw);     /* bytes */
/* imgs [n,3,h,w] (NCHW as the reference holds them) -> out[(view, y, x) * out_stride + out_off + c], c < 32.
 * tf32x1: 0 = 3xTF32 tensor-core products (fp32 accuracy: parity with the fp32 reference, the default of the Python layer);
 * 1 = one TF32 pass per product, i.e. what the reference computes on a GPU under torch's default
 * torch.backends.cudnn.allow_tf32 = True (~1e-3 relative). */
int nr_image_encoder_fwd(const float* packed, const float* imgs, int n, int h, int w, float* out, int out_stride, int out_off,
                         int tf32x1, void* workspace, long long workspace_bytes, void* stream);
/* feat [n,fh,fw,64]: channels 0..31 = the init net's ray_feats, 32..63 = img_feats; channels 0..31 are overwritten with
 * vis_encoder(ray_feats, img_feats). */
int nr_vis_encoder_fwd(const float* packed, float* feat, int n, int fh, int fw, int tf32x1, void* workspace, long long workspace_bytes,
                       void* stream);

/* DepthInitNet (reference network/init_net.py:63-101; the init net of the neuray_gen_depth model), forward only:
 *   nr_extract_depth  extract_depth_for_init_impl (:63-74): metric depth [n,1,h,w] + depth_range [n,2] -> normalised inverse depth
 *   nr_diff_feats     get_diff_feats (:29-61), declared above
 *   nr_depth_init_fwd res_net = ResEncoder (ops.py:232-312) on cat([imgs, depth, diff_feats]), depth_skip, conv_out (:93-101)
 * `params`: the module's 72 tensors in state_dict() order (res_net.*, depth_skip.*, conv_out.*).  The 32 output channels go to
 * out[(view, y, x) * out_stride + out_off + c] at nr_depth_init_dims (h/4 x w/4 for multiples of 16), e.g. straight into
 * channels 0..31 of the frame pack, where nr_vis_encoder_fwd expects the init net's ray_feats. */
int nr_extract_depth(const float* depth, const float* depth_range, int n, int h, int w, float* out, void* stream);
int nr_depth_init_dims(int h, int w, int* fh, int* fw);
long long nr_depth_init_workspace(int n, int h, int w);        /* bytes */
int nr_depth_init_pack(const float* const* params, int n_params, float* packed, void* stream);
int nr_depth_init_fwd(const float* packed, const float* imgs, const float* depth_norm, const float* diff_feats, int n, int h, int w,
                      float* out, int out_stride, int out_off, int tf32x1, void* workspace, long long workspace_bytes, void* stream);

/* ---- CostVolumeInitNet (SURVEY.md 8(f) row f4; reference network/init_net.py:113-254) ----------------------------------
 * nr_mvsnet_*: the frozen MVSNet (network/mvsnet/mvsnet.py: FeatureNet, homography cost volume, CostRegNet) behind
 * construct_cost_volume_with_src (init_net.py:113-160), inference.  `params`: the 89 tensors of MVSNet.state_dict() without
 * num_batches_tracked, in order: per layer the conv weight, then the norm's weight, bias, running_mean, running_var (or the
 * conv bias for feature.feature / cost_regularization.prob); BatchNorm is folded at pack time.  Outputs, channel-last:
 * prob [rfn,ho,wo,dn] = softmax over the depth planes of the regularised cost volume (what volume_conv2d consumes) and
 * depth [rfn,ho,wo] = the regressed metric depth, ho x wo from nr_mvsnet_dims (h/4 x w/4; evaluation at 800x800 / 768x1024
 * runs the network at 640x640 / 576x768 and resizes the cost volume back, init_net.py:120-139,155). */
typedef struct NrMvsIn {
  const float* ref_imgs; const float* src_imgs;   /* [rfn,3,h,w], [sn,3,h,w], values in 0..1 */
  const float* ref_Ks; const float* ref_poses;    /* [rfn,3,3], [rfn,3,4] */
  const float* src_Ks; const float* src_poses;    /* [sn,3,3], [sn,3,4] */
  const float* depth_range;                       /* [rfn,2] */
  const int32_t* nn_ids;                          /* [rfn,nn]: the source views of each reference view */
  int32_t rfn, sn, nn, h, w, dn, is_train;
} NrMvsIn;
int nr_mvsnet_layout(int* n_tensors, long long* packed_floats);
int nr_mvsnet_pack(const float* const* params, int n_params, float* packed, void* stream);
int nr_mvsnet_dims(int h, int w, int is_train, int* ho, int* wo);
long long nr_mvsnet_workspace(const NrMvsIn* in);   /* bytes; 0: unsupported shape */
int nr_mvsnet_fwd(const float* packed, const NrMvsIn* in, float* prob, float* depth, void* workspace, long long workspace_bytes, void* stream);

/* nr_cost_volume_head_*: CostVolumeInitNet.forward after construct_cost_volume_with_src (init_net.py:247-254): res_net =
 * ResUNetLight(out_dim=32) on the images, volume_conv2d on the softmaxed cost volume, depth_conv on the normalised regressed
 * depth (nr_extract_depth of nr_mvsnet_fwd's depth), out_conv on their concatenation -> 32 channels into an output slot
 * (e.g. channels 0..31 of the frame pack).  `params`: the module's tensors after `mvsnet.*` in state_dict() order (res_net.*,
 * volume_conv2d.*, depth_conv.*, out_conv.*: 120 tensors).  prob / depth_norm: [n,h/4,w/4,cost_volume_sn] / [n,h/4,w/4]. */
int nr_cost_volume_head_layout(int cost_volume_sn, int* n_tensors, long long* packed_floats);
int nr_cost_volume_head_pack(int cost_volume_sn, const float* const* params, int n_params, float* packed, void* stream);
long long nr_cost_volume_head_workspace(int cost_volume_sn, int n, int h, int w);
int nr_cost_volume_head_fwd(int cost_volume_sn, const float* packed, const float* imgs, const float* prob, const float* depth_norm, int n, int h, int w,
                            float* out, int out_stride, int out_off, int tf32x1, void* workspace, long long workspace_bytes, void* stream);

/* Building blocks (channel-last).  nr_conv2d_nhwc: k x k convolution (k <= 8), stride 1 / 2, reflect or zero padding of
 * `pad` (-1: (ks-1)/2), cout in {32, 64, 128}, cin a multiple of 16, as an implicit GEMM on the tensor cores (3xTF32: fp32 accuracy);
 * y = conv(x) [+ bias] [+ res]; when `stats` is given, sum and sum of squares of y per (image, channel) are ADDED to
 * stats [n][cout][2] (fp64) for a following nr_instance_norm_act.  Pixel (i, y, x) channel c of a tensor sits at
 * base[((i*H + y)*W + x) * stride + off + c]. */
typedef struct NrConv2d {
  const float* x; const float* w_packed; const float* bias; const float* res;
  float* y; double* stats;
  int32_t n, h, w, cin, cout, ks, stride, reflect;
  int32_t x_stride, x_off, y_stride, y_off, res_stride, res_off;
  int32_t tf32x1;            /* 0: 3xTF32 (fp32 accuracy); 1: one TF32 pass */
  int32_t pad;               /* -1: (ks-1)/2 */
  int32_t bm;                /* output pixels per CTA: 0 = chosen by the library, else 64 / 128 (cout 64, 128) or 128 / 256 (cout 32) */
} NrConv2d;
int nr_conv2d_nhwc(const NrConv2d* c, void* stream);
/* [cout][cin][ks][ks] -> [tap][cin][cout]; packed input channel c reads reference channel (c + cin_rot) % cin */
int nr_conv_pack_weight(const float* w, int cout, int cin, int ks, int cin_rot, float* packed, void* stream);
/* y = act(IN(x) * gamma + beta [+ res | + IN(res) * res_gamma + res_beta]) on dense [n,hw,c] tensors; act 0 none, 1 ReLU,
 * 2 ELU; statistics from nr_conv2d_nhwc (biased variance, eps 1e-5 = nn.InstanceNorm2d). */
int nr_instance_norm_act(const float* x, const double* stats, const float* gamma, const float* beta, const float* res,
                         const double* res_stats, const float* res_gamma, const float* res_beta, int n, int hw, int c, int act, float* y,
                         void* stream);
int nr_nchw_to_nhwc(const float* x, int n, int c, int h, int w, float* y, int y_stride, int y_off, void* stream);
int nr_nhwc_to_nchw(const float* x, int n, int c, int h, int w, int x_stride, int x_off, float* y, void* stream);

/* ---- training extras next to the ray path (SURVEY.md 8(f) row f3) ------------------------------------------------ */

/* NeuralRayGenRenderer.predict_mean_for_depth_loss (reference renderer.py:280-316): per reference view, the view's
 * ray_feats sampled at `coords` (interpolate_feature_map, border clamp) and decoded by the MEAN head of the coarse
 * (index 0) and, optionally, the fine (index 1) dist decoder.  d_mean[k] == NULL: forward only (writes mean[k]);
 * otherwise also the backward of decoder k: weight gradients are ADDED to d_w_point[k] (packed w_point layout), the map
 * gradient to d_map (may be NULL). */
typedef struct NrDepthMeanParams {
  const float* map;            /* [rfn,32,fh,fw] ray_feats */
  const float* coords;         /* [rfn,pn,2], pixels of the h x w reference images, in the order the reference passes them */
  const float* w_point[2];     /* packed weights of the coarse / fine pass (fine may be NULL) */
  int32_t rfn, pn, h, w, fh, fw;
  float* mean[2];              /* [rfn,pn,2] softplus outputs (depth_mean = [...,0], depth_mean_2 = [...,1]) */
  const float* d_mean[2];      /* [rfn,pn,2] or NULL */
  float* d_w_point[2];         /* [NrWeightLayout.total_point] accumulated */
  float* d_map;                /* [rfn,32,fh,fw] accumulated, or NULL */
} NrDepthMeanParams;
int nr_depth_mean(const NrDepthMeanParams* p, void* stream);

/* RenderLoss (reference network/loss.py:46-76): loss[q] = sum_r mask * |pr - gt|^2 / (sum_r mask + 1e-3), or the plain mean
 * over rays when ray_mask == NULL.  g == NULL: forward (writes loss [qn]); otherwise the backward: d_pr [qn,rn,3] =
 * g[q] * d loss[q] / d pr. */
int nr_render_loss(const float* pr, const float* gt, const uint8_t* ray_mask, int qn, int rn, float* loss, const float* g, float* d_pr,
                   void* stream);

/* DepthLoss (reference network/loss.py:78-132): the decoder means against the ground-truth depth maps sampled at the same
 * coordinates, both in normalised inverse depth; loss_type 0 = l2, 1 = smooth_l1(beta); aug_depth != NULL = the 'gso'
 * branch (mean over the coordinates whose augmented depth agrees with the true depth within correct_thresh).
 * g == NULL: forward (loss [rfn]); otherwise d_depth_pr [rfn,pn] = g[view] * d loss / d depth_pr. */
typedef struct NrDepthLossParams {
  const float* depth_pr;       /* [rfn,pn] */
  const float* coords;         /* [rfn,pn,2] */
  const float* true_depth;     /* [rfn,h,w] */
  const float* aug_depth;      /* [rfn,h,w] or NULL */
  const float* depth_range;    /* [rfn,2] */
  int32_t rfn, pn, h, w, loss_type;
  float beta, correct_thresh;
  float* loss;                 /* [rfn] */
  const float* g;              /* [rfn] or NULL */
  float* d_depth_pr;           /* [rfn,pn] */
} NrDepthLossParams;
int nr_depth_loss(const NrDepthLossParams* p, void* stream);

/* ConsistencyLoss (reference network/loss.py:17-44): loss[q] = mean over rays and samples of the cross entropy between
 * prob0 (the rendered hit probability, a constant) and prob1 (hit_prob_self).  g == NULL: forward; otherwise d_prob1. */
int nr_consistency_loss(const float* prob0, const float* prob1, int qn, int rn, int dn, float* loss, const float* g, float* d_prob1,
                        void* stream);

/* ---- validation metrics ---------------------------------------------------------------------------------------- */

#define NR_METRICS_MAX_PRED 8   /* predictions scored per nr_image_metrics call */

/* PSNR_SSIM (reference network/metrics.py:13-79): the ground truth `gt` against each of `preds[0..n_pred)` (a HOST array of
 * device pointers), all [h,w,3] fp32 in raster order.  Each image is quantised like color_map_backward (x*255 in fp32,
 * clipped to [0,255], truncated) and cropped by margin_h rows top and bottom and margin_w columns left and right.
 * out[n][4] (fp64) = the three per-channel sums of squared errors over the crop (exact integers) and the SSIM of
 * skimage's structural_similarity(win_size=11, data_range=255): uniform 11x11 windows, sample covariance, the map less 5
 * pixels on every side averaged per channel, then over the channels.  PSNR = 10 log10(255^2 / mse) with mse the mean of
 * the three sse / ((h - 2 margin_h) (w - 2 margin_w)).  The result is the same bit for bit from run to run.  A crop
 * smaller than 11 x 11 is NR_E_INVALID. */
long long nr_image_metrics_workspace(int n_pred, int h, int w, int margin_h, int margin_w);   /* bytes */
int nr_image_metrics(const float* gt, const float* const* preds, int n_pred, int h, int w, int margin_h, int margin_w, double* out,
                     void* workspace, long long workspace_bytes, void* stream);

/* Scores of the reference's eval.py for n pairs of uint8 [h,w,3] images in raster order, gt[n,h,w,3] against pr[n,h,w,3]
 * (device pointers).  Each value is converted like color_map_forward, float(v) / 255 in fp32.
 *
 * nr_eval_metrics: out[n][2] (fp64) = tf.image.psnr(max_val 1) and tf.image.ssim(max_val 1, filter 11, sigma 1.5, k1 0.01,
 * k2 0.03) of each pair, evaluated in fp64: PSNR = 10 log10(1 / mse) with mse over h*w*3 (inf for identical images); SSIM =
 * the mean over the VALID (h-10) x (w-10) region and the channels of luminance * cs, from Gaussian-weighted means (window
 * g (x) g, population covariance).  The result is the same bit for bit from run to run and for any n.  Images smaller than
 * 11 x 11 are NR_E_INVALID. */
long long nr_eval_metrics_workspace(int n, int h, int w);   /* bytes */
int nr_eval_metrics(const uint8_t* gt, const uint8_t* pr, int n, int h, int w, double* out, void* workspace, long long workspace_bytes,
                    void* stream);

/* LPIPS-VGG (lpips.LPIPS(net='vgg'), version 0.1, called as eval.py calls it on x * 2 - 1): the scaling layer, torchvision's
 * vgg16.features[0:30] with taps after relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3, per tap each image's features divided
 * by (their channel norm + 1e-10), the squared difference, the 1x1 lin weights and the spatial mean; out[n] (fp64) = the sum
 * over the taps.  `params`: 31 tensors, features.{0,2,5,7,10,12,14,17,19,21,24,26,28}.weight and .bias in that order, then
 * lin0..lin4.model.1.weight.  tf32x1 as for the encoders (0: 3xTF32, 1: one TF32 pass, what cuDNN runs under torch's
 * default allow_tf32).  Images must be at least 32 x 32: a limit of this library, not of lpips (which takes 16 x 16), because
 * nr_conv2d_nhwc needs conv5's input, h/16 x w/16, to be at least 2 x 2.  LPIPS of identical images is exactly 0.  The workspace
 * grows with n (two [2n,h,w,64] fp32 buffers). */
int nr_lpips_vgg_layout(int* n_tensors, long long* packed_floats);
int nr_lpips_vgg_pack(const float* const* params, int n_params, float* packed, void* stream);
long long nr_lpips_vgg_workspace(int n, int h, int w);   /* bytes */
int nr_lpips_vgg_fwd(const float* packed, const uint8_t* gt, const uint8_t* pr, int n, int h, int w, double* out, int tf32x1,
                     void* workspace, long long workspace_bytes, void* stream);

/* ---- diagnostics ------------------------------------------------------------------------------------------- */

/* Self-test of the wgmma layer primitive the point kernel uses: D[128,n] = A[128,k] * W[n,k]^T with A in the shared-memory
 * activation tile and W in swizzled shared memory; mode 0 = one TF32 pass, 1 = 3xTF32 (fp32-accurate), 2 = 3xTF32 with A
 * from registers (n 16 or 32).  (n,k) in {(32,32),(64,64),(16,64)}. */
int nr_tc_selftest(const float* A, const float* W, float* D, int n, int k, int mode, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEURAY_B200_H */

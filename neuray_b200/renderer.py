"""Host side of the per-ray rendering path: the reference's NeuralRayBaseRenderer API over the fused CUDA kernels.

Mirrors reference network/renderer.py:24-254 for the hot path (SURVEY.md section 8a rows a8-a16):

    render_by_depth   :168-203      one point-kernel + one ray-kernel launch (nr_render_pass_fwd)
    fine_render_impl  :205-215      the resampling is fused into the coarse pass' ray kernel
    render_impl       :217-226
    render            :228-254      chunk loop; per-frame NCHW -> channel-last repack hoisted out of it

Two ways to use it:
  * `NeuralRayRenderPath` -- a self-contained nn.Module holding the hot path's parameters under the reference's
    state-dict names (loads a reference checkpoint with strict=False); `render()` takes encoder outputs.
  * `neuray_b200.patch.install()` -- rebinds the same functions onto the reference's own NeuralRayBaseRenderer so
    render.py / run_training.py run unchanged.

The functions below are written against "owner": any nn.Module that has `.cfg` (reference base_cfg keys) and the
sub-modules dist_decoder / agg_net (/ fine_dist_decoder / fine_agg_net) with the reference's parameter names.
"""
import ctypes as C
from dataclasses import dataclass
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib, encoders, init_nets, modules
from .render_ops import fine_sample_u, interpolate_feats, sample_depth
from .weights import camera_blocks, pack_pass, pack_pass_tf32, point_index_map, posenc_table

PACK_KEY = "_nr_frame_pack"        # ref_imgs_info: the FramePack of the frame being rendered (lives for one render() call)
CAM_KEY = "_nr_que_cam"            # que_imgs_info: que_cam block of the frame being rendered (same lifetime)

base_cfg = {
    "vis_encoder_type": "default", "vis_encoder_cfg": {},
    "dist_decoder_type": "mixture_logistics", "dist_decoder_cfg": {},
    "agg_net_type": "default", "agg_net_cfg": {},
    "use_hierarchical_sampling": False, "fine_agg_net_cfg": {}, "fine_dist_decoder_cfg": {},
    "fine_depth_sample_num": 64, "fine_depth_use_all": False,
    "ray_batch_num": 2048, "depth_sample_num": 64, "alpha_value_ground_state": -15,
    "use_dr_prediction": False, "use_nr_color_for_dr": False, "use_self_hit_prob": False,
    "use_ray_mask": True, "ray_mask_view_num": 2, "ray_mask_point_num": 8,
    "render_depth": False,
    # each pass' visibility_nr [1,rn,rfn]: every pixel's visibility from each working view (nr_view_visibility)
    "render_visibility": False,
    # each pass' blend_weights_nr [1,rn,rfn]: every pixel's colour-blend weight per working view (nr_render_pass_fwd_blend)
    "render_blend_weights": False,
    # each pass' neuray_weights_nr and geometry_weights_nr [1,rn,rfn]: every pixel's weight per working view in the
    # aggregation net's two view poolings, weight0 and the vis weight (nr_render_pass_fwd_agg)
    "render_agg_weights": False,
    # each pass' view_hit_nr and view_depth_nr [1,rn,rfn]: Σ_d of every working view's masked hit probability along the
    # pixel's ray, alone and times the sample depth; view_depth_nr / view_hit_nr is where the view puts the surface
    # (nr_render_pass_fwd_view)
    "render_view_depth": False,
    # each pass' view_colors_nr [1,rn,rfn,3]: the colour every working view puts into the pixel, Σ_d hit_prob · blend
    # weight · the view's colour; Σ_v view_colors_nr = pixel_colors_nr (nr_view_colors)
    "render_view_colors": False,
    # NeuralRayGenRenderer.default_cfg (renderer.py:256-261), read by predict_mean_for_depth_loss
    "use_depth_loss": False, "depth_loss_coords_num": 8192,
}


# Arithmetic of the point kernel's tensor-core layers in render passes that record no gradient.
# "fp32": 3xTF32, fp32 accuracy (the default).  "tf32": one TF32 pass per product on operands rounded to nearest, what
# torch 1.7 to 1.11 ran nn.Linear in on Ampere and later GPUs by default (the reference pins torch 1.7.1); about 1e-3
# relative per layer.  The ray kernel and the encoders (encoders.set_precision) do not depend on it.
PRECISION = "fp32"


def set_precision(mode):
    """Selects the render passes' point-kernel arithmetic: "fp32" (3xTF32) or "tf32" (one TF32 pass per product).

    A pass that records a gradient (autograd on, and a parameter or the feature maps require grad) always runs in fp32:
    nr_render_pass_bwd recomputes the forward in fp32, so a TF32 forward would return values of a different function
    than the one its gradients belong to.  Under torch.no_grad() (inference, the validation loop of run_training.py)
    "tf32" applies to every pass, whichever entry point reaches it."""
    global PRECISION
    if mode not in ("fp32", "tf32"):
        raise ValueError(f"render precision {mode!r}: 'fp32' or 'tf32'")
    PRECISION = mode


_PACK_POOL = {}      # (device, feat shape, rgb shape) -> [(feat, rgb)] of dropped FramePacks, at most two kept


_PACK_SOURCES = ("ray_feats", "img_feats", "imgs", "poses", "Ks", "depth_range")


class FramePack:
    """Per-frame device data shared by every chunk and both passes: channel-last maps + per-view parameters.

    A pack keeps strong references to the tensors it was built from and is valid only for exactly those tensor objects
    at exactly those versions (`matches`): a fresh encoder output that happens to get a recycled address is a different
    object, and an in-place edit bumps `_version`."""

    def __del__(self):
        try:
            pool = _PACK_POOL.setdefault(self._pool_key, [])
            if len(pool) < 2:
                pool.append((self.feat, self.rgb))
        except Exception:      # interpreter shutdown
            pass

    def __init__(self, ref_imgs_info, encoder_owner=None):
        """encoder_owner: a module with image_encoder / vis_encoder (reference parameter names).  The pack then takes the INIT
        net's ray_feats from ref_imgs_info, runs both encoders natively into the channel-last buffer (encoders.encode_frame,
        reference renderer.py:229-231) and leaves their NCHW results in ref_imgs_info['img_feats'] / ['ray_feats']."""
        imgs = ref_imgs_info["imgs"]
        if not imgs.is_cuda:
            raise _lib.NeurayB200Error("the rendering path needs CUDA tensors (no CPU fallback)")
        rfn, _, h, w = imgs.shape
        rf = ref_imgs_info.get("ray_feats")
        if encoder_owner is not None:
            fh, fw = encoders.image_dims(h, w)
            if rf is None:       # the owner's init net writes its ray_feats straight into the pack (encoders.encode_frame)
                if not hasattr(encoder_owner.init_net, "mvsnet") and init_nets.dims(h, w) != (fh, fw):
                    raise _lib.NeurayB200Error(f"init net and image encoder disagree on the map size for {h}x{w} images")
            elif tuple(rf.shape[-2:]) != (fh, fw) or rf.shape[1] != 32:
                raise _lib.NeurayB200Error(f"ray_feats {tuple(rf.shape)} do not match the image encoder's output size {(fh, fw)} for {h}x{w} images")
        else:
            imf = ref_imgs_info.get("img_feats")
            if rf is None or imf is None:
                raise _lib.NeurayB200Error("ref_imgs_info needs the encoder outputs 'ray_feats' and 'img_feats' [rfn,32,fh,fw] "
                                           "(or render through an owner with native encoders: NeuralRayFrameRenderer)")
            if rf.shape != imf.shape or rf.shape[1] != 32:
                raise _lib.NeurayB200Error(f"ray_feats {tuple(rf.shape)} and img_feats {tuple(imf.shape)} must both be [rfn,32,fh,fw]")
            fh, fw = rf.shape[-2:]
        if rfn > _lib.NR_MAX_VIEWS:
            raise _lib.NeurayB200Error(f"at most {_lib.NR_MAX_VIEWS} reference views per call, got {rfn}")
        dev = imgs.device
        self.rfn, self.h, self.w, self.fh, self.fw = rfn, h, w, fh, fw
        self._pool_key = (str(dev), (rfn, fh, fw, 64), (rfn, h, w, 4))
        spare = _PACK_POOL.get(self._pool_key)
        if spare:
            self.feat, self.rgb = spare.pop()
        else:
            self.feat = torch.empty(rfn, fh, fw, 64, dtype=torch.float32, device=dev)
            self.rgb = torch.empty(rfn, h, w, 4, dtype=torch.float32, device=dev)
        if encoder_owner is not None:
            encoders.encode_frame(encoder_owner, ref_imgs_info, self.feat)
            with _lib.on_device(imgs):
                _lib.check(_lib.lib().nr_pack_feature_maps(None, None, _lib.ptr(imgs.detach().contiguous().float()), rfn, h, w, fh, fw,
                                                           None, _lib.ptr(self.rgb), _lib.stream_of(imgs)), "nr_pack_feature_maps (rgb)")
            _lib.count_launches(1)
        else:
            with _lib.on_device(imgs):
                _lib.check(_lib.lib().nr_pack_feature_maps(
                    _lib.ptr(rf.detach().contiguous().float()), _lib.ptr(imf.detach().contiguous().float()),
                    _lib.ptr(imgs.detach().contiguous().float()), rfn, h, w, fh, fw, _lib.ptr(self.feat), _lib.ptr(self.rgb),
                    _lib.stream_of(imgs)), "nr_pack_feature_maps")
            _lib.count_launches(2)
        _, self.view_params = camera_blocks(None, ref_imgs_info)
        self.src = tuple((ref_imgs_info[k], ref_imgs_info[k]._version) for k in _PACK_SOURCES)

    def matches(self, ref_imgs_info):
        return all(ref_imgs_info.get(k) is t and t._version == ver for k, (t, ver) in zip(_PACK_SOURCES, self.src))


def frame_pack(ref_imgs_info):
    """The pack of the frame in flight (installed by render_chunks for the duration of one render() call), or a fresh one
    for a direct render_by_depth / render_impl call.  A fresh pack is NOT left in the caller's dict."""
    pack = ref_imgs_info.get(PACK_KEY)
    if pack is None or not pack.matches(ref_imgs_info):
        pack = FramePack(ref_imgs_info)
    return pack


class PassParams(NamedTuple):
    """One pass' modules, their state-dict prefixes and its parameters as [(state-dict name, tensor)]: the decoder's
    named_parameters(), then the aggregation net's.  backward.RenderPassFn and backward.layer_table read the gradients
    by these names in this order."""
    is_fine: bool
    dec: nn.Module
    agg: nn.Module
    dec_name: str
    agg_name: str
    named: list


def pass_params(owner, is_fine):
    dec_name, agg_name = ("fine_dist_decoder", "fine_agg_net") if is_fine else ("dist_decoder", "agg_net")
    dec, agg = getattr(owner, dec_name), getattr(owner, agg_name)
    named = [(f"{dec_name}.{k}", v) for k, v in dec.named_parameters()] + [(f"{agg_name}.{k}", v) for k, v in agg.named_parameters()]
    return PassParams(is_fine, dec, agg, dec_name, agg_name, named)


@dataclass
class _PackedPass:
    """The owner's cache entry of one pass' packed weights."""
    stamp: tuple            # (data_ptr, _version) of every parameter, then the device packed for
    w_point: torch.Tensor   # nr_pack_weights' buffers: fresh on every re-pack
    w_ray: torch.Tensor
    w_tc: torch.Tensor
    pos_enc: dict           # dn -> posenc table on the device; kept across re-packs
    w_tc_tf32: torch.Tensor = None      # nr_pack_weights_tf32's w_tc, made on first use after each re-pack


def pass_weights(owner, is_fine, dn, device, tf32=False):
    """(w_point, w_ray, pos_enc, w_tc) of one pass (nr_pack_weights), cached on the owner and re-packed when any parameter
    changed (optimizer steps bump tensor._version).  Every re-pack gets fresh buffers: an autograd graph recorded before
    the parameter update keeps reading the buffers it was recorded with.  tf32: w_tc is the TF32 mode's pack
    (nr_pack_weights_tf32), made on first use after each re-pack and cached next to the other one."""
    pp = pass_params(owner, is_fine)
    params = dict(pp.named)
    stamp = tuple((v.data_ptr(), v._version) for v in params.values()) + (str(device),)
    cache = owner.__dict__.setdefault("_nr_wcache", {})
    entry = cache.get(is_fine)
    if entry is None or entry.stamp != stamp:
        first = pp.named[0][1]
        if first.device != torch.device(device):
            raise _lib.NeurayB200Error(f"parameters live on {first.device} but the rays are on {device}")
        w_point, w_ray, w_tc = pack_pass(params, pp.dec_name, pp.agg_name)
        pos_enc = entry.pos_enc if entry is not None else {}
        entry = cache[is_fine] = _PackedPass(stamp, w_point, w_ray, w_tc, pos_enc)
    pe = entry.pos_enc.get(dn)
    if pe is None:
        n_samples = pp.agg.agg_impl.n_samples
        if n_samples != dn:
            # the reference fails with a broadcast error here (ibrnet.py:356); keep that behaviour explicit
            raise _lib.NeurayB200Error(
                f"{pp.agg_name}: pos_encoding was built for sample_num={n_samples} but the pass has {dn} samples per ray")
        pe = entry.pos_enc[dn] = posenc_table(dn).to(device).contiguous()
    if tf32 and entry.w_tc_tf32 is None:
        entry.w_tc_tf32 = pack_pass_tf32(params, pp.dec_name, pp.agg_name)
    return entry.w_point, entry.w_ray, pe, entry.w_tc_tf32 if tf32 else entry.w_tc


def pass_index_map(owner, pp, dev):
    """weights.point_index_map of the pass pp (packed w_point position -> parameter element), cached on the owner."""
    maps = owner.__dict__.setdefault("_nr_index_maps", {})
    key = (pp.is_fine, str(dev), tuple(n for n, _ in pp.named))
    if key not in maps:
        maps[key] = point_index_map(dict(pp.named), pp.dec_name, pp.agg_name)
    return maps[key]


# SphericalHarmonicsSolver(3).regs (reference sph_solver.py:6-12): the diagonal added to the SH fit's normal matrix
_SH_REGS = (0.0,) + (0.001,) * 3 + (0.005,) * 5 + (0.05,) * 7


def _sh_regs(owner):
    """The owner's sph_fitter.regs (read once per buffer version), or the solver's constructor defaults."""
    fitter = getattr(owner, "sph_fitter", None)
    if fitter is None:
        return _SH_REGS
    regs = fitter.regs
    stamp = (regs.data_ptr(), regs._version)
    hit = owner.__dict__.get("_nr_sh_regs")
    if hit is None or hit[0] != stamp:
        if regs.numel() != len(_SH_REGS):
            raise _lib.NeurayB200Error(f"sph_fitter.regs has {regs.numel()} entries: direct rendering fits degree 3 (16)")
        hit = (stamp, tuple(float(x) for x in regs.detach().float().cpu()))
        owner.__dict__["_nr_sh_regs"] = hit
    return hit[1]


def _direct_render(owner, launch, rn, dn, dev):
    """use_dr_prediction (reference renderer.py:85-125, 181-185): nr_direct_render enqueued right behind the pass `launch`
    describes, while that pass' point record is still in the shared workspace.  Returns pixel_colors_dr [1,rn,3] and
    hit_prob_dr [1,rn,dn]."""
    res = {"pixel_colors_dr": torch.empty(1, rn, 3, dtype=torch.float32, device=dev),
           "hit_prob_dr": torch.empty(1, rn, dn, dtype=torch.float32, device=dev)}
    if launch is None:          # rn == 0: nothing was launched
        return res
    d = _lib.NrDrParams()
    d.regs[:] = _sh_regs(owner)
    d.alpha_ground_state = float(owner.cfg["alpha_value_ground_state"])
    d.use_nr_color = 1 if owner.cfg["use_nr_color_for_dr"] else 0
    d.point_colors = _lib.ptr(_lib.workspace("dr_point_colors", rn * dn * 3, dev))
    d.pixel_colors_dr, d.hit_prob_dr = _lib.ptr(res["pixel_colors_dr"]), _lib.ptr(res["hit_prob_dr"])
    with _lib.on_device(res["hit_prob_dr"]):
        _lib.check(_lib.lib().nr_direct_render(C.byref(launch.params), C.byref(d), launch.stream), "nr_direct_render")
    _lib.count_launches(2)
    return res


def _view_visibility(launch, hit_prob, rn, rfn, dev):
    """render_visibility: nr_view_visibility enqueued right behind the pass `launch` describes, on its hit_prob.  Returns
    visibility [1,rn,rfn]: Σ_d hit_prob · the masked prj_dict['vis'] of each view (renderer.py:79-82)."""
    vis = torch.empty(1, rn, rfn, dtype=torch.float32, device=dev)
    if launch is None:          # rn == 0: nothing was launched
        return vis
    q = _lib.NrVisParams()
    q.hit_prob, q.visibility = _lib.ptr(hit_prob), _lib.ptr(vis)
    with _lib.on_device(vis):
        _lib.check(_lib.lib().nr_view_visibility(C.byref(launch.params), C.byref(q), launch.stream), "nr_view_visibility")
    _lib.count_launches(1)
    return vis


class PassLaunch(NamedTuple):
    """A launched pass, for what runs on the same inputs after it: direct rendering, visibility and nr_render_pass_bwd
    (the autograd node keeps it alive; otherwise it is dropped with the pass' outputs)."""
    params: _lib.NrPassParams
    keep: tuple             # the tensors params points into
    feat_shape: tuple       # [rfn,fh,fw,64] of the channel-last feature-map gradient
    stream: int


def _launch_pass(owner, que_depth, que_imgs_info, ref_imgs_info, pp, fine, want_hit, tf32, blend=False, agg=False, view=False,
                 colors=False):
    """Enqueues the two kernels of the pass pp; returns its raw outputs (ray_mask as uint8) and its PassLaunch, None when
    there are no rays.  tf32: the point kernel in TF32 mode (set_precision).  blend: the point kernel also exports its
    colour-blend weights and a reduction forms blend_weights [1,rn,rfn] (nr_render_pass_fwd_blend, _tf32_blend): Σ_d
    hit_prob · the reference's blending_weights_valid (ibrnet.py:362-366) of each view.  agg: the point kernel also
    exports its two pooling weights and reductions form neuray_weights and geometry_weights [1,rn,rfn]
    (nr_render_pass_fwd_agg, _tf32_agg): Σ_d hit_prob · the reference's weight0 (ibrnet.py:334-337) and weight
    (ibrnet.py:349-350) of each view; with blend as well, the same launch forms blend_weights.  view: the point kernel
    also exports each view's masked hit probability hit_v (the reference's prj_dict['hit_prob'], renderer.py:75-82) and
    reductions form view_hit = Σ_d hit_v and view_depth = Σ_d hit_v · que_depth [1,rn,rfn] (nr_render_pass_fwd_view,
    _tf32_view); the same launch forms whichever of the blend and agg outputs are asked for.  colors: nr_view_colors runs
    behind whichever of those launches runs (nr_render_pass_fwd_blend without its reduction when none is asked for), on
    its blend row and hit_prob, and forms view_colors [1,rn,rfn,3] = Σ_d hit_prob · blending_weights_valid · the masked
    prj_dict['rgb'] (ibrnet.py:366-367, render_ops.py:132-139) of each view."""
    cfg = owner.cfg
    coords = que_imgs_info["coords"]
    dev = coords.device
    pack = frame_pack(ref_imgs_info)
    _, rn, dn = que_depth.shape
    dec = pp.dec
    w_point, w_ray, pos_enc, w_tc = pass_weights(owner, pp.is_fine, dn, dev, tf32)
    cam = que_imgs_info.get(CAM_KEY)
    if cam is None:
        cam, _ = camera_blocks(que_imgs_info, None)
    coords_c = coords[0].detach().contiguous().float()

    out = {
        "pixel_colors": torch.empty(1, rn, 3, dtype=torch.float32, device=dev),
        "hit_prob": torch.empty(1, rn, dn, dtype=torch.float32, device=dev) if (want_hit or fine) else None,
        "render_depth": torch.empty(1, rn, dtype=torch.float32, device=dev),
        "ray_mask_u8": torch.empty(1, rn, dtype=torch.uint8, device=dev),
    }
    if blend:
        out["blend_weights"] = torch.empty(1, rn, pack.rfn, dtype=torch.float32, device=dev)
    if agg:
        out["neuray_weights"] = torch.empty(1, rn, pack.rfn, dtype=torch.float32, device=dev)
        out["geometry_weights"] = torch.empty(1, rn, pack.rfn, dtype=torch.float32, device=dev)
    if view:
        out["view_hit"] = torch.empty(1, rn, pack.rfn, dtype=torch.float32, device=dev)
        out["view_depth"] = torch.empty(1, rn, pack.rfn, dtype=torch.float32, device=dev)
    if colors:
        out["view_colors"] = torch.empty(1, rn, pack.rfn, 3, dtype=torch.float32, device=dev)
    rec = _lib.workspace("point_rec", rn * dn * _lib.NR_POINT_REC, dev)
    p = _lib.NrPassParams()
    p.coords, p.que_depth, p.que_cam = _lib.ptr(coords_c), _lib.ptr(que_depth), _lib.ptr(cam)
    p.rn, p.dn = rn, dn
    p.feat, p.rgb, p.view_params = _lib.ptr(pack.feat), _lib.ptr(pack.rgb), _lib.ptr(pack.view_params)
    p.rfn, p.h, p.w, p.fh, p.fw = pack.rfn, pack.h, pack.w, pack.fh, pack.fw
    p.w_point, p.w_ray, p.pos_enc = _lib.ptr(w_point), _lib.ptr(w_ray), _lib.ptr(pos_enc)
    p.w_tc = _lib.ptr(w_tc)
    # compute_prob is always the COARSE decoder's method (reference renderer.py:75): its use_vis decides
    p.use_vis = 1 if owner.dist_decoder.cfg["use_vis"] else 0
    if p.use_vis and not dec.cfg["use_vis"]:
        raise _lib.NeurayB200Error("coarse dist_decoder has use_vis but the active decoder has no vis head (the reference fails too)")
    p.var_bias = float(dec.cfg["bias_val"])
    p.ray_mask_view_num, p.ray_mask_point_num = int(cfg["ray_mask_view_num"]), int(cfg["ray_mask_point_num"])
    p.point_rec = _lib.ptr(rec)
    p.pixel_colors, p.hit_prob = _lib.ptr(out["pixel_colors"]), _lib.ptr(out["hit_prob"])
    p.render_depth, p.ray_mask = _lib.ptr(out["render_depth"]), _lib.ptr(out["ray_mask_u8"])
    if fine:
        m = fine["dn"] + (dn if fine["use_all"] else 0)
        out["fine_depth"] = torch.empty(1, rn, m, dtype=torch.float32, device=dev)
        p.fine_dn, p.fine_use_all = int(fine["dn"]), 1 if fine["use_all"] else 0
        p.fine_u, p.fine_u_stride, p.fine_depth = _lib.ptr(fine["u"]), int(fine["u_stride"]), _lib.ptr(out["fine_depth"])
    stream = _lib.stream_of(coords)
    if rn == 0:          # nothing to render: the (empty) outputs are already in place
        return out, None
    with _lib.on_device(coords):
        if view:
            if _lib.PROFILE is not None:
                raise _lib.NeurayB200Error("the point kernel is timed alone only without render_view_depth")
            w = _lib.NrViewParams()
            rows = _lib.workspace("row_view", 4 * pack.rfn * rn * dn, dev)
            w.rows = _lib.ptr(rows)
            w.view_hit, w.view_depth = _lib.ptr(out["view_hit"]), _lib.ptr(out["view_depth"])
            w.blend_weights = _lib.ptr(out.get("blend_weights"))
            w.neuray_weights, w.geometry_weights = _lib.ptr(out.get("neuray_weights")), _lib.ptr(out.get("geometry_weights"))
            entry = "nr_render_pass_fwd_tf32_view" if tf32 else "nr_render_pass_fwd_view"
            _lib.check(getattr(_lib.lib(), entry)(C.byref(p), C.byref(w), stream), entry)
        elif agg:
            if _lib.PROFILE is not None:
                raise _lib.NeurayB200Error("the point kernel is timed alone only without render_agg_weights")
            a = _lib.NrAggParams()
            rows = _lib.workspace("row_agg", 3 * pack.rfn * rn * dn, dev)
            a.rows = _lib.ptr(rows)
            a.neuray_weights, a.geometry_weights = _lib.ptr(out["neuray_weights"]), _lib.ptr(out["geometry_weights"])
            a.blend_weights = _lib.ptr(out.get("blend_weights"))
            entry = "nr_render_pass_fwd_tf32_agg" if tf32 else "nr_render_pass_fwd_agg"
            _lib.check(getattr(_lib.lib(), entry)(C.byref(p), C.byref(a), stream), entry)
        elif blend or colors:
            if _lib.PROFILE is not None:
                raise _lib.NeurayB200Error("the point kernel is timed alone only without render_blend_weights and render_view_colors")
            b = _lib.NrBlendParams()
            rows = _lib.workspace("row_blend", pack.rfn * rn * dn, dev)
            b.row_blend = _lib.ptr(rows)
            b.blend_weights = _lib.ptr(out.get("blend_weights"))   # NULL with colors alone: the reduction is skipped
            entry = "nr_render_pass_fwd_tf32_blend" if tf32 else "nr_render_pass_fwd_blend"
            _lib.check(getattr(_lib.lib(), entry)(C.byref(p), C.byref(b), stream), entry)
        elif _lib.PROFILE is not None:
            # bench.py: time the dominant kernel alone, with CUDA events on the launching stream
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            if tf32:
                _lib.check(_lib.lib().nr_point_kernel_tf32(C.byref(p), stream), "nr_point_kernel_tf32")
            else:
                _lib.check(_lib.lib().nr_point_kernel(C.byref(p), stream), "nr_point_kernel")
            e1.record()
            _lib.check(_lib.lib().nr_ray_kernel(C.byref(p), stream), "nr_ray_kernel")
            e2.record()
            _lib.PROFILE.append((e0, e1, rn * dn, e2))
        elif tf32:
            _lib.check(_lib.lib().nr_render_pass_fwd_tf32(C.byref(p), stream), "nr_render_pass_fwd_tf32")
        else:
            _lib.check(_lib.lib().nr_render_pass_fwd(C.byref(p), stream), "nr_render_pass_fwd")
        if colors:       # plane 0 of each export workspace is the blend row
            c = _lib.NrColorParams()
            c.row_blend, c.hit_prob, c.view_colors = _lib.ptr(rows), _lib.ptr(out["hit_prob"]), _lib.ptr(out["view_colors"])
            _lib.check(_lib.lib().nr_view_colors(C.byref(p), C.byref(c), stream), "nr_view_colors")
    _lib.count_launches(2 + (2 if view else 0) + (2 if agg else 0) + (1 if blend else 0) + (1 if colors else 0))
    return out, PassLaunch(p, (coords_c, que_depth, cam, pack, w_point, w_ray, pos_enc, w_tc), (pack.rfn, pack.fh, pack.fw, 64), stream)


def run_pass(owner, que_depth, que_imgs_info, ref_imgs_info, is_fine, fine=None, want_hit=True):
    """One fused pass.  que_depth [1,rn,dn].  `fine`: None or dict(dn=, use_all=, u=, u_stride=) to also emit the
    next pass' depths.  Returns dict with pixel_colors [1,rn,3], hit_prob [1,rn,dn], render_depth [1,rn],
    ray_mask [1,rn] (bool), optionally fine_depth [1,rn,M], with cfg use_dr_prediction, pixel_colors_dr [1,rn,3] and
    hit_prob_dr [1,rn,dn] (direct rendering, forward only: under autograd their backward raises), with cfg
    render_visibility, visibility [1,rn,rfn], with cfg render_blend_weights, blend_weights [1,rn,rfn] and, with cfg
    render_agg_weights, neuray_weights and geometry_weights [1,rn,rfn], with cfg render_view_depth, view_hit and
    view_depth [1,rn,rfn] and, with cfg render_view_colors, view_colors [1,rn,rfn,3] (none of these has a gradient:
    requires_grad is False).

    When gradients are being recorded and the reference feature maps or any parameter of the pass require them, the
    outputs are attached to autograd through backward.RenderPassFn (forward values still come from the kernels), and the
    pass runs in fp32 whatever set_precision chose: the backward recomputes it in fp32.  Otherwise PRECISION applies."""
    coords = que_imgs_info["coords"]
    if coords.shape[0] != 1:
        raise _lib.NeurayB200Error("one query view per call (qn == 1), like every call site of the reference")
    que_depth = que_depth.detach().contiguous().float()
    _, rn, dn = que_depth.shape
    if dn > _lib.NR_MAX_SAMPLES:
        raise _lib.NeurayB200Error(f"at most {_lib.NR_MAX_SAMPLES} samples per ray per pass, got {dn}")
    pp = pass_params(owner, is_fine)
    rf, imf = ref_imgs_info["ray_feats"], ref_imgs_info["img_feats"]
    params = [v for _, v in pp.named]
    needs_grad = torch.is_grad_enabled() and (rf.requires_grad or imf.requires_grad or any(v.requires_grad for v in params))
    want_dr, want_vis = owner.cfg["use_dr_prediction"], owner.cfg.get("render_visibility", False)
    want_blend, want_agg = owner.cfg.get("render_blend_weights", False), owner.cfg.get("render_agg_weights", False)
    want_view, want_colors = owner.cfg.get("render_view_depth", False), owner.cfg.get("render_view_colors", False)
    out, launch = _launch_pass(owner, que_depth, que_imgs_info, ref_imgs_info, pp, fine,
                               want_hit or want_vis or want_blend or want_agg or want_colors, PRECISION == "tf32" and not needs_grad,
                               want_blend, want_agg, want_view, want_colors)
    dr = _direct_render(owner, launch, rn, dn, coords.device) if want_dr else None
    if want_vis:
        out["visibility"] = _view_visibility(launch, out["hit_prob"], rn, rf.shape[0], coords.device)
    if needs_grad:
        from .backward import DirectRenderFn, RenderPassFn
        meta = {"names": [n for n, _ in pp.named], "dec": pp.dec_name, "agg": pp.agg_name}
        res = RenderPassFn.apply(launch, out, meta, rf, imf, *params)
        out.update(zip(("pixel_colors", "hit_prob", "render_depth", "ray_mask_u8", "fine_depth"), res))
        if dr is not None:
            dr = dict(zip(("pixel_colors_dr", "hit_prob_dr"), DirectRenderFn.apply(dr, rf, imf, *params)))
    if dr is not None:
        out.update(dr)
    out["ray_mask"] = out.pop("ray_mask_u8").bool()
    return out


# the optional outputs of a pass: (cfg switch, run_pass key, output key)
_OPTIONAL_OUTPUTS = (("use_dr_prediction", "pixel_colors_dr", "pixel_colors_dr"), ("use_dr_prediction", "hit_prob_dr", "hit_prob_dr"),
                     ("use_ray_mask", "ray_mask", "ray_mask"), ("render_depth", "render_depth", "render_depth"),
                     ("render_visibility", "visibility", "visibility_nr"), ("render_blend_weights", "blend_weights", "blend_weights_nr"),
                     ("render_agg_weights", "neuray_weights", "neuray_weights_nr"),
                     ("render_agg_weights", "geometry_weights", "geometry_weights_nr"),
                     ("render_view_depth", "view_hit", "view_hit_nr"), ("render_view_depth", "view_depth", "view_depth_nr"),
                     ("render_view_colors", "view_colors", "view_colors_nr"))


def _finish_outputs(owner, res, que_imgs_info):
    outputs = {"pixel_colors_nr": res["pixel_colors"], "hit_prob_nr": res["hit_prob"]}
    if "imgs" in que_imgs_info:
        outputs["pixel_colors_gt"] = interpolate_feats(que_imgs_info["imgs"], que_imgs_info["coords"], align_corners=True)
    outputs.update((key, res[raw]) for switch, raw, key in _OPTIONAL_OUTPUTS if owner.cfg.get(switch, False))
    return outputs


def _self_hit_prob(self, que_depth, que_imgs_info, is_fine):
    """a17 predict_self_hit_prob (reference renderer.py:137-155): the query view's own ray_feats decoded along its rays
    (fine-tuning configs).  nr_self_hit_prob, forward and backward."""
    pp = pass_params(self, is_fine)
    dec = pp.dec
    feats = que_imgs_info["ray_feats"]
    coords = que_imgs_info["coords"]
    h, w = que_imgs_info["imgs"].shape[-2:]
    if feats.shape[0] != 1 or coords.shape[0] != 1:
        raise _lib.NeurayB200Error("one query view per call (qn == 1), like every call site of the reference")
    from .backward import SelfHitProbFn
    dev = coords.device
    _, rn, dn = que_depth.shape
    w_point = pass_weights(self, is_fine, dn, dev)[0]
    index_map = pass_index_map(self, pp, dev)
    fmap = feats[0].detach().contiguous().float()
    cc, qd = coords[0].detach().contiguous().float(), que_depth[0].detach().contiguous().float()
    rng = que_imgs_info["depth_range"][0].detach().float().contiguous()
    use_vis, var_bias = 1 if dec.cfg["use_vis"] else 0, float(dec.cfg["bias_val"])

    def params():
        p = _lib.NrSelfParams()
        p.map, p.coords, p.que_depth, p.w_point = _lib.ptr(fmap), _lib.ptr(cc), _lib.ptr(qd), _lib.ptr(w_point)
        p.rn, p.dn, p.h, p.w, p.fh, p.fw, p.use_vis = rn, dn, int(h), int(w), fmap.shape[1], fmap.shape[2], use_vis
        p.depth_range, p.var_bias = _lib.ptr(rng), var_bias
        return p

    named = [(n, v) for n, v in pp.named if n.startswith(pp.dec_name + ".")]
    meta = {"params": params, "index_map": index_map, "stream": _lib.stream_of(coords), "map_shape": tuple(fmap.shape),
            "dec_names": [n for n, _ in named], "keep": (fmap, cc, qd, w_point, rng)}
    return SelfHitProbFn.apply(meta, feats, *[v for _, v in named])


def render_by_depth(self, que_depth, que_imgs_info, ref_imgs_info, is_train, is_fine):
    """reference renderer.py:168-203."""
    res = run_pass(self, que_depth, que_imgs_info, ref_imgs_info, is_fine)
    outputs = _finish_outputs(self, res, que_imgs_info)
    if is_train and self.cfg["use_self_hit_prob"]:
        outputs["hit_prob_self"] = _self_hit_prob(self, que_depth, que_imgs_info, is_fine)
    return outputs


def _fine_request(self, rn, is_train, device):
    fdn = int(self.cfg["fine_depth_sample_num"])
    if is_train:
        u = torch.rand([1, rn, fdn]).to(device).contiguous()       # CPU generator, as reference render_ops.py:205-209
        return {"dn": fdn, "use_all": bool(self.cfg["fine_depth_use_all"]), "u": u, "u_stride": fdn}
    return {"dn": fdn, "use_all": bool(self.cfg["fine_depth_use_all"]), "u": fine_sample_u(fdn, device), "u_stride": 0}


def fine_render_impl(self, coarse_render_info, que_imgs_info, ref_imgs_info, is_train):
    """reference renderer.py:205-215 (stand-alone form: resample with the CUDA sample_fine_depth, then a fine pass)."""
    from .render_ops import sample_fine_depth
    fine_depth = sample_fine_depth(coarse_render_info["depth"], coarse_render_info["hit_prob"].detach(),
                                   que_imgs_info["depth_range"], self.cfg["fine_depth_sample_num"], is_train)
    if self.cfg["fine_depth_use_all"]:
        que_depth = torch.sort(torch.cat([coarse_render_info["depth"], fine_depth], -1), -1)[0]
    else:
        que_depth = torch.sort(fine_depth, -1)[0]
    return render_by_depth(self, que_depth, que_imgs_info, ref_imgs_info, is_train, True)


def render_impl(self, que_imgs_info, ref_imgs_info, is_train):
    """reference renderer.py:217-226: coarse pass, fused resampling, fine pass."""
    que_depth, _ = sample_depth(que_imgs_info["depth_range"], que_imgs_info["coords"], self.cfg["depth_sample_num"], False)
    hier = bool(self.cfg["use_hierarchical_sampling"])
    rn = que_imgs_info["coords"].shape[1]
    fine = _fine_request(self, rn, is_train, que_depth.device) if hier else None
    res = run_pass(self, que_depth, que_imgs_info, ref_imgs_info, False, fine=fine)
    outputs = _finish_outputs(self, res, que_imgs_info)
    self_hit = is_train and self.cfg["use_self_hit_prob"]
    if self_hit:
        outputs["hit_prob_self"] = _self_hit_prob(self, que_depth, que_imgs_info, False)
    if hier:
        res_f = run_pass(self, res["fine_depth"], que_imgs_info, ref_imgs_info, True)
        fine_out = _finish_outputs(self, res_f, que_imgs_info)
        if self_hit:
            fine_out["hit_prob_self"] = _self_hit_prob(self, res["fine_depth"], que_imgs_info, True)
        for k, v in fine_out.items():
            outputs[k + "_fine"] = v
    return outputs


def render_chunks(self, que_imgs_info, ref_imgs_info, is_train, pack=None):
    """The chunk loop of reference renderer.py:236-254 (everything after the encoders).  The per-frame pack (channel-last
    maps, per-view parameters) and the query camera block are built once here and live exactly as long as this call: they
    are handed to the per-chunk functions through the two info dicts and removed again before returning."""
    ray_batch_num = self.cfg["ray_batch_num"]
    coords = que_imgs_info["coords"]
    ray_num = coords.shape[1]
    render_info_all = {}
    ref_imgs_info[PACK_KEY] = pack if pack is not None else FramePack(ref_imgs_info)
    que_imgs_info[CAM_KEY] = camera_blocks(que_imgs_info, None)[0]
    try:
        # an empty ray set still runs one (empty) chunk so that the caller gets every key with a zero-length ray axis
        for ray_id in range(0, max(ray_num, 1), ray_batch_num):
            que_imgs_info["coords"] = coords[:, ray_id:ray_id + ray_batch_num]
            render_info = render_impl(self, que_imgs_info, ref_imgs_info, is_train)
            for k, v in render_info.items():
                if is_train or (not k.startswith("hit_prob")):
                    render_info_all.setdefault(k, []).append(v)
    finally:
        que_imgs_info["coords"] = coords
        ref_imgs_info.pop(PACK_KEY, None)
        que_imgs_info.pop(CAM_KEY, None)
    return {k: (v[0] if len(v) == 1 else torch.cat(v, 1)) for k, v in render_info_all.items()}


def render(self, que_imgs_info, ref_imgs_info, is_train):
    """reference renderer.py:228-254, for an owner that has the reference's encoders.  Inference runs the two encoders
    natively, straight into the channel-last frame pack (encoders.encode_frame); when a gradient is wanted through them
    (training) the owner's own torch modules run, upstream of the boundary, exactly as in the reference."""
    pack = None
    if encoders.usable(self, ref_imgs_info):
        pack = FramePack(ref_imgs_info, encoder_owner=self)
    else:
        ref_img_feats = self.image_encoder(ref_imgs_info["imgs"])
        ref_imgs_info["img_feats"] = ref_img_feats
        ref_imgs_info["ray_feats"] = self.vis_encoder(ref_imgs_info["ray_feats"], ref_img_feats)
    if is_train and self.cfg["use_self_hit_prob"]:
        que_img_feats = self.image_encoder(que_imgs_info["imgs"])
        que_imgs_info["ray_feats"] = self.vis_encoder(que_imgs_info["ray_feats"], que_img_feats)
    return render_chunks(self, que_imgs_info, ref_imgs_info, is_train, pack)


class NeuralRayRenderPath(nn.Module):
    """The hot path as a stand-alone module: parameters under the reference's state-dict names, kernels for the math.

    `render(que_imgs_info, ref_imgs_info, is_train)` expects ref_imgs_info to already hold the encoder outputs
    'ray_feats' and 'img_feats' [rfn,32,H/4,W/4] (reference renderer.py:229-231 produces them; the CNN encoders are
    out of scope, SURVEY.md section 8f)."""
    base_cfg = base_cfg

    def __init__(self, cfg):
        super().__init__()
        self.cfg = {**self.base_cfg, **cfg}
        self.dist_decoder = modules.name2dist_decoder[self.cfg["dist_decoder_type"]](self.cfg["dist_decoder_cfg"])
        self.agg_net = modules.name2agg_net[self.cfg["agg_net_type"]](self.cfg["agg_net_cfg"])
        if self.cfg["use_hierarchical_sampling"]:
            self.fine_dist_decoder = modules.name2dist_decoder[self.cfg["dist_decoder_type"]](self.cfg["fine_dist_decoder_cfg"])
            self.fine_agg_net = modules.name2agg_net[self.cfg["agg_net_type"]](self.cfg["fine_agg_net_cfg"])

    render_by_depth = render_by_depth
    fine_render_impl = fine_render_impl
    render_impl = render_impl

    def predict_mean_for_depth_loss(self, ref_imgs_info):
        """NeuralRayGenRenderer.predict_mean_for_depth_loss (reference renderer.py:280-316); cfg 'depth_loss_coords_num'."""
        from . import losses
        return losses.predict_mean_for_depth_loss(self, ref_imgs_info)

    def render(self, que_imgs_info, ref_imgs_info, is_train):
        return render_chunks(self, dict(que_imgs_info), ref_imgs_info, is_train)

    def forward(self, data):
        is_train = "eval" not in data
        return self.render(data["que_imgs_info"].copy(), data["ref_imgs_info"].copy(), is_train)


class NeuralRayFrameRenderer(NeuralRayRenderPath):
    """NeuralRayRenderPath plus the two encoders of NeuralRayBaseRenderer (renderer.py:56-59), under the reference's
    state-dict names `image_encoder.*` / `vis_encoder.*`: `render()` is the reference's `render` (renderer.py:228-254) --
    ref_imgs_info carries the INIT net's 'ray_feats' [rfn,32,H/4,W/4]; both encoders run natively into the frame pack."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.image_encoder = encoders.ImageEncoder()
        self.vis_encoder = encoders.VisEncoder(self.cfg["vis_encoder_cfg"])

    def render(self, que_imgs_info, ref_imgs_info, is_train):
        return render(self, dict(que_imgs_info), ref_imgs_info, is_train)


class NeuralRayGenFrameRenderer(NeuralRayFrameRenderer):
    """The inference frame path of NeuralRayGenRenderer (reference renderer.py:255-327; init_net_type 'depth' = the neuray_gen_depth
    model, 'cost_volume' = neuray_gen_cost_volume with its MVSNet): init net -> image_encoder + vis_encoder -> chunk loop, every stage native, the three front
    stages writing the channel-last frame pack in place.  State-dict names are the reference's (`init_net.*`,
    `image_encoder.*`, `vis_encoder.*`, `dist_decoder.*`, ...), so a gen-model checkpoint loads unchanged.
    ref_imgs_info carries imgs, depth_range, poses, Ks and depth (DepthInitNet) or nn_ids + data['src_imgs_info'] (CostVolumeInitNet);
    forward(data) like the reference."""

    def __init__(self, cfg):
        super().__init__(cfg)
        kind = self.cfg.get("init_net_type", "depth")
        if kind not in ("depth", "cost_volume"):
            raise ValueError(f"init_net_type {kind!r}")
        self.init_net = (init_nets.DepthInitNet if kind == "depth" else init_nets.CostVolumeInitNet)(self.cfg.get("init_net_cfg", {}))

    def render_call(self, que_imgs_info, ref_imgs_info, is_train, src_imgs_info=None):
        """renderer.py:268-270: the init net's ray_feats go straight into the frame pack (no 'ray_feats' entry needed)."""
        ref_imgs_info.pop("ray_feats", None)
        ref_imgs_info[init_nets.SRC_KEY] = src_imgs_info
        if not encoders.usable(self, ref_imgs_info):
            raise _lib.NeurayB200Error("NeuralRayGenFrameRenderer is the INFERENCE frame path (CUDA tensors, torch.no_grad() or frozen front-end "
                                       "parameters); training goes through patch.install() on the reference's NeuralRayGenRenderer")
        return render(self, dict(que_imgs_info), ref_imgs_info, is_train)

    def forward(self, data):
        ref_imgs_info, que_imgs_info = data["ref_imgs_info"].copy(), data["que_imgs_info"].copy()
        is_train = "eval" not in data
        out = self.render_call(que_imgs_info, ref_imgs_info, is_train, data.get("src_imgs_info"))
        if (self.cfg["use_depth_loss"] and "true_depth" in ref_imgs_info) or (not is_train):
            out.update(self.predict_mean_for_depth_loss(ref_imgs_info))
        return out

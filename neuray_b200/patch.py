"""Installs the native path into an importable reference tree so that its own entry points (render.py,
run_training.py, eval.py) run unchanged:

    import neuray_b200.patch as patch
    patch.install()            # before the reference builds its network
    ...                        # the reference's code, untouched

What is rebound (SURVEY.md section 8b):
  * every function of network/render_ops.py  -> neuray_b200.render_ops (also inside network.renderer's and
    network.init_net's namespaces, which star-/name-import them)
  * NeuralRayBaseRenderer.render_by_depth / fine_render_impl / render_impl / render -> neuray_b200.renderer
  * network.init_net.get_diff_feats (DepthInitNet, SURVEY.md 8f row 2) -> neuray_b200.init_ops.get_diff_feats;
    DepthInitNet.forward / CostVolumeInitNet.forward -> neuray_b200.init_nets (inference: the whole init net natively, MVSNet included)
  * NeuralRayGenRenderer.predict_mean_for_depth_loss and network.loss.{RenderLoss, DepthLoss, ConsistencyLoss, name2loss}
    (SURVEY.md 8f row 3) -> neuray_b200.losses
  * network.metrics.{PSNR_SSIM, name2metrics['psnr_ssim']} -> neuray_b200.metrics (the validation PSNR / SSIM on the GPU;
    vis_img stays the reference's, it writes the JPEGs)
  * inference only: `render` runs image_encoder / vis_encoder natively into the frame pack (SURVEY.md 8f row 1,
    neuray_b200.encoders); with a gradient wanted through them the reference's own torch modules run
Constructors, cfg keys, sub-module and state-dict names, and the output dict stay the reference's own.
The IBRNetWithNeuRay.pos_encoding attribute pinned to cuda:0 (ibrnet.py:312) is no longer used on the path: the
kernels get a per-device table built by neuray_b200.weights.posenc_table.
"""
import importlib

from . import init_nets, init_ops, losses, metrics, render_ops, renderer

_ORIGINALS = []          # (object, attribute name, original value) of everything install() rebound


def _rebind(obj, name, value):
    if isinstance(obj, dict):
        _ORIGINALS.append((obj, name, obj[name]))
        obj[name] = value
        return
    _ORIGINALS.append((obj, name, getattr(obj, name)))
    setattr(obj, name, value)


def install():
    """Idempotent.  Autograd: the renderer methods attach their outputs to the graph (backward.RenderPassFn /
    SelfHitProbFn); of the render_ops drop-ins only interpolate_feats / interpolate_feature_map are differentiated by the
    reference (with respect to the map: predict_mean_for_depth_loss, predict_self_hit_prob) and carry a native backward;
    the others raise if handed an input that requires grad instead of silently cutting the graph."""
    if _ORIGINALS:
        return importlib.import_module("network.renderer").NeuralRayBaseRenderer
    ref_ops = importlib.import_module("network.render_ops")
    ref_renderer = importlib.import_module("network.renderer")
    targets = [ref_ops, ref_renderer]
    try:
        ref_init = importlib.import_module("network.init_net")
        targets.append(ref_init)
        _rebind(ref_init, "get_diff_feats", init_ops.get_diff_feats)      # DepthInitNet's per-frame reprojection features
        # inference: the whole DepthInitNet natively (ResEncoder on the tensor cores); with a gradient wanted, the reference's
        _rebind(ref_init.DepthInitNet, "forward", init_nets.forward_or_reference(ref_init.DepthInitNet.forward))
        _rebind(ref_init.CostVolumeInitNet, "forward", init_nets.cost_volume_forward_or_reference(ref_init.CostVolumeInitNet.forward))
    except Exception:      # init_net needs inplace_abn / kornia; the rendering path does not
        pass
    for name in render_ops.__all__:
        fn = getattr(render_ops, name)
        for mod in targets:
            if hasattr(mod, name):
                _rebind(mod, name, fn)
    base = ref_renderer.NeuralRayBaseRenderer
    _rebind(base, "render_by_depth", renderer.render_by_depth)
    _rebind(base, "fine_render_impl", renderer.fine_render_impl)
    _rebind(base, "render_impl", renderer.render_impl)
    _rebind(base, "render", renderer.render)
    _rebind(ref_renderer.NeuralRayGenRenderer, "predict_mean_for_depth_loss", losses.predict_mean_for_depth_loss)
    try:
        ref_loss = importlib.import_module("network.loss")
        for key, cls in losses.name2loss.items():
            _rebind(ref_loss.name2loss, key, cls)
            _rebind(ref_loss, cls.__name__, cls)
    except Exception:      # a trimmed reference tree without the training code
        pass
    try:
        ref_metrics = importlib.import_module("network.metrics")
        _rebind(ref_metrics.name2metrics, "psnr_ssim", metrics.PSNR_SSIM)
        _rebind(ref_metrics, "PSNR_SSIM", metrics.PSNR_SSIM)
    except Exception:      # network.metrics needs skimage; a trimmed tree may not have it
        pass
    return base


def uninstall():
    """Puts the reference's own functions back (tests compare patched and unpatched runs in one process)."""
    while _ORIGINALS:
        obj, name, value = _ORIGINALS.pop()
        if isinstance(obj, dict):
            obj[name] = value
        else:
            setattr(obj, name, value)

"""neuray_b200 -- H100-native (sm_90a) implementation of NeuRay's per-ray rendering hot path.

Drop-in surface (SURVEY.md section 8b):
    neuray_b200.render_ops      mirrors reference network/render_ops.py (same 12 function names)
    neuray_b200.renderer        NeuralRayBaseRenderer-compatible render_by_depth / render_impl / render
    neuray_b200.init_ops        get_diff_feats of the reference's DepthInitNet (network/init_net.py:29-61)
    neuray_b200.init_nets       DepthInitNet and CostVolumeInitNet (with its frozen MVSNet), inference (network/init_net.py:63-254)
    neuray_b200.encoders        image_encoder (ResUNetLight) and vis_encoder, inference, channel-last into the frame pack
    neuray_b200.losses          predict_mean_for_depth_loss, RenderLoss / DepthLoss / ConsistencyLoss (forward + backward)
    neuray_b200.metrics         PSNR_SSIM, the validation PSNR / SSIM (network/metrics.py:13-79)
    neuray_b200.eval_metrics    eval.py's scores: TensorFlow's PSNR / SSIM and LPIPS-VGG (python -m neuray_b200.eval scores a folder)
    neuray_b200.patch           installs them into an importable reference tree (render.py / run_training.py unchanged)
    neuray_b200.dist            ray-sharded rendering + gradient all-reduce over torch.distributed (NCCL)

All arithmetic runs in hand-written CUDA kernels behind the C-ABI declared in include/neuray_b200.h
(libneuray_b200.so, loaded with ctypes).  There is no CPU or PyTorch fallback: calling any op without the
built library, or with non-CUDA tensors, raises.
"""
__version__ = "0.3.0"

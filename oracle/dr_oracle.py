"""TEST INFRASTRUCTURE ONLY -- CPU oracle for direct rendering (cfg use_dr_prediction), next to oracle/neuray_oracle.py.

A functional restatement of the reference (liuyuan-pal/NeuRay) on top of the intermediates that
neuray_oracle.render_by_depth(..., keep=...) records:

    network/renderer.py:85-125, 181-185   predict_alpha_values_dr, predict_colors_dr, direct_rendering
    network/sph_solver.py:5-59            SphericalHarmonicsSolver (degree 3), the normal equations solved in fp64

Pinned against the unmodified reference's outputs in tests/golden/dr.npz (oracle/gen_golden_dr.py; checked by
tests/test_dr_cpu.py).  Only tests/ may import this file: the product path (neuray_b200/) never does.
"""
import torch

import neuray_oracle as orc

SH_REGS = [0.0] + [0.001] * 3 + [0.005] * 5 + [0.05] * 7      # SphericalHarmonicsSolver(3).regs


def sh_basis(d):
    """sph_solver.py:14-30, degree 3: [..., 3] -> [..., 16]."""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    return torch.stack([torch.ones_like(x), x, y, z,
                        x * y, y * z, -x ** 2 - y ** 2 + 2 * z ** 2, z * x, x ** 2 - y ** 2,
                        (3 * x ** 2 - y ** 2) * y, x * y * z, y * (4 * z ** 2 - x ** 2 - y ** 2), z * (2 * z ** 2 - 3 * x ** 2 - 3 * y ** 2),
                        x * (4 * z ** 2 - x ** 2 - y ** 2), (x ** 2 - y ** 2) * z, (x ** 2 - 3 * y ** 2) * x], -1)


def sh_normal_equations(dirs, colors, weights, regs):
    """sph_solver.py:32-49 up to the inverse: dirs / colors [b,n,3], weights [b,n] -> M [b,16,16], rhs [b,16,3]."""
    A = sh_basis(dirs)
    weights = weights + (weights.sum(1, keepdim=True) < 1e-4).to(weights.dtype) * 1e-4
    A_ = (A * weights[..., None]).transpose(1, 2)
    return A_ @ A + torch.diag(regs), A_ @ colors


def direct_rendering(cfg, keep, regs=None, dtype=torch.float64, info=None):
    """predict_alpha_values_dr, predict_colors_dr and direct_rendering (renderer.py:85-125) on the intermediates that
    render_by_depth(..., keep=keep) recorded for the same pass; computed in `dtype`.  Returns pixel_colors_dr [qn,rn,3]
    and hit_prob_dr [qn,rn,dn].  `info` (optional dict) receives the normal matrices' 2-norm condition numbers 'cond'
    [qn,rn,dn] (None with use_nr_color_for_dr)."""
    gs = float(cfg.get("alpha_value_ground_state", -15))
    mask = keep["prj_mask"].to(dtype)                                           # rfn,qn,rn,dn,1
    hit, vis = keep["prj_hit_prob"].to(dtype), keep["prj_vis"].to(dtype)
    # predict_proj_ray_prob (renderer.py:79-82): where the mask is 1 the masked values are the raw ones
    alpha = torch.where(mask > 0, torch.log(hit / (vis - hit + 1e-5) + 1e-5), torch.full_like(hit, gs))
    alpha_dr = (vis * alpha).sum(0) / (vis.sum(0) + 1e-5)
    alpha_dr = torch.where(mask.sum(0) == 0, torch.full_like(alpha_dr, gs), alpha_dr)[..., 0]   # qn,rn,dn
    qn, rn, dn = alpha_dr.shape
    if cfg.get("use_nr_color_for_dr", False):
        colors = keep["colors"].to(dtype)
        cond = None
    else:
        rfn = mask.shape[0]
        pn = qn * rn * dn
        w = hit.reshape(rfn, pn)
        w = w / (w.sum(0, keepdim=True) + 1e-3)
        M, rhs = sh_normal_equations(keep["prj_dir"].to(dtype).reshape(rfn, pn, 3).transpose(0, 1),
                                     keep["prj_rgb"].to(dtype).reshape(rfn, pn, 3).transpose(0, 1), w.t(),
                                     torch.tensor(SH_REGS if regs is None else regs, dtype=dtype))
        theta = torch.linalg.solve(M, rhs)                                        # pn,16,3
        colors = (sh_basis(keep["que_dir"].to(dtype).reshape(pn, 1, 3)) @ theta).reshape(qn, rn, dn, 3)
        cond = torch.linalg.cond(M).reshape(qn, rn, dn)
    if info is not None:
        info["cond"] = cond
    hit_dr = orc.alpha_values2hit_prob(torch.sigmoid(alpha_dr))
    return (hit_dr[..., None] * colors).sum(2), hit_dr


def render_impl_dr(W, cfg, que, ref, is_train, fine_u=None, fine_depth_override=None, regs=None, dtype=torch.float64, info=None):
    """render_impl with use_dr_prediction: its outputs plus pixel_colors_dr / hit_prob_dr of each pass (and '_fine'
    twins).  `info` (optional dict) receives 'cond' and 'cond_fine' (see direct_rendering)."""
    out = orc.render_impl(W, cfg, que, ref, is_train, fine_u, fine_depth_override)
    passes = [("", out["que_depth"], False)]
    if cfg["use_hierarchical_sampling"]:
        passes.append(("_fine", out["que_depth_fine"], True))
    for sfx, depth, is_fine in passes:
        keep, pinfo = {}, {}
        orc.render_by_depth(W, cfg, depth, que, ref, is_train, is_fine, keep)
        out["pixel_colors_dr" + sfx], out["hit_prob_dr" + sfx] = direct_rendering(cfg, keep, regs, dtype, pinfo)
        if info is not None:
            info["cond" + sfx] = pinfo["cond"]
    return out

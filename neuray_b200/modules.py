"""Parameter containers for the per-ray rendering path.

These mirror the *types* of the reference hot path (SURVEY.md section 8, row a18) so that a reference
checkpoint loads unchanged -- the state-dict key names and shapes are the compatibility surface:

    MixtureLogisticsDistDecoder   reference network/dist_decoder.py:53-97
    DefaultAggregationNet         reference network/aggregate_net.py:16-32
    IBRNetWithNeuRay              reference network/ibrnet.py:239-300
    MultiHeadAttention            reference network/ibrnet.py:52-72

They hold parameters only.  There is deliberately no torch `forward`: the arithmetic runs in the CUDA
kernels (neuray_b200/csrc).
"""
import torch
import torch.nn as nn


def _kaiming(seq):
    for m in seq:
        if isinstance(m, nn.Linear):
            nn.init.kaiming_normal_(m.weight.data)
            if m.bias is not None:
                nn.init.zeros_(m.bias.data)


class _NoForward(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; the math lives in the CUDA path")


class AddBias(_NoForward):
    """reference network/ops.py:78-84 AddBias: a constant (not a parameter) added to the variance head."""
    def __init__(self, val):
        super().__init__()
        self.val = val


def _head(din, dhid, dout, act):
    # indices 0,2,4 carry the Linear layers, exactly like the reference nn.Sequential
    return [nn.Linear(din, dhid), nn.ELU(), nn.Linear(dhid, dhid), nn.ELU(), nn.Linear(dhid, dout), act]


class MixtureLogisticsDistDecoder(_NoForward):
    default_cfg = {"feats_dim": 32, "bias_val": 0.05, "use_vis": True}

    def __init__(self, cfg):
        super().__init__()
        self.cfg = {**self.default_cfg, **cfg}
        d = self.cfg["feats_dim"]
        self.mean_decoder = nn.Sequential(*_head(d, d, 2, nn.Softplus()))
        self.var_decoder = nn.Sequential(*_head(d, d, 2, nn.Softplus()), AddBias(self.cfg["bias_val"]))
        self.aw_decoder = nn.Sequential(*_head(d, d, 1, nn.Sigmoid()))
        if self.cfg["use_vis"]:
            self.vis_decoder = nn.Sequential(*_head(d, d, 1, nn.Sigmoid()))


class MultiHeadAttention(_NoForward):
    def __init__(self, n_head=4, d_model=16, d_k=4, d_v=4):
        super().__init__()
        self.n_head, self.d_k, self.d_v = n_head, d_k, d_v
        self.w_qs = nn.Linear(d_model, n_head * d_k, bias=False)
        self.w_ks = nn.Linear(d_model, n_head * d_k, bias=False)
        self.w_vs = nn.Linear(d_model, n_head * d_v, bias=False)
        self.fc = nn.Linear(n_head * d_v, d_model, bias=False)
        self.layer_norm = nn.LayerNorm(d_model, eps=1e-6)


class IBRNetWithNeuRay(_NoForward):
    def __init__(self, neuray_in_dim=32, in_feat_ch=32, n_samples=64):
        super().__init__()
        self.n_samples = n_samples
        act = nn.ELU
        self.ray_dir_fc = nn.Sequential(nn.Linear(4, 16), act(), nn.Linear(16, in_feat_ch + 3), act())
        self.base_fc = nn.Sequential(nn.Linear((in_feat_ch + 3) * 5 + neuray_in_dim, 64), act(), nn.Linear(64, 32), act())
        self.vis_fc = nn.Sequential(nn.Linear(32, 32), act(), nn.Linear(32, 33), act())
        self.vis_fc2 = nn.Sequential(nn.Linear(32, 32), act(), nn.Linear(32, 1), nn.Sigmoid())
        self.geometry_fc = nn.Sequential(nn.Linear(32 * 2 + 1, 64), act(), nn.Linear(64, 16), act())
        self.ray_attention = MultiHeadAttention(4, 16, 4, 4)
        self.out_geometry_fc = nn.Sequential(nn.Linear(16, 16), act(), nn.Linear(16, 1), nn.ReLU())
        self.rgb_fc = nn.Sequential(nn.Linear(32 + 1 + 4, 16), act(), nn.Linear(16, 8), act(), nn.Linear(8, 1))
        self.neuray_fc = nn.Sequential(nn.Linear(neuray_in_dim, 8), act(), nn.Linear(8, 1))
        for seq in (self.base_fc, self.vis_fc2, self.vis_fc, self.geometry_fc, self.rgb_fc, self.neuray_fc):
            _kaiming(seq)

    def change_pos_encoding(self, n_samples):
        self.n_samples = n_samples


class DefaultAggregationNet(_NoForward):
    default_cfg = {"sample_num": 64, "neuray_dim": 32, "use_img_feats": False}

    def __init__(self, cfg):
        super().__init__()
        self.cfg = {**self.default_cfg, **cfg}
        dim = self.cfg["neuray_dim"]
        self.agg_impl = IBRNetWithNeuRay(dim, n_samples=self.cfg["sample_num"])
        self.prob_embed = nn.Sequential(nn.Linear(2 + 32, dim), nn.ReLU(), nn.Linear(dim, dim))


name2dist_decoder = {"mixture_logistics": MixtureLogisticsDistDecoder}
name2agg_net = {"default": DefaultAggregationNet}

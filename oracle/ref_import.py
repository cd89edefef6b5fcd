"""TEST INFRASTRUCTURE ONLY -- loads the *unmodified* reference (liuyuan-pal/NeuRay) from
/root/reference so that golden vectors can be generated from it (oracle/gen_golden.py).

The reference is pure Python/PyTorch but `network/renderer.py` transitively imports packages that
are absent from this image (skimage, easydict, h5py, plyfile, transforms3d, imageio, matplotlib,
tensorboardX, inplace_abn, kornia).  None of them is touched by the per-ray rendering path, so we
register empty module stubs (with a __spec__, otherwise torch._dynamo's find_spec probes break) and
let the reference import.  `IBRNetWithNeuRay.posenc` pins its table to "cuda:0"
(network/ibrnet.py:312); on a GPU-less box we make that particular `.to("cuda:0")` a no-op.

Nothing in neuray_b200/, tests/ or bench.py may import this file: only the golden generators under oracle/ do.  Root of the
reference tree: $NEURAY_REFERENCE_ROOT, else /root/reference.  `inplace_abn` (ABN / InPlaceABN = batch-norm + leaky_relu(0.01), loads network/mvsnet/mvsnet_pl.ckpt strictly)
and `kornia.utils.create_meshgrid` get functional stand-ins because CostVolumeInitNet / MVSNet really call them.
"""
import importlib.machinery
import os
import sys
import types

def _find_root():
    return os.environ.get("NEURAY_REFERENCE_ROOT", "/root/reference")


REFERENCE_ROOT = _find_root()

_STUBS = [
    "easydict", "skimage", "skimage.io", "skimage.metrics", "kornia", "kornia.utils", "h5py", "plyfile",
    "transforms3d", "transforms3d.axangles", "transforms3d.euler", "imageio", "matplotlib",
    "matplotlib.pyplot", "matplotlib.lines", "matplotlib.cm", "tensorboardX", "lpips", "inplace_abn",
    "sklearn", "sklearn.decomposition", "sklearn.manifold", "tensorflow", "ipdb", "cv2",
]


class _Anything:
    """Placeholder for names imported from stubbed packages; never called on the rendering path."""
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        raise RuntimeError("stubbed third-party symbol was called")


def _make_stub(name):
    mod = types.ModuleType(name)
    mod.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    mod.__path__ = []

    def _getattr(attr):
        if attr.startswith("__"):
            raise AttributeError(attr)
        return _Anything
    mod.__getattr__ = _getattr
    return mod


def _functional_stubs():
    """inplace_abn.ABN / InPlaceABN and kornia.utils.create_meshgrid as plain torch code (SURVEY.md section 8c)."""
    import torch
    import torch.nn as nn
    import torch.nn.functional as F

    class ABN(nn.Module):
        def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, activation="leaky_relu", activation_param=0.01):
            super().__init__()
            self.eps, self.momentum, self.slope = eps, momentum, activation_param
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
            self.register_buffer("running_mean", torch.zeros(num_features))
            self.register_buffer("running_var", torch.ones(num_features))

        def forward(self, x):
            x = F.batch_norm(x, self.running_mean, self.running_var, self.weight, self.bias, self.training, self.momentum, self.eps)
            return F.leaky_relu(x, self.slope)

    def ours(mod):
        return mod is not None and getattr(mod, "__spec__", None) is not None and mod.__spec__.loader is None

    abn = sys.modules.get("inplace_abn")
    if ours(abn):
        abn.ABN = ABN
        abn.InPlaceABN = ABN

    def create_meshgrid(height, width, normalized_coordinates=True, device=None, dtype=torch.float32):
        assert not normalized_coordinates
        xs = torch.linspace(0, width - 1, width, device=device, dtype=dtype)
        ys = torch.linspace(0, height - 1, height, device=device, dtype=dtype)
        gy, gx = torch.meshgrid(ys, xs, indexing="ij")
        return torch.stack([gx, gy], -1)[None]

    ku = sys.modules.get("kornia.utils")
    if ours(ku):
        ku.create_meshgrid = create_meshgrid


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "network"))


def load_reference():
    """Returns the reference's `network.renderer` module (imports it under stubs)."""
    if not available():
        raise RuntimeError("reference tree not found at %s" % REFERENCE_ROOT)
    import torch
    for name in _STUBS:
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                sys.modules[name] = _make_stub(name)
    _functional_stubs()
    if not torch.cuda.is_available():
        _orig_to = torch.Tensor.to

        def _to(self, *args, **kwargs):
            if args and isinstance(args[0], str) and args[0].startswith("cuda"):
                args = args[1:]
                if not args and not kwargs:
                    return self
            return _orig_to(self, *args, **kwargs)
        torch.Tensor.to = _to
        torch.Tensor.cuda = lambda self, *a, **k: self          # init_net.py:219-220 builds buffers with .cuda()
        torch.cuda.synchronize = lambda *a, **k: None           # init_net.py:149-150
        torch.cuda.empty_cache = lambda *a, **k: None
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    cwd = os.getcwd()
    os.chdir(REFERENCE_ROOT)  # the reference opens relative paths (configs/, network/mvsnet/*.ckpt)
    try:
        import network.renderer as ref_renderer
    finally:
        os.chdir(cwd)
    return ref_renderer

"""LPIPS with the VGG16 network on sm_90a (csrc/lpips.cu): the value lpipsPyTorch's lpips(x, y, net_type='vgg') returns,
which render_hierarchy.py reports beside PSNR and SSIM.

The weights are loaded and packed once (LpipsVGG.from_state_dicts / from_torch_hub), not per call as lpips() does, and
never downloaded.  The conv stack runs on TF32 tensor cores with fp32 accumulation -- the arithmetic class of torch's
default cuDNN convolutions, which the reference's published numbers come from.  Nothing here synchronises the host.
"""
import ctypes as C
import os

import torch

from . import _lib

CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)          # vgg16().features indices of the 13 convs
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
                 (512, 512), (512, 512), (512, 512), (512, 512))
TAP_CHANNELS = (64, 128, 256, 512, 512)
VGG_FILE, LIN_FILE = "vgg16-397923af.pth", "vgg.pth"       # what torchvision and lpipsPyTorch cache under torch.hub


def _checked(sd, key, shape):
    if key not in sd:
        raise ValueError(f"missing key {key!r}")
    t = sd[key]
    if not isinstance(t, torch.Tensor) or not t.is_floating_point() or tuple(t.shape) != shape:
        got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{key!r}: expected a float tensor of shape {shape}, got {got}")
    return t.detach().to("cpu", torch.float32).contiguous()


def checked_weights(vgg_features_sd, lin_sd):
    """Validate the two state dicts -> (13 conv weights, 13 biases, 5 linear weights [C]) as CPU fp32 tensors.
    vgg_features_sd: torchvision's vgg16 state dict (keys features.N.weight / .bias; other keys are ignored) or
    vgg16().features' own (keys N.weight / .bias); lin_sd: LPIPS' vgg.pth (keys lin{k}.model.1.weight [1,C,1,1]).
    Raises ValueError naming the first missing or malformed key."""
    prefix = "features." if any(str(k).startswith("features.") for k in vgg_features_sd) else ""
    convs, biases = [], []
    for i, (ci, co) in zip(CONV_INDICES, CONV_CHANNELS):
        convs.append(_checked(vgg_features_sd, f"{prefix}{i}.weight", (co, ci, 3, 3)))
        biases.append(_checked(vgg_features_sd, f"{prefix}{i}.bias", (co,)))
    lins = [_checked(lin_sd, f"lin{k}.model.1.weight", (1, c, 1, 1)).reshape(c) for k, c in enumerate(TAP_CHANNELS)]
    return convs, biases, lins


def pack(L, convs, biases, lins):
    """the kernels' packed weight buffer (CPU fp32) through h3dgs_lpips_pack_weights of library L"""
    out = torch.empty(int(L.h3dgs_lpips_weight_floats()), dtype=torch.float32)
    arr = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    if L.h3dgs_lpips_pack_weights(arr(convs), arr(biases), arr(lins), out.data_ptr()) < 0:
        raise RuntimeError(L.h3dgs_last_error().decode())
    return out


def _frame(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise ValueError(f"{name}: a CUDA float32 tensor is needed")
    if t.dim() == 4 and t.shape[0] == 1:
        t = t[0]
    if t.dim() != 3 or t.shape[0] != 3:
        raise ValueError(f"{name}: shape [3,H,W] or [1,3,H,W] is needed, got {tuple(t.shape)}")
    return t.contiguous()


class LpipsVGG:
    """net(x, y) -> the [1,1,1,1] float64 value of lpips(x, y, 'vgg').  Scratch buffers are held per frame size."""

    def __init__(self, weights):
        """weights: the packed device buffer (see from_state_dicts)"""
        self.L = _lib.lib()
        self.weights = weights
        self.dev = weights.device
        self._scratch = {}

    @classmethod
    def from_state_dicts(cls, vgg_features_sd, lin_sd, device="cuda"):
        return cls(pack(_lib.lib(), *checked_weights(vgg_features_sd, lin_sd)).to(device))

    @classmethod
    def from_torch_hub(cls, device="cuda"):
        """The two files the reference's own LPIPS('vgg') caches under torch.hub.get_dir()/checkpoints; never downloads."""
        sds = []
        for name in (VGG_FILE, LIN_FILE):
            path = os.path.join(torch.hub.get_dir(), "checkpoints", name)
            if not os.path.isfile(path):
                raise FileNotFoundError(f"{path} is missing: it is cached there by the reference's first LPIPS('vgg') run")
            sds.append(torch.load(path, map_location="cpu", weights_only=True))
        return cls.from_state_dicts(*sds, device=device)

    def scratch(self, H, Wc):
        """-> dict(act, taps, partials): the device buffers of an H x Wc network input (allocated on first use)"""
        H, Wc = int(H), int(Wc)
        if min(H, Wc) < _lib.LPIPS_MIN_SIZE:
            raise ValueError(f"LPIPS needs at least {_lib.LPIPS_MIN_SIZE} pixels per side, got {H} x {Wc}: "
                             "a smaller frame leaves a zero-size pooling level")
        if (H, Wc) not in self._scratch:
            a, t, p = C.c_int64(), C.c_int64(), C.c_int64()
            _lib.check(self.L.h3dgs_lpips_scratch_floats(H, Wc, C.byref(a), C.byref(t), C.byref(p)))
            f = lambda n, dt: torch.empty(n, dtype=dt, device=self.dev)
            self._scratch[(H, Wc)] = dict(act=f(a.value, torch.float32), taps=f(t.value, torch.float32),
                                          partials=f(p.value, torch.float64))
        return self._scratch[(H, Wc)]

    def features(self, frame, x0=0, exposure=None, mask=None, clamp=False, stream=None):
        """the target side: frame [3,H,W]'s taps into scratch(H, W - x0)["taps"] (clamp: the evaluator's preprocessing,
        see include/h3dgs.h)"""
        H, W = frame.shape[-2:]
        s = self.scratch(H, W - x0)
        _lib.check(self.L.h3dgs_lpips_features(H, W, x0, frame.data_ptr(), _lib.ptr(exposure), _lib.ptr(mask), int(clamp),
                                               self.weights.data_ptr(), s["act"].data_ptr(), s["taps"].data_ptr(),
                                               self._stream(stream)))

    def distance(self, frame, out, x0=0, exposure=None, mask=None, clamp=False, counter=None, stream=None):
        """the image side against the stored taps: the value goes to out[*counter - 1] (out[0] without a counter)"""
        H, W = frame.shape[-2:]
        s = self.scratch(H, W - x0)
        _lib.check(self.L.h3dgs_lpips_distance(H, W, x0, frame.data_ptr(), _lib.ptr(exposure), _lib.ptr(mask), int(clamp),
                                               self.weights.data_ptr(), s["act"].data_ptr(), s["taps"].data_ptr(),
                                               s["partials"].data_ptr(), _lib.ptr(counter), out.data_ptr(), out.numel(),
                                               self._stream(stream)))

    def _stream(self, stream):
        return torch.cuda.current_stream(self.dev).cuda_stream if stream is None else stream

    def __call__(self, x, y):
        x, y = _frame(x, "x"), _frame(y, "y")
        if x.shape != y.shape:
            raise ValueError(f"x and y differ in shape: {tuple(x.shape)} and {tuple(y.shape)}")
        out = torch.empty(1, dtype=torch.float64, device=self.dev)
        self.features(y)
        self.distance(x, out)
        return out.view(1, 1, 1, 1)

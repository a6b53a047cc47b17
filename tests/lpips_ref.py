"""float64 restatement of LPIPS with the VGG16 network (lpipsPyTorch v0.1, net_type='vgg'), written from its description
(DESIGN.md §3), on the CPU with torch float64 conv2d; and the seeded weights every LPIPS test uses.

  z = (x - mean) / std on the [0,1] input as it is; vgg16().features[0..29] (13 conv3x3 pad 1 + ReLU, max-pool 2x2/2
  before conv 3, 5, 8, 11); taps after conv 2, 4, 7, 10, 13; per tap n = f / (sqrt(sum_c f^2) + 1e-10),
  d = sum_c lin_c (n_x - n_y)^2, its mean over the tap's pixels; the value is the sum of the five means.
"""
import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
                 (512, 512), (512, 512), (512, 512), (512, 512))
TAP_CHANNELS = (64, 128, 256, 512, 512)
POOL_BEFORE = (2, 4, 7, 10)
TAP_AFTER = (1, 3, 6, 9, 12)
MEAN = torch.tensor([-.030, -.088, -.188], dtype=torch.float32)       # the fp32 buffers of the reference's BaseNet
STD = torch.tensor([.458, .448, .450], dtype=torch.float32)
MIN_SIZE = 16


def seeded_state_dicts(seed):
    """(torchvision vgg16 state dict with the features keys, LPIPS vgg.pth state dict) of the given seed: He-scaled
    normal conv weights (activations stay O(1) through the 13 layers), small biases, non-negative linear weights"""
    g = torch.Generator().manual_seed(seed)
    vgg = {}
    for i, (ci, co) in zip(CONV_INDICES, CONV_CHANNELS):
        vgg[f"features.{i}.weight"] = torch.randn((co, ci, 3, 3), generator=g) * math.sqrt(2.0 / (9 * ci))
        vgg[f"features.{i}.bias"] = torch.randn((co,), generator=g) * 0.05
    lin = {f"lin{k}.model.1.weight": torch.rand((1, c, 1, 1), generator=g) * (8.0 / c) for k, c in enumerate(TAP_CHANNELS)}
    return vgg, lin


def checksum(vgg, lin):
    """sha256 of every weight's fp32 bytes, in key order"""
    h = hashlib.sha256()
    for sd in (vgg, lin):
        for k in sorted(sd):
            h.update(k.encode())
            h.update(np.ascontiguousarray(sd[k].numpy().astype(np.float32)).tobytes())
    return h.hexdigest()


def z_score(x):
    """x [3,H,W] -> float64 network input (the fp32 constants, widened)"""
    return (x.double() - MEAN.double()[:, None, None]) / STD.double()[:, None, None]


def conv_layer(x, w, b, with_bound=False):
    """one conv3x3 + bias + ReLU in float64 on x [C,H,W]; with_bound also returns the per-element sum |w||x| + |b| (the
    scale of its rounding errors; ReLU is 1-Lipschitz, so a bound before it holds after it)"""
    x, w, b = x.double()[None], w.double(), b.double()
    y = F.relu(F.conv2d(x, w, b, padding=1))[0]
    if not with_bound:
        return y
    return y, (F.conv2d(x.abs(), w.abs(), padding=1) + b.abs()[:, None, None])[0]


def features(x, vgg):
    """x: the z-scored input [3,H,W] -> the five taps [C_k,H_k,W_k] (float64)"""
    if min(x.shape[-2:]) < MIN_SIZE:
        raise ValueError(f"a {x.shape[-2]} x {x.shape[-1]} input leaves a zero-size pooling level")
    taps = []
    for l, i in enumerate(CONV_INDICES):
        if l in POOL_BEFORE:
            x = F.max_pool2d(x[None], 2)[0]
        x = conv_layer(x, vgg[f"features.{i}.weight"], vgg[f"features.{i}.bias"])
        if l in TAP_AFTER:
            taps.append(x)
    return taps


def normalize(f):
    return f / (torch.sqrt((f * f).sum(0, keepdim=True)) + 1e-10)


def head(tx, ty, lin):
    """-> the five per-tap means (float64)"""
    out = []
    for k, (a, b) in enumerate(zip(tx, ty)):
        w = lin[f"lin{k}.model.1.weight"].double().reshape(-1, 1, 1)
        out.append(float((w * (normalize(a.double()) - normalize(b.double())) ** 2).sum(0).mean()))
    return out


def head_bound(tx, ty, lin):
    """-> per tap: a bound on |fp32 head - float64 head| of the tap mean.  With e = n_x - n_y, |e_c| <= |n_x,c| + |n_y,c|:
    each norm's sum of C squares, sqrt and division cost (C / 2 + 3) 2^-24 relative, so e is off by at most
    (|n_x| + |n_y|)(C / 2 + 3) 2^-24 and 2 |e| de by (C + 6) 2^-24 (|n_x| + |n_y|)^2; the weighted sum of C terms adds
    (C + 1) 2^-24 of sum |w| e^2.  Together (2C + 8) 2^-24 sum_c |w_c| (|n_x,c| + |n_y,c|)^2, averaged over the pixels."""
    out = []
    for k, (a, b) in enumerate(zip(tx, ty)):
        C = a.shape[0]
        w = lin[f"lin{k}.model.1.weight"].double().abs().reshape(-1, 1, 1)
        s = (w * (normalize(a.double()).abs() + normalize(b.double()).abs()) ** 2).sum(0).mean()
        out.append(float((2 * C + 8) * 2.0 ** -24 * s))
    return out


def lpips(x, y, vgg, lin):
    """lpips(x, y, 'vgg') of two [3,H,W] frames in float64 -> (five tap means, value)"""
    t = head(features(z_score(x), vgg), features(z_score(y), vgg), lin)
    return t, sum(t)


def preprocess(raw, mask=None, crop=False):
    """render_hierarchy.py's pair preprocessing without an exposure: clamp to [0,1], the right half when crop, times the
    mask [H,W] (cropped alike)"""
    v = raw.clamp(0.0, 1.0)
    if crop:
        v = v[..., v.shape[-1] // 2:]
    if mask is not None:
        v = v * (mask[..., mask.shape[-1] // 2:] if crop else mask)
    return v


def split_taps(flat, H, Wc):
    """the library's tap buffer (NHWC [H_k][W_k][C_k], one tap after the other) -> five [C_k,H_k,W_k] tensors"""
    flat = torch.as_tensor(flat)
    out, off = [], 0
    for k, C in enumerate(TAP_CHANNELS):
        h, w = H >> k, Wc >> k
        out.append(flat[off:off + h * w * C].reshape(h, w, C).permute(2, 0, 1))
        off += h * w * C
    return out


def layer_budget(K, bound):
    """|fp32 TF32 conv - float64 conv| <= (2^-10 + 2^-21 + (K + 1) 2^-23) (sum |w||x| + |b|): each operand rounded to
    TF32 (2^-11 relative, so a product is off by at most 2^-10 + 2^-22), then K products and the bias summed in fp32"""
    return (2.0 ** -10 + 2.0 ** -21 + (K + 1) * 2.0 ** -23) * bound

"""Plain-PyTorch implementations of every Caffe op with Caffe's exact semantics.

These serve three purposes: (1) the CPU path (LeNet plumbing config), (2) the
"vendor" GPU baseline (cuDNN/cuBLAS through PyTorch) that the sm_90a kernels are
measured against, (3) the fp32 numerical oracle for every hand-written CUDA kernel.

Semantics follow SURVEY.md Appendix A; file:line citations are on each function.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F


# ---- convolution / inner product ---------------------------------------------------
def conv2d(x, w, b, stride, pad, groups):
    """reference: src/caffe/layers/conv_layer.cpp:114-155 (floor output size), conv_layer.cu:13-44."""
    return F.conv2d(x, w.to(x.dtype), None if b is None else b.to(x.dtype), stride, pad, 1, groups)


def inner_product(x, w, b):
    """top = X·Wᵀ + b with X flattened to (M, K). reference: inner_product_layer.cpp:84-95."""
    x2 = x.reshape(x.shape[0], -1)
    return F.linear(x2, w.to(x.dtype), None if b is None else b.to(x.dtype))


# ---- pooling -------------------------------------------------------------------------
def pool_out_size(h, k, s, p):
    """ceil((H+2p-k)/s)+1, minus one if the last window starts in the padding.
    reference: src/caffe/layers/pooling_layer.cpp:72-87."""
    o = int(math.ceil(float(h + 2 * p - k) / s)) + 1
    if p > 0 and (o - 1) * s >= h + p:
        o -= 1
    return o


def max_pool(x, kernel, stride, pad, return_mask=False):
    """MAX pooling; mask is the argmax index h*W+w inside the (n,c) plane.
    reference: src/caffe/layers/pooling_layer.cu:12-47."""
    out = F.max_pool2d(x, kernel, stride, pad, ceil_mode=True, return_indices=return_mask)
    if return_mask:
        y, idx = out
        return y, idx.to(x.dtype)
    return out


def ave_pool(x, kernel, stride, pad):
    """AVE pooling, divisor = window clipped to the *padded* extent.
    reference: src/caffe/layers/pooling_layer.cu:50-78."""
    return F.avg_pool2d(x, kernel, stride, pad, ceil_mode=True, count_include_pad=True)


def _pool_windows(x, kernel, stride):
    """(N, C, OH, OW, kh*kw) windows with -inf/0 padding on the ceil overhang (no pad)."""
    n, c, h, w = x.shape
    kh, kw = kernel
    sh, sw = stride
    oh, ow = pool_out_size(h, kh, sh, 0), pool_out_size(w, kw, sw, 0)
    need_h, need_w = (oh - 1) * sh + kh, (ow - 1) * sw + kw
    xp = F.pad(x, (0, max(0, need_w - w), 0, max(0, need_h - h)))
    cols = F.unfold(xp, (kh, kw), stride=(sh, sw))            # (N, C*kh*kw, OH*OW)
    cols = cols.view(n, c, kh * kw, oh, ow).permute(0, 1, 3, 4, 2)
    return cols, oh, ow


def stochastic_pool(x, kernel, stride, train: bool, generator=None):
    """train: sample an element with probability ∝ activation; test: Σx²/Σx.
    reference: src/caffe/layers/pooling_layer.cu:81-150 (no padding allowed)."""
    cols, oh, ow = _pool_windows(x, kernel, stride)
    s = cols.sum(-1)
    if not train:
        return (cols * cols).sum(-1) / s.clamp_min(torch.finfo(x.dtype).tiny)
    thresh = torch.rand(s.shape, device=x.device, dtype=x.dtype, generator=generator) * s
    cum = cols.cumsum(-1)
    idx = (cum < thresh.unsqueeze(-1)).sum(-1).clamp_max(cols.shape[-1] - 1)
    return cols.gather(-1, idx.unsqueeze(-1)).squeeze(-1)


# ---- LRN -----------------------------------------------------------------------------
def lrn_across(x, size, alpha, beta):
    """scale = 1 + (α/n)·Σ_{window} x²; y = x·scale^{-β}; window pre_pad=(n-1)/2.
    reference: src/caffe/layers/lrn_layer.cu:10-53,73-78; lrn_layer.cpp:112-155."""
    n, c, h, w = x.shape
    sq = (x * x).unsqueeze(1)                                   # (N,1,C,H,W)
    pre = (size - 1) // 2
    sq = F.pad(sq, (0, 0, 0, 0, pre, size - 1 - pre))
    ssum = F.avg_pool3d(sq, (size, 1, 1), stride=1).squeeze(1) * size
    scale = 1.0 + (alpha / size) * ssum
    return x * scale.pow(-beta)


def lrn_within(x, size, alpha, beta):
    """Split → x² → AVE-pool(k=n,pad=(n-1)/2) → (1+α·s)^{-β} → PROD.
    reference: src/caffe/layers/lrn_layer.cpp:20-69,159-165."""
    pre = (size - 1) // 2
    s = ave_pool(x * x, (size, size), (1, 1), (pre, pre))
    s = s[..., : x.shape[2], : x.shape[3]]
    return x * (1.0 + alpha * s).pow(-beta)


# ---- neurons -------------------------------------------------------------------------
def relu(x, negative_slope=0.0):
    """reference: src/caffe/layers/relu_layer.cu:10-42."""
    return F.relu(x) if negative_slope == 0 else F.leaky_relu(x, negative_slope)


def bnll(x):
    """log(1+eˣ) in the overflow-safe form. reference: src/caffe/layers/bnll_layer.cpp:19-20."""
    return torch.where(x > 0, x + torch.log1p(torch.exp(-x)), torch.log1p(torch.exp(x)))


def power(x, pw, scale, shift):
    """(shift + scale·x)^power. reference: src/caffe/layers/power_layer.cpp:22-45."""
    y = x * scale + shift if (scale != 1 or shift != 0) else x
    if pw == 1:
        return y
    if pw == 2:
        return y * y
    return y.pow(pw)


def dropout(x, ratio, train, generator=None):
    """train: y = x·mask/(1-p); test: identity. reference: dropout_layer.cpp:37-47."""
    if not train or ratio == 0:
        return x
    keep = 1.0 - ratio
    mask = (torch.rand(x.shape, device=x.device, generator=generator) < keep).to(x.dtype)
    return x * mask * (1.0 / keep)


def mvn(x, normalize_variance=True, across_channels=False, eps=1e-10):
    """reference: src/caffe/layers/mvn_layer.cpp:39-69 (eps added to the std)."""
    n, c = x.shape[:2]
    v = x.reshape(n, -1) if across_channels else x.reshape(n * c, -1)
    mean = v.mean(1, keepdim=True)
    out = v - mean
    if normalize_variance:
        var = (v * v).mean(1, keepdim=True) - mean * mean
        out = out / (var.clamp_min(0).sqrt() + eps)
    return out.reshape(x.shape)


# ---- softmax / losses ----------------------------------------------------------------
def softmax(x):
    """softmax over the channel axis per (n, h·w). reference: softmax_layer.cu:88-125."""
    return F.softmax(_f(x), dim=1).to(x.dtype)


_FLT_MIN = 1.17549435e-38


def _f(x: torch.Tensor) -> torch.Tensor:
    """Accumulation dtype: fp32 for bf16/fp16/fp32 activations, fp64 kept (the gradient checker runs in double)."""
    return x if x.dtype == torch.float64 else x.float()


def softmax_loss(x, label, return_prob=False):
    """loss = -Σ log(max(p[label], FLT_MIN)) / (num·spatial).
    reference: src/caffe/layers/softmax_loss_layer.cpp:38-87."""
    xf = _f(x)
    if xf.dim() == 2:
        xf = xf[:, :, None, None]
    n, c, h, w = xf.shape
    prob = F.softmax(xf, dim=1)
    lab = label.reshape(n, 1, h, w).long()
    p = prob.gather(1, lab).clamp_min(_FLT_MIN)
    loss = -(p.log()).sum() / (n * h * w)
    return (loss, prob) if return_prob else loss


def euclidean_loss(a, b):
    """‖a−b‖²/(2N). reference: src/caffe/layers/euclidean_loss_layer.cpp:30-46."""
    d = _f(a - b)
    return (d * d).sum() / (2.0 * a.shape[0])


def hinge_loss(x, label, norm="L1"):
    """reference: src/caffe/layers/hinge_loss_layer.cpp:33-67."""
    xf = _f(x).reshape(x.shape[0], -1)
    sign = torch.ones_like(xf)
    sign.scatter_(1, label.reshape(-1, 1).long(), -1.0)
    m = (1.0 + sign * xf).clamp_min(0)
    if norm == "L1":
        return m.sum() / x.shape[0]
    return (m * m).sum() / x.shape[0]


def sigmoid_cross_entropy_loss(x, target):
    """-Σ[x(t−[x≥0]) − log(1+e^{x−2x[x≥0]})]/N.
    reference: src/caffe/layers/sigmoid_cross_entropy_loss_layer.cpp:47-52."""
    xf = _f(x)
    t = target.to(xf.dtype).reshape(x.shape)
    pos = (xf >= 0).to(xf.dtype)
    l = xf * (t - pos) - torch.log1p(torch.exp(xf - 2 * xf * pos))
    return -l.sum() / x.shape[0]


def multinomial_logistic_loss(prob, label):
    """-Σ log(max(p[label], 1e-20))/N. reference: multinomial_logistic_loss_layer.cpp:29-36."""
    p = _f(prob).reshape(prob.shape[0], -1).gather(1, label.reshape(-1, 1).long())
    return -(p.clamp_min(1e-20).log()).sum() / prob.shape[0]


def infogain_loss(prob, label, H):
    """-Σ_i Σ_j H[l_i,j] log(max(p_ij,1e-20))/N. reference: infogain_loss_layer.cpp:65-73."""
    p = _f(prob).reshape(prob.shape[0], -1).clamp_min(1e-20).log()
    rows = H.to(p.device).to(p.dtype)[label.reshape(-1).long()]
    return -(rows * p).sum() / prob.shape[0]


def contrastive_loss(a, b, sim, margin):
    """(Σ_sim d² + Σ_dis max(m−d²,0))/(2N). reference: contrastive_loss_layer.cpp:46-58."""
    d2 = (_f(a - b).reshape(a.shape[0], -1) ** 2).sum(1)
    s = sim.reshape(-1).to(d2.dtype)
    loss = s * d2 + (1 - s) * (margin - d2).clamp_min(0)
    return loss.sum() / (2.0 * a.shape[0])


def accuracy(x, label, top_k=1):
    """fraction of rows whose label is within the top-k scores. reference: accuracy_layer.cpp:34-66."""
    xf = _f(x).reshape(x.shape[0], -1)
    topk = xf.topk(top_k, dim=1).indices
    hit = (topk == label.reshape(-1, 1).long()).any(1)
    return hit.float().mean()


def argmax(x, top_k=1, out_max_val=False):
    """reference: src/caffe/layers/argmax_layer.cpp:10-60. Output (N, 1|2, top_k, 1)."""
    xf = _f(x).reshape(x.shape[0], -1)
    vals, idx = xf.topk(top_k, dim=1)
    out = idx.float().unsqueeze(1)
    if out_max_val:
        out = torch.cat([out, vals.unsqueeze(1)], dim=1)
    return out.unsqueeze(-1)


def eltwise(xs: Sequence[torch.Tensor], op="SUM", coeffs: Optional[Sequence[float]] = None):
    """reference: src/caffe/layers/eltwise_layer.cpp:12-80."""
    if op == "PROD":
        y = xs[0]
        for t in xs[1:]:
            y = y * t
        return y
    if op == "SUM":
        coeffs = coeffs or [1.0] * len(xs)
        y = xs[0] * coeffs[0] if coeffs[0] != 1 else xs[0]
        for t, c in zip(xs[1:], coeffs[1:]):
            y = y + (t * c if c != 1 else t)
        return y
    y = xs[0]
    for t in xs[1:]:
        y = torch.maximum(y, t)
    return y


def im2col(x, kernel, stride, pad):
    """(N, C·kh·kw, OH, OW). reference: src/caffe/util/im2col.cu:12-40, im2col_layer.cpp."""
    n, c, h, w = x.shape
    kh, kw = kernel
    oh = (h + 2 * pad[0] - kh) // stride[0] + 1
    ow = (w + 2 * pad[1] - kw) // stride[1] + 1
    return F.unfold(x, kernel, padding=pad, stride=stride).view(n, c * kh * kw, oh, ow)


# ---- optimizer steps (the oracle for the fused update kernels) --------------------------
def sgd_step(w, g, h, lr, momentum, decay, l1=False):
    """g += wd·w (L2) | wd·sign(w) (L1); h = lr·g + μ·h; w -= h.
    reference: src/caffe/solver.cpp:815-892, blob.cpp:182-205."""
    if decay:
        g = g + decay * (torch.sign(w) if l1 else w)
    h.mul_(momentum).add_(g, alpha=lr)
    w.sub_(h)


def nesterov_step(w, g, h, lr, momentum, decay, l1=False):
    """h_old=h; h = lr·g + μ·h; step = (1+μ)·h − μ·h_old. reference: solver.cpp:1013-1120."""
    if decay:
        g = g + decay * (torch.sign(w) if l1 else w)
    h_old = h.clone()
    h.mul_(momentum).add_(g, alpha=lr)
    w.sub_((1 + momentum) * h - momentum * h_old)


def adagrad_step(w, g, h, lr, delta, decay, l1=False):
    """H += g²; step = lr·g/(√H + δ). reference: solver.cpp:1240-1364."""
    if decay:
        g = g + decay * (torch.sign(w) if l1 else w)
    h.add_(g * g)
    w.sub_(lr * g / (h.sqrt() + delta))

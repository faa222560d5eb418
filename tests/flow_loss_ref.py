"""fp64 restatement of PWC-Net's multi-scale training objective (unsupervised_detection_b200/flow_train_graph.py, as defined there) and of
TF-Adam with L2 weight decay (cis_adam_l2), in torch on the CPU: the reference the flow-training tests compare the kernels against."""
import math

import torch

from oracle import tf_ops as T

LEVELS = (6, 5, 4, 3, 2)
ALPHAS = (0.32, 0.08, 0.02, 0.01, 0.005)


def level_target(gt, h, w, l, s0=1.0, s1=1.0):
    """g_l = resize_bilinear_legacy(gt, h, w) * (s_c / 2^l) per channel."""
    return T.resize_bilinear_legacy(gt, h, w) * torch.tensor([s0, s1], dtype=gt.dtype) / 2.0 ** l


def rho(d, robust=False, eps=0.01, q=0.4):
    """Per-pixel penalty of d [..., 2]: ||d||_2, or (|d0| + |d1| + eps)^q.  The norm's gradient at d = 0 is 0 (safe sqrt)."""
    if robust:
        return (d.abs().sum(-1) + eps) ** q
    sq = (d * d).sum(-1)
    nz = sq > 0
    return torch.where(nz, torch.sqrt(torch.where(nz, sq, torch.ones_like(sq))), torch.zeros_like(sq))


def level_sums(flows, gt, robust=False, eps=0.01, q=0.4, s0=1.0, s1=1.0):
    """flows: the five level flows [B,h_l,w_l,2], l = 6..2; gt [B,GH,GW,2] -> [B,5] per-sample sums of rho over each level's pixels."""
    out = []
    for l, f in zip(LEVELS, flows):
        g = level_target(gt.to(f.dtype), f.shape[1], f.shape[2], l, s0, s1)
        out.append(rho(f - g, robust, eps, q).sum((1, 2)))
    return torch.stack(out, 1)


def flow_loss(flows, gt, global_batch=None, alphas=ALPHAS, **kw):
    """-> (data term sum_l alpha_l / B sum_b sum rho, the five level terms)."""
    s = level_sums(flows, gt, **kw)
    gb = global_batch or s.shape[0]
    terms = [a * s[:, i].sum() / gb for i, a in enumerate(alphas)]
    return sum(terms), terms


def l2_term(params, gamma=4e-4):
    """(gamma / 2) * sum of ||w||^2 over the variables named */kernel (biases are not decayed)."""
    return 0.5 * gamma * sum((v.double() ** 2).sum() for n, v in params.items() if n.endswith('/kernel'))


def adam_l2_step(params, grads, m, v, t, lr=1e-4, decay=4e-4, b1=0.9, b2=0.999, eps=1e-8):
    """One TF-Adam update (step t, 1-based) of fp64 tensors on grad + decay * w for */kernel, in place; m / v dicts updated."""
    lr_t = lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    for n, w in params.items():
        g = grads[n] + (decay * w if n.endswith('/kernel') else 0.0)
        m[n] = b1 * m.get(n, torch.zeros_like(w)) + (1 - b1) * g
        v[n] = b2 * v.get(n, torch.zeros_like(w)) + (1 - b2) * g * g
        w -= lr_t * m[n] / (v[n].sqrt() + eps)

"""fp64 restatement of the unsupervised PWC-Net fine-tuning objective (cis_unsup_flow_loss in include/cis_b200.h, FlowTrainGraph with
loss='unsupervised'), in torch and differentiable in the flow: the reference the unsupervised-loss tests compare the kernels
and the training step against.  It restates UnFlow's published recipe as defined here; it is not checked against any other
implementation.  Every function runs on the device of its inputs."""
import torch
import torch.nn.functional as F

R = 3                  # census window radius: 7 x 7
OCC_A, OCC_B = 0.01, 0.5


def gray(img):
    """g(I) = 255 (0.2989 R + 0.5870 G + 0.1140 B) of I + 0.5; img [..., 3] in [-0.5, 0.5] -> [...]."""
    x = img + 0.5
    return 255.0 * (0.2989 * x[..., 0] + 0.5870 * x[..., 1] + 0.1140 * x[..., 2])


def directions(img1, img2):
    """(S, T) of the 2B directions: n < B the pairs (img1, img2), n >= B the swapped pairs."""
    return torch.cat([img1, img2]), torch.cat([img2, img1])


def partner(flow):
    """flow [2B, ...] -> the partner direction's flow of each direction (n +- B)."""
    B = flow.shape[0] // 2
    return torch.cat([flow[B:], flow[:B]])


def sample_points(flow):
    """q = (y - F0, x - F1) of every pixel -> (qy, qx), [N,H,W]."""
    N, H, W, _ = flow.shape
    gy, gx = torch.meshgrid(torch.arange(H, dtype=flow.dtype, device=flow.device), torch.arange(W, dtype=flow.dtype, device=flow.device),
                            indexing='ij')
    return gy - flow[..., 0], gx - flow[..., 1]


def dense_image_warp(image, flow):
    """oracle.pwcnet.dense_image_warp on any device: image [N,H,W,C] sampled at q = p - flow, floor clamped to [0, size-2], alpha =
    clip(q - floor, 0, 1) (its gradient passes where 0 <= q - floor <= 1)."""
    N, H, W, C = image.shape
    qy, qx = sample_points(flow)

    def prep(q, size):
        fl = torch.clamp(torch.floor(q), 0.0, float(size - 2))
        return fl.long(), torch.clamp(q - fl, 0.0, 1.0).unsqueeze(-1)
    fy, ay = prep(qy, H)
    fx, ax = prep(qx, W)
    flat = image.reshape(N, H * W, C)

    def gather(yy, xx):
        return torch.gather(flat, 1, (yy * W + xx).reshape(N, H * W, 1).expand(-1, -1, C)).reshape(N, H, W, C)
    tl, tr, bl, br = gather(fy, fx), gather(fy, fx + 1), gather(fy + 1, fx), gather(fy + 1, fx + 1)
    top = ax * (tr - tl) + tl
    bot = ax * (br - bl) + bl
    return ay * (bot - top) + top


def occlusion_terms(f, fh):
    """(|F + F^|^2, 0.01 (|F|^2 + |F^|^2) + 0.5): occluded where the first exceeds the second."""
    return ((f + fh) ** 2).sum(-1), OCC_A * ((f ** 2).sum(-1) + (fh ** 2).sum(-1)) + OCC_B


def mask(flow):
    """M = V (1 - O) of every direction of flow [2B,H,W,2] (fp64) -> (M, V, lhs, rhs), M and V as 0 / 1 doubles."""
    flow = flow.detach()
    H, W = flow.shape[1], flow.shape[2]
    qy, qx = sample_points(flow)
    vis = (qy >= 0) & (qy <= H - 1) & (qx >= 0) & (qx <= W - 1)
    fh = dense_image_warp(partner(flow), flow)
    lhs, rhs = occlusion_terms(flow, fh)
    return (vis & ~(lhs > rhs)).to(flow.dtype), vis.to(flow.dtype), lhs, rhs


def _shift(x, dy, dx):
    """x [N,H,W] read at (y + dy, x + dx), 0 outside, and the 0 / 1 mask of where that is inside."""
    H, W = x.shape[1], x.shape[2]
    xp = F.pad(x, (R, R, R, R))
    ins = F.pad(torch.ones_like(x[:1]), (R, R, R, R))
    sl = (slice(None), slice(R + dy, R + dy + H), slice(R + dx, R + dx + W))
    return xp[sl], ins[sl]


def census(gs, tw):
    """c(p) = sum over the 7x7 offsets d != 0 with p + d inside of e^2 / (0.1 + e^2), e = t(g(S)) - t(T~) -> [N,H,W]."""
    t = lambda v: v / torch.sqrt(0.81 + v * v)
    c = torch.zeros_like(tw)
    for dy in range(-R, R + 1):
        for dx in range(-R, R + 1):
            if dy == 0 and dx == 0:
                continue
            s2, ins = _shift(gs, dy, dx)
            t2, _ = _shift(tw, dy, dx)
            e = t(s2 - gs) - t(t2 - tw)
            c = c + ins * e * e / (0.1 + e * e)
    return c


def psi(c):
    return (c + 0.01) ** 0.4


ROUNDING = 2.0 ** -18      # a second difference at most this fraction of |F(p+e)| + 2|F(p)| + |F(p-e)| counts as 0


def second_difference(a, b, c):
    """a - 2b + c, set to 0 (value and gradient) where it is within the rounding level of fp32 flows."""
    l = a - 2 * b + c
    return torch.where(l.abs() <= ROUNDING * (a.abs() + 2 * b.abs() + c.abs()), torch.zeros_like(l), l)


def smoothness(flow, S):
    """sum over pixels and axes of w_a s_a per direction -> [N]: s_a = sum_c |l_c|, l_c = F_c(p+e) - 2 F_c(p) + F_c(p-e) (second_difference),
    w_a = exp(-10 * mean_RGB |S(p+e) - S(p-e)| / 2), where p +- e_a are inside the frame."""
    ly = second_difference(flow[:, 2:], flow[:, 1:-1], flow[:, :-2])
    wy = torch.exp(-10.0 * (S[:, 2:] - S[:, :-2]).abs().mean(-1) / 2)
    lx = second_difference(flow[:, :, 2:], flow[:, :, 1:-1], flow[:, :, :-2])
    wx = torch.exp(-10.0 * (S[:, :, 2:] - S[:, :, :-2]).abs().mean(-1) / 2)
    return (wy * ly.abs().sum(-1)).sum((1, 2)) + (wx * lx.abs().sum(-1)).sum((1, 2))


def direction_sums(flow, img1, img2, m=None):
    """flow [2B,H,W,2], frames [B,H,W,3] -> (sums [2B,2] = {sum M psi, sum w s}, dict of the per-pixel terms: M, warped T~, c).  m: the
    mask to use in place of the one computed here (M carries no gradient)."""
    S, T = directions(img1.to(flow.dtype), img2.to(flow.dtype))
    if m is None:
        m = mask(flow)[0]
    tw = dense_image_warp(gray(T).unsqueeze(-1), flow)[..., 0]
    c = census(gray(S), tw)
    photo = (m * psi(c)).sum((1, 2))
    return torch.stack([photo, smoothness(flow, S)], 1), dict(M=m, warped=tw, c=c)


def loss(flow, img1, img2, global_batch=None, smooth_weight=3.0, m=None):
    """L = 1 / GB * sum over the 2B directions of (P_n + lambda_s Sm_n), P_n = sum M psi / (H W), Sm_n = sum w s / (H W)."""
    s, _ = direction_sums(flow, img1, img2, m)
    gb = global_batch or flow.shape[0] // 2
    hw = flow.shape[1] * flow.shape[2]
    return (s[:, 0].sum() + smooth_weight * s[:, 1].sum()) / (gb * hw)

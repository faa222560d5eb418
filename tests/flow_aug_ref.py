"""fp64 restatement of the augmentation of supervised PWC-Net training pairs (cis_flow_aug_params / cis_flow_augment, include/cis_b200.h).

The counter hash is restated in uint64, so every draw is the kernel's bit for bit; the parameters and the per-pixel pass are then
evaluated in double.  Parameter rows use the kernel's layout (ROW floats per sample).  tolerances() bounds how far the kernel's fp32
per-pixel pass may lie from augment()."""
import math

import numpy as np

ROW = 32
AUG_DOMAIN = 0x466c6f774175676d
NOISE_DOMAIN = 0x4175674e6f697365
_M = (1 << 64) - 1
EPS = 2.0 ** -24          # fp32 unit roundoff, for the tolerances of the kernel's fp32 positions
# the defaults of flow_train_graph.AUG_RANGES, restated
DEFAULTS = dict(scale=(0.9, 2.0), rotate=(-17.0, 17.0), translate=(-0.2, 0.2), rel_scale=(0.95, 1.05), rel_rotate=(-3.0, 3.0),
                rel_translate=(-0.03, 0.03), color=(0.5, 2.0), contrast=(-0.8, 0.4), brightness=0.2, gamma=(0.7, 1.5), noise=(0.0, 0.04))
NO_PHOTO = dict(color=(1.0, 1.0), contrast=(0.0, 0.0), brightness=0.0, gamma=(1.0, 1.0), noise=(0.0, 0.0))


def hash32(x):
    """The 64-bit MurmurHash3 finaliser truncated to 32 bits, on a Python int."""
    x &= _M
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & _M
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & _M
    x ^= x >> 33
    return x & 0xffffffff


def hash32_np(x):
    """The same on a uint64 array."""
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over='ignore'):
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return (x & np.uint64(0xffffffff)).astype(np.float64)


def f32(v):
    return float(np.float32(v))


def draw(seed, t, g, k):
    return hash32(seed ^ AUG_DOMAIN ^ (t << 40) ^ (g << 10) ^ k)


def uniform(seed, t, g, k):
    return (draw(seed, t, g, k) + 0.5) * 2.0 ** -32


def _rng(r, u):
    lo, hi = f32(r[0]), f32(r[1])
    return lo + (hi - lo) * u


def affine(s, deg, tx, ty, cx, cy):
    """c + t + R(th)(p - c)/s as (r0..r5): q = (r0 x + r1 y + r2, r3 x + r4 y + r5)."""
    th = deg * (math.pi / 180.0)
    sn, cs = math.sin(th), math.cos(th)
    m = [cs / s, -sn / s, 0.0, sn / s, cs / s, 0.0]
    m[2] = cx + tx - (m[0] * cx + m[1] * cy)
    m[5] = cy + ty - (m[3] * cx + m[4] * cy)
    return m


def compose(m1, mr):
    """m1 o mr."""
    return [m1[0] * mr[0] + m1[1] * mr[3], m1[0] * mr[1] + m1[1] * mr[4], m1[0] * mr[2] + m1[1] * mr[5] + m1[2],
            m1[3] * mr[0] + m1[4] * mr[3], m1[3] * mr[1] + m1[4] * mr[4], m1[3] * mr[2] + m1[4] * mr[5] + m1[5]]


def invert(m):
    det = m[0] * m[4] - m[1] * m[3]
    i0, i1, i3, i4 = m[4] / det, -m[1] / det, -m[3] / det, m[0] / det
    return [i0, i1, -(i0 * m[2] + i1 * m[5]), i3, i4, -(i3 * m[2] + i4 * m[5])]


def apply(m, x, y):
    return m[0] * x + m[1] * y + m[2], m[3] * x + m[4] * y + m[5]


def corners_inside(m, H, W):
    w1, h1 = W - 1.0, H - 1.0
    for x, y in ((0.0, 0.0), (w1, 0.0), (0.0, h1), (w1, h1)):
        qx, qy = apply(m, x, y)
        if not (0.0 <= qx <= w1 and 0.0 <= qy <= h1):
            return False
    return True


def geometry(H, W, s=1.0, deg=0.0, t=(0.0, 0.0), s_r=1.0, deg_r=0.0, t_r=(0.0, 0.0)):
    """(T1, T2) of one draw; t, t_r in pixels (x, y)."""
    cx, cy = 0.5 * (W - 1.0), 0.5 * (H - 1.0)
    m1 = affine(s, deg, t[0], t[1], cx, cy)
    return m1, compose(m1, affine(s_r, deg_r, t_r[0], t_r[1], cx, cy))


def row(t1, t2, m=(1.0, 1.0, 1.0), contrast=1.0, beta=0.0, gamma=1.0, sigma=0.0, key=0, attempt=0):
    """One parameter row in the kernel's layout, fp64 (the key as its uint32 value, not its float bits)."""
    r = np.zeros(ROW, dtype=np.float64)
    r[0:6], r[6:12], r[12:18] = t1, t2, invert(t2)
    r[18:21], r[21], r[22], r[23], r[24], r[25], r[26] = m, contrast, beta, gamma, sigma, key, attempt
    return r


def sample_params(ranges, H, W, g, t, seed):
    """The parameter row of global sample g at step t (fp64, before the kernel's rounding to fp32)."""
    a = dict(DEFAULTS, **ranges)
    cx, cy = 0.5 * (W - 1.0), 0.5 * (H - 1.0)
    t1 = t2 = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    att = 64
    for k in range(64):
        u = [uniform(seed, t, g, 8 * k + j) for j in range(8)]
        m1 = affine(_rng(a['scale'], u[0]), _rng(a['rotate'], u[1]), _rng(a['translate'], u[2]) * W, _rng(a['translate'], u[3]) * H, cx, cy)
        mr = affine(_rng(a['rel_scale'], u[4]), _rng(a['rel_rotate'], u[5]), _rng(a['rel_translate'], u[6]) * W,
                    _rng(a['rel_translate'], u[7]) * H, cx, cy)
        m2 = compose(m1, mr)
        if corners_inside(m1, H, W) and corners_inside(m2, H, W):
            t1, t2, att = m1, m2, k
            break
    lc0, lc1 = math.log(f32(a['color'][0])), math.log(f32(a['color'][1]))
    m = [math.exp(lc0 + (lc1 - lc0) * uniform(seed, t, g, 512 + c)) for c in range(3)]
    beta = f32(a['brightness']) * math.sqrt(-2.0 * math.log(uniform(seed, t, g, 516))) * math.cos(2.0 * math.pi * uniform(seed, t, g, 517))
    return row(t1, t2, m, 1.0 + _rng(a['contrast'], uniform(seed, t, g, 515)), beta, _rng(a['gamma'], uniform(seed, t, g, 518)),
               _rng(a['noise'], uniform(seed, t, g, 519)), draw(seed, t, g, 520), att)


def params(ranges, B, H, W, sample_offset, t, seed):
    return np.stack([sample_params(ranges, H, W, sample_offset + b, t, seed) for b in range(B)])


def bilinear(img, qx, qy):
    """dense_image_warp's rule on img [H, W, C] at the float64 points (qx, qy): floor clamped to [0, size-2], fraction to [0, 1]."""
    H, W = img.shape[:2]
    x0 = np.clip(np.floor(qx), 0, W - 2)
    y0 = np.clip(np.floor(qy), 0, H - 2)
    ax = np.clip(qx - x0, 0, 1)[..., None]
    ay = np.clip(qy - y0, 0, 1)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    tl, tr, bl, br = img[y0, x0], img[y0, x0 + 1], img[y0 + 1, x0], img[y0 + 1, x0 + 1]
    top = tl + ax * (tr - tl)
    bot = bl + ax * (br - bl)
    return top + ay * (bot - top)


def noise(key, f, H, W):
    """n ~ N(0, 1) of frame f: [H, W, 3]."""
    i = ((np.uint64(f * H) + np.arange(H, dtype=np.uint64)[:, None, None]) * np.uint64(W) + np.arange(W, dtype=np.uint64)[None, :, None]) \
        * np.uint64(3) + np.arange(3, dtype=np.uint64)[None, None, :]
    base = np.uint64(NOISE_DOMAIN) ^ (np.uint64(key) << np.uint64(32)) ^ (i << np.uint64(1))
    u1 = (hash32_np(base) + 0.5) * 2.0 ** -32
    u2 = (hash32_np(base ^ np.uint64(1)) + 0.5) * 2.0 ** -32
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def photometric(v, r, n):
    """The chain on a sample in [-0.5, 0.5] (fp64 [..., 3]) with row r and the frame's noise n."""
    v = (v + 0.5) * r[18:21]
    v = 0.5 + r[21] * (v - 0.5)
    v = np.clip(v + r[22], 0.0, 1.0) ** r[23]
    return np.clip(v + r[24] * n, 0.0, 1.0) - 0.5


def augment(img1, img2, gt, P):
    """img1, img2 [B, H, W, 3], gt [B, H, W, 2] (PWC-Net order) and parameter rows P [B, ROW] (the key as its uint32 value) ->
    (img1_out, img2_out, gt_out) in fp64."""
    img1, img2, gt = (np.asarray(a, dtype=np.float64) for a in (img1, img2, gt))
    B, H, W = gt.shape[:3]
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    o1, o2, og = np.empty_like(img1), np.empty_like(img2), np.empty_like(gt)
    for b in range(B):
        r = P[b]
        q1x, q1y = apply(r[0:6], x, y)
        q2x, q2y = apply(r[6:12], x, y)
        key = int(r[25])
        o1[b] = photometric(bilinear(img1[b], q1x, q1y), r, noise(key, 0, H, W) if r[24] else 0.0)
        o2[b] = photometric(bilinear(img2[b], q2x, q2y), r, noise(key, 1, H, W) if r[24] else 0.0)
        g = bilinear(gt[b], q1x, q1y)
        p2x, p2y = apply(r[12:18], q1x - g[..., 1], q1y - g[..., 0])        # q + (u, v), (u, v) = (-ch1, -ch0)
        og[b] = np.stack([y - p2y, x - p2x], -1)
    return o1, o2, og


def table_rows(table):
    """A kernel table (fp32 [B, ROW]) as fp64 rows with the key as its uint32 value."""
    t = np.asarray(table, dtype=np.float32)
    P = t.astype(np.float64)
    P[:, 25] = t[:, 25].view(np.uint32).astype(np.float64)
    return P


def lipschitz(a):
    """max |difference| between neighbouring pixels of a [H, W, C] field: its Lipschitz bound per pixel of the bilinear sample."""
    return max(float(np.abs(np.diff(a, axis=0)).max()), float(np.abs(np.diff(a, axis=1)).max()))


def position_error(m, H, W):
    """bound on the fp32 error of r0 x + r1 y + r2 (and the second row) over the grid"""
    return 4 * EPS * max(abs(m[0]) * W + abs(m[1]) * H + abs(m[2]), abs(m[3]) * W + abs(m[4]) * H + abs(m[5]))


def tolerances(img1, img2, gt, r):
    """Per-element tolerances of cis_flow_augment's result for one sample (fp64 img1, img2 [H,W,3], gt [H,W,2], parameter row r) against
    augment(): (frame 1 [H,W,3], frame 2 [H,W,3], flow scalar).  They come from the fp32 rounding of the sample positions."""
    H, W = gt.shape[:2]
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing='ij')
    out = []
    for src, m in ((img1, r[0:6]), (img2, r[6:12])):
        # the sample moves by at most 2 * position error * Lipschitz bound; the affine part of the chain scales it by m_c (1 + kappa),
        # gamma maps the interval around the pre-gamma value; fp32 arithmetic adds a few ulps of 1
        qx, qy = apply(m, x, y)
        s = bilinear(src, qx, qy)
        pre = 0.5 + r[21] * ((s + 0.5) * r[18:21] - 0.5) + r[22]
        e = np.abs(r[21] * r[18:21]) * 2 * position_error(m, H, W) * lipschitz(src) + 1e-6
        g_ = lambda v: np.clip(v, 0, 1) ** r[23]  # noqa: E731
        out.append(g_(pre + e) - g_(pre - e) + 8e-6)
    # flow: q moves by dq; gt at q by 2 dq Lip(gt); T2^-1 scales the sum by its row norm and adds its own rounding; then - p
    dq = position_error(r[0:6], H, W)
    s_max = float(max(W, H) + np.abs(gt).max())
    inv = r[12:18]
    row = max(abs(inv[0]) + abs(inv[1]), abs(inv[3]) + abs(inv[4]))
    out.append(row * (dq + 2 * dq * lipschitz(gt) + 4 * EPS * s_max) + 4 * EPS * (row * s_max + max(abs(inv[2]), abs(inv[5]))) + 2 * EPS * max(W, H))
    return out

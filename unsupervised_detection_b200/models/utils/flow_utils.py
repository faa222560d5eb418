"""Flow visualisation for the TensorBoard images (reference models/utils/flow_utils.py:14-109): the Middlebury colour code
(Baker et al., "A Database and Evaluation Methodology for Optical Flow") as used by `flow_to_image_tf`.  Host side, numpy;
the device path never calls this.  `preprocess_flow_batch` (flow_utils.py:5-12) is the device call of ..functional."""
import numpy as np


def preprocess_flow_batch(flow):
    """Function-level API of the reference (flow_utils.py:5-12); see models/functional.py."""
    from .. import functional
    return functional.preprocess_flow_batch(flow)

# (segment length, channel that ramps, ramp direction, channel held at 255): R->Y->G->C->B->M->R
_SEGMENTS = ((15, 1, +1, 0), (6, 0, -1, 1), (4, 2, +1, 1), (11, 1, -1, 2), (13, 0, +1, 2), (6, 2, -1, 0))


def color_wheel():
    """55x3 hue table of the Middlebury code (flow_utils.py:14-43)."""
    rows = []
    for n, ramp, sign, full in _SEGMENTS:
        seg = np.zeros((n, 3))
        r = np.floor(255.0 * np.arange(n) / n)
        seg[:, full] = 255.0
        seg[:, ramp] = r if sign > 0 else 255.0 - r
        rows.append(seg)
    return np.concatenate(rows, 0)


_WHEEL = color_wheel()


def compute_color(u, v):
    """[H,W] normalised flow components -> [H,W,3] colour in 0..255 (flow_utils.py:47-72): hue from the angle by linear
    interpolation on the wheel, saturation from the radius (desaturate towards white inside the unit circle, x0.75 outside)."""
    nan = np.isnan(u) | np.isnan(v)
    u = np.where(nan, 0.0, u)
    v = np.where(nan, 0.0, v)
    n = _WHEEL.shape[0]
    rad = np.sqrt(u * u + v * v)
    fk = (np.arctan2(-v, -u) / np.pi + 1.0) / 2.0 * (n - 1)          # 0-based position on the wheel
    k0 = np.floor(fk).astype(np.int64)
    k1 = np.where(k0 + 1 >= n, 0, k0 + 1)
    f = (fk - k0)[..., None]
    col = (1.0 - f) * (_WHEEL[k0] / 255.0) + f * (_WHEEL[k1] / 255.0)
    inside = (rad <= 1.0)[..., None]
    col = np.where(inside, 1.0 - rad[..., None] * (1.0 - col), col * 0.75)
    return np.float64(np.uint8(np.floor(255.0 * col * (1 - nan)[..., None])))


def flow_to_image(flow):
    """[B,H,W,2] -> float32 [B,H,W,3] in 0..255 (flow_utils.py:74-100).  Like the reference, the normalising radius is the
    running maximum over the batch elements seen so far (element i is scaled by max_{j<=i} |flow_j|)."""
    out, maxrad = [], -1.0
    for i in range(flow.shape[0]):
        u = np.array(flow[i, :, :, 0])                         # input precision (fp32): the radius and its maximum are
        v = np.array(flow[i, :, :, 1])                         # rounded like the reference's, the division is in fp64
        unknown = (np.abs(u) > 1e7) | (np.abs(v) > 1e7)
        u[unknown] = 0
        v[unknown] = 0
        maxrad = max(maxrad, np.max(np.sqrt(u * u + v * v)))
        s = np.float64(maxrad) + np.finfo(float).eps
        out.append(compute_color(u.astype(np.float64) / s, v.astype(np.float64) / s))
    return np.float32(np.uint8(out))


def flow_to_image_pm(flow):
    """flow_to_image_tf (flow_utils.py:102-109): colour image shifted to [-0.5, 0.5]."""
    return flow_to_image(flow) / 255.0 - 0.5

"""Reference for tf.image.resize_bilinear with TF 1.13 semantics (SURVEY.md App. A.6 / A.6a), torch-CPU, test infra only; kept apart
from the product code it checks.  The step in -> out is taken in fp32, as TF 1.13 does: (in-1)/(out-1) with align_corners and out > 1
(any step when out = 1: dst 0 reads src 0, so 0 is used), else in/out; src = dst * step in fp32, lo = floor(src), hi = min(lo+1, in-1),
weights from the fp32 fraction.  oracle.tf_ops.resize_bilinear_legacy takes the legacy step in fp64, which differs by up to ~1e-5 of
the values where in/out is not a binary fraction (53 -> 20); its call sites resize by exact ratios."""
import torch


def resize_bilinear(x, out_h, out_w, align_corners):
    """x: NHWC tensor (any float dtype; the interpolation runs in that dtype) -> [N, out_h, out_w, C]."""

    def axis(n_in, n_out):
        if align_corners:
            step = torch.tensor(n_in - 1, dtype=torch.float32) / (n_out - 1) if n_out > 1 else torch.tensor(0.0)
        else:
            step = torch.tensor(n_in, dtype=torch.float32) / n_out
        src = torch.arange(n_out, dtype=torch.float32) * step
        lo = torch.floor(src)
        return lo.long(), torch.clamp(lo.long() + 1, max=n_in - 1), (src - lo).to(x.dtype)

    (hl, hh, hf), (wl, wh, wf) = axis(x.shape[1], out_h), axis(x.shape[2], out_w)
    top, bot = x[:, hl], x[:, hh]
    hf, wf = hf.view(1, -1, 1, 1), wf.view(1, 1, -1, 1)
    t = top[:, :, wl] + (top[:, :, wh] - top[:, :, wl]) * wf
    b = bot[:, :, wl] + (bot[:, :, wh] - bot[:, :, wl]) * wf
    return t + (b - t) * hf

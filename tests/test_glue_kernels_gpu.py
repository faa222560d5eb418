"""cis_resize_concat_bf16 and its transpose, bit for bit, against a host restatement of the kernels' arithmetic in the same order.

On the exact x2 and same-resolution paths every product is by 0, 0.25, 0.5 or 1, so it is exact and a fused multiply-add rounds like
the separate multiply and add of the restatement; bf16 rounding is round-to-nearest-even on both sides.  The cases cover one to four
sources, a batch-broadcast source (n_mod), odd sizes, one-pixel rows / columns, slices at channel offsets, and, for the transpose,
unwanted sources and accumulation onto an existing gradient."""
import ctypes as C

import pytest
import torch

from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200._lib import CisSrc

pytestmark = pytest.mark.gpu
ST = lambda: torch.cuda.current_stream().cuda_stream


def bf16_randn(*shape, gen):
    return torch.randn(*shape, generator=gen).to(torch.bfloat16)


def ref_resize(x, OH, OW):
    """The kernels' legacy bilinear resize of x [n, H, W, C] (fp32 holding bf16 values) to OH = H or 2H, OW = W or 2W, fp32."""
    n, H, W, c = x.shape
    if (OH, OW) == (H, W):
        return x.clone()
    assert (OH, OW) == (2 * H, 2 * W)
    y1 = torch.clamp(torch.arange(H) + 1, max=H - 1)
    x1 = torch.clamp(torch.arange(W) + 1, max=W - 1)
    s00, s01, s10 = x, x[:, :, x1], x[:, y1]
    s11 = s10[:, :, x1]
    out = torch.empty(n, OH, OW, c)
    for qy in (0, 1):
        for qx in (0, 1):
            fy, fx = 0.5 * qy, 0.5 * qx
            tp = s00 + (s01 - s00) * fx
            bo = s10 + (s11 - s10) * fx
            out[:, qy::2, qx::2] = tp + (bo - tp) * fy
    return out


def ref_resize_t(d, H, W, acc, reps, n_mod):
    """Transpose for one source: d [N, OH, OW, C] fp32, acc [rows, H, W, C] fp32 start value; rows are summed over replicas r in order
    inside every window position, window rows then columns in ascending order, as the kernel does."""
    N, OH, OW, c = d.shape
    rows = acc.shape[0]
    acc = acc.clone()
    if (OH, OW) == (H, W):
        for r in range(reps):
            acc = acc + d[r * n_mod:r * n_mod + rows]
        return acc
    assert (OH, OW) == (2 * H, 2 * W)
    ys, xs = torch.arange(H), torch.arange(W)
    for j in range(3):
        dy = 2 * ys - 1 + j
        wy = torch.full((H,), 0.5) if j != 1 else torch.ones(H)
        if j == 2:
            wy[H - 1] = 1.0
        for k in range(3):
            dx = 2 * xs - 1 + k
            wx = torch.full((W,), 0.5) if k != 1 else torch.ones(W)
            if k == 2:
                wx[W - 1] = 1.0
            ok = (dy >= 0)[:, None] & (dx >= 0)[None, :]
            wt = (wy[:, None] * wx[None, :])[None, :, :, None]
            for r in range(reps):
                v = d[r * n_mod:r * n_mod + rows][:, dy.clamp(min=0)][:, :, dx.clamp(min=0)]
                acc = torch.where(ok[None, :, :, None], acc + wt * v, acc)
    return acc


# (H, W, OH, OW, N, chans of the sources, n_mod of each source)
CASES = [
    (7, 9, 14, 18, 6, (16, 8, 24, 8), (0, 2, 0, 0)),
    (16, 28, 32, 56, 12, (128, 128, 128, 8), (0, 0, 4, 0)),
    (5, 1, 10, 2, 3, (8,), (0,)),
    (1, 6, 2, 12, 4, (24, 8), (2, 0)),
    (13, 11, 13, 11, 6, (16, 16, 16, 8), (0, 0, 3, 0)),
    (4, 5, 8, 10, 4, (8, 16, 8), (0, 0, 1)),
]


@pytest.mark.parametrize('H,W,OH,OW,N,chans,nmods', CASES)
def test_resize_concat_bit_exact(H, W, OH, OW, N, chans, nmods):
    gen = torch.Generator().manual_seed(H * 131 + W * 7 + len(chans))
    xs = [bf16_randn(nm or N, H, W, c, gen=gen) for c, nm in zip(chans, nmods)]
    xd = [x.cuda().contiguous() for x in xs]
    tot = sum(chans)
    pitch = tot + 16
    out = torch.zeros(N, OH, OW, pitch, dtype=torch.bfloat16, device='cuda')     # destination slice at channel offset 8
    arr = (CisSrc * len(xs))(*[CisSrc(t.data_ptr(), c, 0, c // 8, nm) for t, c, nm in zip(xd, chans, nmods)])
    _lib.call('cis_resize_concat_bf16', arr, len(xs), N, H, W, out.data_ptr(), pitch, 8, OH, OW, ST())
    torch.cuda.synchronize()
    ref = torch.cat([ref_resize(x.float()[torch.arange(N) % nm] if nm else x.float(), OH, OW) for x, nm in zip(xs, nmods)], 3)
    got = out.cpu()
    assert torch.equal(got[..., 8:8 + tot], ref.to(torch.bfloat16))
    assert float(got[..., :8].abs().max()) == 0 and float(got[..., 8 + tot:].abs().max()) == 0


@pytest.mark.parametrize('H,W,OH,OW,N,chans,nmods', CASES)
def test_resize_concat_transpose_bit_exact(H, W, OH, OW, N, chans, nmods):
    gen = torch.Generator().manual_seed(H * 17 + W * 3 + len(chans))
    ns = len(chans)
    tot = sum(chans)
    dp = tot + 8
    d = bf16_randn(N, OH, OW, tot, gen=gen)
    dd = torch.zeros(N, OH, OW, dp, dtype=torch.bfloat16)
    dd[..., 8:] = d
    dd = dd.cuda()
    # source i: wanted unless it is the third of four; accumulated when i is odd; gradient slice at channel offset 8 of a wider buffer
    want = [0 if (ns == 4 and i == 2) else 1 for i in range(ns)]
    acc = [i % 2 for i in range(ns)]
    pre = [bf16_randn(nm or N, H, W, c + 16, gen=gen) for c, nm in zip(chans, nmods)]
    grads = [p.cuda().contiguous() for p in pre]
    ga = (CisSrc * ns)(*[CisSrc(t.data_ptr(), c + 16, 8, c // 8, nm) for t, c, nm in zip(grads, chans, nmods)])
    _lib.call('cis_resize_concat_bf16_bwd', dd.data_ptr(), dp, 8, N, OH, OW, ga, (C.c_int32 * ns)(*want), (C.c_int32 * ns)(*acc), ns, H, W,
              ST())
    torch.cuda.synchronize()
    c0 = 0
    for i, (c, nm) in enumerate(zip(chans, nmods)):
        got = grads[i].cpu()
        assert torch.equal(got[..., :8], pre[i][..., :8]) and torch.equal(got[..., 8 + c:], pre[i][..., 8 + c:])
        if not want[i]:
            assert torch.equal(got, pre[i])
        else:
            start = pre[i][..., 8:8 + c].float() if acc[i] else torch.zeros(nm or N, H, W, c)
            ref = ref_resize_t(d[..., c0:c0 + c].float(), H, W, start, N // nm if nm else 1, nm or N)
            assert torch.equal(got[..., 8:8 + c], ref.to(torch.bfloat16)), i
        c0 += c

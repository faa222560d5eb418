"""The train step's fused loss head and optimiser kernels (csrc/misc_kernels.cu) against an fp64 reference of the same operation.

The reference of the loss algebra is oracle.losses.loss_head evaluated in float64, with torch.autograd for every backward coefficient;
the upsample of `flow1` is tests/resize_ref.resize_bilinear, whose step is taken in fp32 like the kernels'.  The networks are left out
(the step-graph tests read the graph's own fp32 `flow`, `mask` and `flow1` back), so the bounds are fp32-level:

- bit-exact: cis_mask_apply, the lanes of cis_mask_bwd, two runs of cis_cis_loss_fwd, the noise branch of cis_clip_adam run twice;
- fp32 elementwise, |err| <= 1e-5 * max|ref| (per slice): pred_out, dpred, the Adam update, m and v;
- dmask, a sum of cancelling terms: |err| <= 1e-5 * (|a e0| + |a_c e1| + |(c - c_q) e2|) per pixel;
- sums, recover loss, 1/(hw GB) and coef: 1e-5 relative; the red-rate terms 1 - rec/den: 1e-6 absolute;
- bf16 outputs: 2^-8 |ref| + 1e-30, plus the fp32 accumulation bound of the kernel (2e-6 * the same sum over |terms|) where its
  result is a sum of terms of both signs: without it a single cancelling pixel fails the relative bf16 bound;
- cis_grad_avg_abs: 2e-5 relative.

dpred and dmask are compared with the reference evaluated at the kernel's own upsampled `pred` (pred_out, itself checked against the fp64
upsample): the Charbonnier derivative has slope 1/sqrt(1e-6) = 1e3 (cbn = 0.5) and ~1e4 (cbn = 0.3) around d = gt - pred = 0, so the
fp32 rounding of pred alone (~3e-8) would move it by 3e-5 .. 5e-5 of its maximum at pixels where the recovered flow is exact.

Measured worst cases on an H100 (80 GB), as a fraction of each bound (run with -s to print them):
- kernel level: pred_out 0.0073, sums 0.0049 (256x448 B=4: 0.00035), coef 0.011, recover loss 0.0054, red-rate terms 0.042,
  dpred 0.025, dmask 0.23, Adam update 0.37 (m 0.010, v 0.0081), grad_avg_abs 0.0088, noise-branch KS distance 0.54;
- bf16 outputs: cis_resize_f32_bwd_to_bf16 0.994, cis_mask_bwd 0.991: round-to-nearest bf16 is off by up to half an ulp = 2^-8 |x| just
  above a power of two, so these bounds are tight by construction and a real error of more than one bf16 ulp fails them;
- step graph: pred 0.0081, sums 0.0011, coef 0.0052, diagnostics 0.0058, red-rate 0.0044, dpred 0.025 (G) / 0.030 (R), dmask 0.043,
  flow1 gradient 0.993 (G) / 0.991 (R), logits gradient 0.984;
- generator-step data-parallel split: scalars 0.097 of 1e-6 relative, 1 - cosine 5e-15, norm ratio exact.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import losses as OL, params as OP
from unsupervised_detection_b200 import _lib
from resize_ref import resize_bilinear

pytestmark = pytest.mark.gpu
ST = lambda: torch.cuda.current_stream().cuda_stream
f32 = lambda v: float(np.float32(v))      # a hyper-parameter as the kernels receive it (fp32 argument)
WORST = {}


def _note(key, ratio):
    """Record err / bound of one check (<= 1 passes) for the measured-worst-case table."""
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


@pytest.fixture(scope='module', autouse=True)
def _print_worst():
    yield
    for k in sorted(WORST):
        print('worst %-28s %.3g of the bound' % (k, WORST[k]))


def _close(key, got, ref, tol):
    """got, ref: tensors; tol: per-element bound (tensor or float).  Asserts |got - ref| <= tol everywhere."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(ref)
    err = (got - ref).abs()
    assert bool(torch.isfinite(got).all()), key
    r = float((err / tol.clamp_min(1e-300)).max())
    _note(key, r)
    assert r <= 1.0, (key, r, float(err.max()), float(ref.abs().max()))


def _rel(key, got, ref, rel):
    _close(key, got, ref, rel * ref.detach().double().cpu().abs())


def _fp32(key, got, ref, rel=1e-5):
    _close(key, got, ref, rel * float(ref.detach().abs().max()))


def _bf16(key, got, ref, fp32_scale=None):
    """bf16 output: 2^-8 |ref| + 1e-30 (+ 2e-6 * fp32_scale, the accumulation bound of an fp32 sum of signed terms)."""
    ref = ref.detach().double().cpu()
    tol = 2.0 ** -8 * ref.abs() + 1e-30
    if fp32_scale is not None:
        tol = tol + 2e-6 * fp32_scale.detach().double().cpu()
    _close(key, got, ref, tol)


def _smooth(B, H, W, C, amp, gen, div=8):
    lo = torch.randn(B, C, max(H // div, 2), max(W // div, 2), generator=gen)
    return (F.interpolate(lo, size=(H, W), mode='bicubic', align_corners=False) * amp).permute(0, 2, 3, 1).contiguous()


def _upsample(flow1, H, W):
    """fp64 reference of the upsample fused into the loss kernels (legacy bilinear, step in fp32)."""
    return resize_bilinear(flow1.detach().double().cpu(), H, W, align_corners=False)


def _adjoint(dd, h1, w1):
    """fp64 transpose of _upsample: dd [N,H,W,C] -> [N,h1,w1,C]."""
    x = torch.zeros(dd.shape[0], h1, w1, dd.shape[3], dtype=torch.float64, requires_grad=True)
    y = resize_bilinear(x, dd.shape[1], dd.shape[2], align_corners=False)
    return torch.autograd.grad(y, x, dd.detach().double().cpu())[0]


def _head(flow, mask, pred3, B, cbn, eps, GB):
    """loss_head in float64 with the mask and the [3B] recovered flows as leaves (grads w.r.t. the mask hold the preds fixed)."""
    H, W = flow.shape[1], flow.shape[2]
    m = mask.detach().double().cpu().reshape(B, H, W, 1).requires_grad_(True)
    p = pred3.detach().double().cpu().requires_grad_(True)
    L = OL.loss_head(flow.detach().double().cpu(), m, p[:B], p[B:2 * B], p[2 * B:], f32(cbn), f32(eps), GB)
    return L, m, p


def _coef_ref(L):
    """[B,4] = d generator / d {rec, den, rec_c, den_c}: the per-sample coefficients of cis_cis_loss_reduce."""
    g = torch.autograd.grad(L['generator'], [L['rec'], L['den'], L['rec_c'], L['den_c']], retain_graph=True)
    return torch.stack(g, dim=1)


def _charb_px(flow, pred, cbn):
    """per-pixel Charbonnier term summed over the two flow channels (scale of the dmask bound only)."""
    return (((flow.double().cpu() - pred) ** 2 + 1e-6) ** f32(cbn)).sum(-1)


def _dmask_scale(flow, p, coef, B, cbn):
    e = [_charb_px(flow, p[j * B:(j + 1) * B].detach(), cbn) for j in range(3)]
    a, c, ac, ccq = (coef[:, k].view(B, 1, 1) for k in range(4))
    return (a * e[0]).abs() + (ac * e[1]).abs() + ((c - ccq) * e[2]).abs()


def _scalars_check(tag, s, L, B, H, W, GB):
    s = s.cpu().double()
    _close(tag + 'red_rate', s[2], L['red_rate'], 1e-6)
    _close(tag + 'red_rate', s[3], L['red_rate_compl'], 1e-6)
    _close(tag + 'red_rate', s[0], L['generator'], 2e-6)
    _rel(tag + 'recover', s[1], L['recover'], 1e-5)
    _rel(tag + 'recover', s[4], torch.tensor(1.0 / (H * W * GB), dtype=torch.float64), 1e-5)


# ---------------------------------------------------------------------------------------------------------------- kernel level
def _loss_inputs(B, H, W, h1, w1, seed, mask_kind='rand'):
    g = torch.Generator().manual_seed(seed)
    flow = _smooth(B, H, W, 2, 0.5, g)
    # recovered flows near the target (as after a few steps) plus their own structure, so d = gt - pred spans 0
    flow1 = torch.cat([F.interpolate(flow.permute(0, 3, 1, 2), size=(h1, w1), mode='area').permute(0, 2, 3, 1)] * 3)
    flow1 = (flow1 + 0.2 * torch.randn(3 * B, h1, w1, 2, generator=g)).contiguous()
    if mask_kind == 'zeros':
        mask = torch.zeros(B, H, W, 1)
    elif mask_kind == 'ones':
        mask = torch.ones(B, H, W, 1)
    else:
        mask = torch.rand(B, H, W, 1, generator=g)
        mask.view(-1)[::7] = 0.0
        mask.view(-1)[3::11] = 1.0
    return flow.cuda(), mask.cuda(), flow1.cuda()


def _run_fwd(flow, mask, flow1, B, H, W, h1, w1, cbn, eps, GB):
    sums = torch.zeros(B, 5, dtype=torch.float64, device='cuda')
    pred = torch.full((3 * B, H, W, 2), float('nan'), device='cuda')
    scalars = torch.full((8,), float('nan'), device='cuda')
    coef = torch.full((B, 4), float('nan'), device='cuda')
    _lib.call('cis_cis_loss_fwd', flow.data_ptr(), mask.data_ptr(), flow1.data_ptr(), B, H, W, h1, w1, cbn, sums.data_ptr(), pred.data_ptr(),
              ST())
    _lib.call('cis_cis_loss_reduce', sums.data_ptr(), B, GB, H * W, eps, scalars.data_ptr(), coef.data_ptr(), ST())
    torch.cuda.synchronize()
    return sums, pred, scalars, coef


def _check_fwd(tag, flow, mask, flow1, B, H, W, h1, w1, cbn, eps, GB):
    sums, pred, scalars, coef = _run_fwd(flow, mask, flow1, B, H, W, h1, w1, cbn, eps, GB)
    pref = _upsample(flow1, H, W)
    for j in range(3):
        _fp32('pred_out', pred[j * B:(j + 1) * B], pref[j * B:(j + 1) * B])
    L, _, _ = _head(flow, mask, pref, B, cbn, eps, GB)
    _rel(tag + 'sums', sums, L['sums'], 1e-5)
    _scalars_check(tag, scalars, L, B, H, W, GB)
    _rel(tag + 'coef', coef, _coef_ref(L), 1e-5)
    return sums


SIZES = [(64, 96, 32, 48), (36, 52, 18, 26), (30, 46, 15, 23), (16, 24, 7, 11), (20, 28, 20, 28)]


def test_mask_apply_is_the_bf16_rounding_of_the_fp32_formulas():
    B, H, W = 3, 37, 53                                                   # 5883 pixels: not a multiple of 256
    g = torch.Generator().manual_seed(1)
    flow = torch.randn(B, H, W, 2, generator=g) * 3
    mask = torch.rand(B, H, W, 1, generator=g)
    mv = mask.view(-1)
    mv[::5], mv[1::7], mv[2::9], mv[3::13] = 0.0, 1.0, 1e-30, 1.0 - 2.0 ** -24
    dst = torch.full((3 * B, H, W, 8), float('nan'), dtype=torch.bfloat16, device='cuda')
    fd, md = flow.cuda(), mask.cuda()
    _lib.call('cis_mask_apply', fd.data_ptr(), md.data_ptr(), B, H * W, dst.data_ptr(), ST())
    torch.cuda.synchronize()
    m, om = mask, 1.0 - mask                                              # fp32 torch arithmetic = the kernel's fp32 expressions
    one, zero = torch.ones_like(m), torch.zeros_like(m)
    want = [torch.cat([flow * om, one, om], -1), torch.cat([flow * m, one, m], -1), torch.cat([zero, zero, one, zero], -1)]
    got = dst.cpu()
    for j in range(3):
        ref = torch.cat([want[j], torch.zeros(B, H, W, 4)], -1).to(torch.bfloat16)
        assert torch.equal(got[j * B:(j + 1) * B].view(torch.int16), ref.view(torch.int16)), j


@pytest.mark.parametrize('eps', [75.0, 0.5])
@pytest.mark.parametrize('cbn', [0.5, 1.0, 0.3])
@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('B,gb_mult', [(1, 1), (1, 2), (3, 1), (3, 2)])
def test_loss_fwd_and_reduce(B, gb_mult, size, cbn, eps):
    H, W, h1, w1 = size
    flow, mask, flow1 = _loss_inputs(B, H, W, h1, w1, seed=H * W + B)
    _check_fwd('', flow, mask, flow1, B, H, W, h1, w1, cbn, eps, B * gb_mult)


@pytest.mark.parametrize('kind', ['zeros', 'ones'])
def test_loss_fwd_with_all_or_nothing_masks(kind):
    """mask = 0: rec = den - eps = 0 (den = eps); mask = 1: rec_c = den_c - eps = 0."""
    B, H, W, h1, w1 = 2, 36, 52, 18, 26
    flow, mask, flow1 = _loss_inputs(B, H, W, h1, w1, seed=5, mask_kind=kind)
    sums = _check_fwd('', flow, mask, flow1, B, H, W, h1, w1, 0.5, 75.0, 2).cpu()
    zero = (0, 3) if kind == 'zeros' else (1, 4)
    assert bool((sums[:, list(zero)] == 0).all())


def test_loss_fwd_bench_size_and_run_to_run_identical_sums():
    """256x448, B = 4: the grid-stride loop gives each thread several pixels (fp32 per-thread accumulation).  The fp64 block atomics
    add fp32-derived values exactly, so two runs on zeroed sums must agree bit for bit (the train step is deterministic)."""
    B, H, W, h1, w1 = 4, 256, 448, 128, 224
    flow, mask, flow1 = _loss_inputs(B, H, W, h1, w1, seed=7)
    s1 = _check_fwd('bench ', flow, mask, flow1, B, H, W, h1, w1, 0.5, 75.0, B)
    s2, _, _, _ = _run_fwd(flow, mask, flow1, B, H, W, h1, w1, 0.5, 75.0, B)
    assert torch.equal(s1.view(torch.int64), s2.view(torch.int64))


@pytest.mark.parametrize('cbn', [0.5, 1.0, 0.3])
@pytest.mark.parametrize('size', SIZES)
@pytest.mark.parametrize('B,GB', [(1, 1), (3, 6)])
@pytest.mark.parametrize('which', [0, 1])
def test_loss_bwd(which, B, GB, size, cbn):
    """which = 0: d recover / d pred for the 3B slices, dmask never written.  which = 1: d generator / d pred and the direct
    d generator / d mask through the sums (preds fixed)."""
    H, W, h1, w1 = size
    eps = 75.0 if B == 1 else 0.5
    flow, mask, flow1 = _loss_inputs(B, H, W, h1, w1, seed=H * W + 17 * B + which)
    _, pred, scalars, coef = _run_fwd(flow, mask, flow1, B, H, W, h1, w1, cbn, eps, GB)
    _fp32('pred_out', pred, _upsample(flow1, H, W))
    dpred = torch.full((3 * B, H, W, 2), float('nan'), device='cuda')
    dmask = torch.full((B, H, W), float('nan'), device='cuda')
    _lib.call('cis_cis_loss_bwd', flow.data_ptr(), mask.data_ptr(), flow1.data_ptr(), coef.data_ptr(), scalars.data_ptr(), B, H, W, h1, w1,
              cbn, which, dpred.data_ptr(), dmask.data_ptr(), ST())
    torch.cuda.synchronize()
    L, m, p = _head(flow, mask, pred, B, cbn, eps, GB)
    loss = L['recover'] if which == 0 else L['generator']
    dp_ref, dm_ref = torch.autograd.grad(loss, [p, m], retain_graph=True, allow_unused=True)
    for j in range(3):
        _fp32('dpred', dpred[j * B:(j + 1) * B], dp_ref[j * B:(j + 1) * B])
    if which == 0:
        assert bool(dmask.isnan().all())
    else:
        _close('dmask', dmask, dm_ref.view(B, H, W), 1e-5 * _dmask_scale(flow, p, _coef_ref(L), B, cbn))


@pytest.mark.parametrize('scale', [None, 0.0125])
@pytest.mark.parametrize('pitch', [8, 24])
@pytest.mark.parametrize('size', SIZES)
def test_resize_f32_bwd_to_bf16(size, pitch, scale):
    """The transpose of the loss's flow1 upsample, stored as bf16 channels [0, 8) of a `pitch`-channel row: 3B rows (recover step)
    and the first 2B rows (generator step); rows and channels it does not own stay untouched."""
    H, W, h1, w1 = size
    B, C = 2, 2
    g = torch.Generator().manual_seed(H + W)
    dd = torch.randn(3 * B, H, W, C, generator=g).cuda()
    for nb in (3 * B, 2 * B):
        ds = torch.full((3 * B, h1, w1, pitch), float('nan'), dtype=torch.bfloat16, device='cuda')
        if scale is None:
            _lib.call('cis_resize_f32_bwd_to_bf16', dd.data_ptr(), nb, H, W, C, h1, w1, ds.data_ptr(), pitch, ST())
        else:
            _lib.call('cis_resize_f32_bwd_to_bf16_scaled', dd.data_ptr(), nb, H, W, C, h1, w1, ds.data_ptr(), pitch, scale, ST())
        torch.cuda.synchronize()
        k = 1.0 if scale is None else f32(scale)
        ref = _adjoint(dd[:nb], h1, w1) * k
        got = ds.cpu().float()
        _bf16('resize_bwd_bf16', got[:nb, ..., :C], ref, _adjoint(dd[:nb].abs(), h1, w1) * k)
        assert bool((got[:nb, ..., C:8] == 0).all())
        assert bool(got[:nb, ..., 8:].isnan().all()) and bool(got[nb:].isnan().all())


@pytest.mark.parametrize('with_din', [False, True])
def test_mask_bwd(with_din):
    """dm = dmask - f . d0[0:2] - d0[3] + f . d1[0:2] + d1[3] on the bf16 gradients the kernel reads, then the softmax chain
    dl = dm m (1 - m) / 10; lane 1 = -lane 0 bit for bit, lanes 2..7 zero."""
    B, H, W = 3, 37, 53
    g = torch.Generator().manual_seed(11 + with_din)
    flow = torch.randn(B, H, W, 2, generator=g)
    mask = torch.rand(B, H, W, 1, generator=g)
    mask.view(-1)[::9] = 0.0
    dmd = torch.randn(B, H, W, generator=g) * 1e-3
    din = (torch.randn(3 * B, H, W, 8, generator=g) * 1e-3).to(torch.bfloat16)
    dl = torch.full((B, H, W, 8), float('nan'), dtype=torch.bfloat16, device='cuda')
    fd, md, gd, dd = flow.cuda(), mask.cuda(), dmd.cuda(), din.cuda()
    _lib.call('cis_mask_bwd', fd.data_ptr(), md.data_ptr(), gd.data_ptr(), dd.data_ptr() if with_din else None, B, H * W, dl.data_ptr(), ST())
    torch.cuda.synchronize()
    got = dl.cpu()
    f, m = flow.double(), mask.double()[..., 0]
    dm, scale = dmd.double(), dmd.double().abs()
    if with_din:
        d0, d1 = din[:B].double(), din[B:2 * B].double()
        terms = [-f[..., 0] * d0[..., 0], -f[..., 1] * d0[..., 1], -d0[..., 3], f[..., 0] * d1[..., 0], f[..., 1] * d1[..., 1], d1[..., 3]]
        for t in terms:
            dm, scale = dm + t, scale + t.abs()
    k = m * (1 - m) / 10
    _bf16('mask_bwd_bf16', got[..., 0].float(), dm * k, scale * k)
    assert torch.equal(got[..., 1].view(torch.int16), (-got[..., 0]).view(torch.int16))
    assert bool((got[..., 2:].float() == 0).all())


def test_grad_avg_abs_uneven_segments():
    """Mean over variables of mean|g| on segments of 1 .. 2.4 M elements (some have fewer elements than the 16 chunks a segment is
    split into), separated by padding the kernel must not read; the result accumulates into the caller-zeroed output."""
    lens = [1, 7, 255, 256, 257, 4097, 2400000]
    g = torch.Generator().manual_seed(2)
    pad = 13
    offs, a = [], pad
    for n in lens:
        offs.append((a, a + n))
        a += n + pad
    buf = torch.full((a,), 1e6)
    for (lo, hi) in offs:
        buf[lo:hi] = torch.randn(hi - lo, generator=g) * torch.rand(1, generator=g) * 1e-3
    seg = torch.tensor([v for pr in offs for v in pr], dtype=torch.int64, device='cuda')
    gd, out = buf.cuda(), torch.zeros(1, device='cuda')
    ref = float(np.mean([buf[lo:hi].double().abs().mean().item() for lo, hi in offs]))
    _lib.call('cis_grad_avg_abs', gd.data_ptr(), seg.data_ptr(), len(offs), out.data_ptr(), ST())
    torch.cuda.synchronize()
    _rel('grad_avg_abs', out.cpu(), torch.tensor([ref]), 2e-5)
    _lib.call('cis_grad_avg_abs', gd.data_ptr(), seg.data_ptr(), len(offs), out.data_ptr(), ST())
    torch.cuda.synchronize()
    _rel('grad_avg_abs', out.cpu(), torch.tensor([2 * ref]), 2e-5)


LR, B1, B2, EPS, CLIP = 1e-4, 0.9, 0.999, 1e-8, 0.2


def _adam_call(p, m, v, grad, n, gscale, step, avg=None, can_change=0, seed=8964, b1=B1):
    _lib.call('cis_clip_adam', p.data_ptr(), m.data_ptr(), v.data_ptr(), grad.data_ptr(), n, gscale, CLIP, LR, b1, B2, EPS, step.data_ptr(),
              avg.data_ptr() if avg is not None else None, can_change, seed, ST())
    torch.cuda.synchronize()


@pytest.mark.parametrize('t0', [0, 997])
@pytest.mark.parametrize('gscale', [1.0, 0.25])
def test_clip_adam_against_fp64_tf_adam(gscale, t0):
    """Five steps of clip + TF-Adam from step t0 (the shared beta-power step).  The parameters are zeroed before each step, so the
    fp32 result is the update itself; the reference starts every step from the kernel's fp32 m and v."""
    n = 2 ** 20 + 3
    g = torch.Generator().manual_seed(t0 + int(gscale * 8))
    if t0 == 0:
        m0, v0 = torch.zeros(n), torch.zeros(n)
    else:
        m0 = torch.randn(n, generator=g) * 0.03
        v0 = m0 ** 2 + (torch.rand(n, generator=g) * 0.05) ** 2
    m, v, p = m0.cuda(), v0.cuda(), torch.zeros(n, device='cuda')
    step = torch.full((1,), t0, dtype=torch.int64, device='cuda')
    lr, b1, b2, eps, clip = f32(LR), f32(B1), f32(B2), f32(EPS), f32(CLIP)
    for k in range(5):
        graw = (torch.rand(n, generator=g) * 4 - 2) * (CLIP / gscale)     # straddles +-clip
        graw[::97] = CLIP / gscale
        graw[1::101] = -CLIP / gscale
        graw = graw.float()
        mb, vb = m.cpu().double(), v.cpu().double()
        p.zero_()
        _adam_call(p, m, v, graw.cuda(), n, gscale, step)
        assert int(step.item()) == t0 + k + 1
        t = t0 + k + 1
        gg = (graw.double() * f32(gscale)).clamp(-clip, clip)
        mr = b1 * mb + (1 - b1) * gg
        vr = b2 * vb + (1 - b2) * gg * gg
        lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        _fp32('adam m', m, mr)
        _fp32('adam v', v, vr)
        _fp32('adam update', p, -lr_t * mr / (vr.sqrt() + eps))


def test_clip_adam_noise_branch():
    """can_change and mean|g| < 1e-5: every g is replaced by |U(-clip, clip)| from a hash of (seed, t, i).  With beta1 = 0 the new m
    is g exactly.  g in [0, clip], KS distance to U(0, clip) <= 1.63 / sqrt(n) (1 % level), identical for the same (seed, t),
    different for another t; with mean|g| = 2e-5 the same call only clips."""
    n = 2 ** 20 + 3
    grad = ((torch.rand(n, generator=torch.Generator().manual_seed(4)) * 2 - 1) * 0.5).cuda()
    avg = torch.full((1,), 0.5e-5, device='cuda')

    def run(t, a):
        m, v, p = torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
        step = torch.full((1,), t, dtype=torch.int64, device='cuda')
        _adam_call(p, m, v, grad, n, 1.0, step, avg=a, can_change=1, b1=0.0)
        assert int(step.item()) == t + 1
        return m

    g1, g2, g3 = run(5, avg), run(5, avg), run(6, avg)
    assert float(g1.min()) >= 0.0 and float(g1.max()) <= f32(CLIP)
    x = torch.sort(g1.double().cpu())[0] / f32(CLIP)
    i = torch.arange(1, n + 1, dtype=torch.float64)
    ks = float(torch.maximum(i / n - x, x - (i - 1) / n).max())
    _note('noise KS (of 1.63/sqrt n)', ks * math.sqrt(n) / 1.63)
    assert ks <= 1.63 / math.sqrt(n), ks
    assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))
    assert float((g1 == g3).double().mean()) < 1e-3
    clipped = run(5, torch.full((1,), 2e-5, device='cuda'))
    assert torch.equal(clipped, grad.clamp(-f32(CLIP), f32(CLIP)))


# ---------------------------------------------------------------------------------------------------------------- inside the step graph
GRAPH_CASES = [(64, 96, 2, 2, 0.5, 75.0), (36, 52, 3, 6, 1.0, 0.5), (128, 224, 1, 1, 0.3, 75.0), (256, 448, 4, 4, 0.5, 75.0)]


def _graph(H, W, B, GB=None, cbn=0.5, eps=75.0, seed=0):
    from unsupervised_detection_b200.step_graph import CISGraph
    gen = torch.Generator().manual_seed(seed)
    g = CISGraph(H, W, B, global_batch=GB, cbn=cbn, epsilon=eps, with_pwc=False)
    g.load_params(OP.make_params(seed=1, jitter=0.1, nets=('MaskNet', 'FlownetS')))
    g.image.copy_(torch.rand(B, H, W, 3, generator=gen) - 0.5)
    g.flow.copy_(_smooth(B, H, W, 2, 0.3, gen, div=16))
    return g


@pytest.fixture(scope='module', params=GRAPH_CASES, ids=lambda c: '%dx%d_B%d_GB%d_cbn%g_eps%g' % c)
def graph_run(request):
    """One graph per case: forward, generator backward, recover backward, with the buffers each phase leaves behind."""
    H, W, B, GB, cbn, eps = request.param
    g = _graph(H, W, B, GB, cbn, eps)
    g.forward()
    torch.cuda.synchronize()
    c = lambda t: t.detach().clone().cpu()
    r = dict(g=g, H=H, W=W, B=B, GB=GB, cbn=cbn, eps=eps, flow=c(g.flow), mask=c(g.mask), flow1=c(g.flow1), pred=c(g.pred), sums=c(g.sums),
             scalars=c(g.scalars), coef=c(g.coef), losses=g.losses(), full=g.losses(full=True))
    g.bwd['G'].run()
    torch.cuda.synchronize()
    r['G'] = dict(dpred=c(g.dpred), dmask=c(g.dmask), fg=c(g.rec.flow1.get_grad().float()), lg=c(g.gen.logits.get_grad().float()),
                  din=c(g.rec_in.get_grad().float()))
    g.bwd['R'].run()
    torch.cuda.synchronize()
    r['R'] = dict(dpred=c(g.dpred), fg=c(g.rec.flow1.get_grad().float()))
    yield r
    del r['g']
    torch.cuda.empty_cache()


def test_graph_forward_head(graph_run):
    r = graph_run
    B, H, W, GB = r['B'], r['H'], r['W'], r['GB']
    pref = _upsample(r['flow1'], H, W)
    _fp32('graph pred', r['pred'], pref)
    L, _, _ = _head(r['flow'], r['mask'], pref, B, r['cbn'], r['eps'], GB)
    _rel('graph sums', r['sums'], L['sums'], 1e-5)
    _scalars_check('graph ', r['scalars'], L, B, H, W, GB)
    _rel('graph coef', r['coef'], _coef_ref(L), 1e-5)
    ls, full = r['losses'], r['full']
    for k in ('generator', 'recover', 'red_rate', 'red_rate_compl'):
        assert ls[k] == full[k] == float(r['scalars'][['generator', 'recover', 'red_rate', 'red_rate_compl'].index(k)])
    # adversarial_learner.py:201-204: the first sample's reconstruction sums and denominators
    for k, ref in (('reconstruction_loss', L['rec'][0]), ('reconstruction_compl_loss', L['rec_c'][0]), ('denominator_red_rate', L['den'][0]),
                   ('denominator_red_rate_compl', L['den_c'][0])):
        _rel('graph diagnostics', torch.tensor(full[k]), ref, 1e-5)


def _graph_dpred_ref(r, which):
    B, H, W = r['B'], r['H'], r['W']
    L, m, p = _head(r['flow'], r['mask'], r['pred'], B, r['cbn'], r['eps'], r['GB'])
    dp, dm = torch.autograd.grad(L['recover'] if which == 0 else L['generator'], [p, m], retain_graph=True)
    return L, m, p, dp, dm


def _check_flow1_grad(key, fg, dp_ref, nb, h1, w1):
    ref = _adjoint(dp_ref[:nb], h1, w1)
    # the kernel transposes its own fp32 dpred (<= 1e-5 max|dpred| from dp_ref per element)
    slack = _adjoint(dp_ref[:nb].abs() + 5.0 * float(dp_ref[:nb].abs().max()), h1, w1)
    _bf16(key, fg[:nb], ref, slack)


def test_graph_generator_backward_head(graph_run):
    r = graph_run
    B, H, W, cbn = r['B'], r['H'], r['W'], r['cbn']
    h1, w1 = r['flow1'].shape[1], r['flow1'].shape[2]
    G = r['G']
    L, m, p, dp, dm = _graph_dpred_ref(r, 1)
    for j in range(3):
        _fp32('graph dpred G', G['dpred'][j * B:(j + 1) * B], dp[j * B:(j + 1) * B])
    dscale = _dmask_scale(r['flow'], p, _coef_ref(L), B, cbn)
    _close('graph dmask', G['dmask'], dm.view(B, H, W), 1e-5 * dscale)
    _check_flow1_grad('graph flow1 grad G', G['fg'], dp, 2 * B, h1, w1)
    # cis_mask_bwd chain on the graph's own recover-input gradient and the reference dmask
    f, mm, din = r['flow'].double(), r['mask'].double()[..., 0], G['din'].double()
    d0, d1 = din[:B], din[B:2 * B]
    terms = [-f[..., 0] * d0[..., 0], -f[..., 1] * d0[..., 1], -d0[..., 3], f[..., 0] * d1[..., 0], f[..., 1] * d1[..., 1], d1[..., 3]]
    dmv = dm.view(B, H, W).detach()
    tot, scale = dmv.clone(), dmv.abs() + 5.0 * dscale        # + the dmask error the kernel's fp32 dmask carries (<= 1e-5 dscale)
    for t in terms:
        tot, scale = tot + t, scale + t.abs()
    k = mm * (1 - mm) / 10
    _bf16('graph logits grad', G['lg'][..., 0], tot * k, scale * k)
    assert torch.equal(G['lg'][..., 1], -G['lg'][..., 0])


def test_graph_recover_backward_head(graph_run):
    r = graph_run
    B = r['B']
    h1, w1 = r['flow1'].shape[1], r['flow1'].shape[2]
    _, _, _, dp, _ = _graph_dpred_ref(r, 0)
    for j in range(3):
        _fp32('graph dpred R', r['R']['dpred'][j * B:(j + 1) * B], dp[j * B:(j + 1) * B])
    _check_flow1_grad('graph flow1 grad R', r['R']['fg'], dp, 3 * B, h1, w1)


def test_generator_step_data_parallel_split_equals_full_batch():
    """Generator-step counterpart of test_api_gpu.py::test_data_parallel_split_equals_full_batch: the gradients of two batch-2 graphs
    with global_batch = 4, summed, equal the batch-4 gradient; so do their loss scalars (each is this half's share)."""
    g4 = _graph(64, 96, 4)
    g4.forward()
    g4.bwd['G'].run()
    torch.cuda.synchronize()
    full, s_full = g4.gen_store.grad.clone(), g4.scalars[:4].double().cpu()
    g2 = _graph(64, 96, 2, GB=4)
    acc, s_acc = torch.zeros_like(g2.gen_store.grad), torch.zeros(4, dtype=torch.float64)
    image, flow = g4.image.clone(), g4.flow.clone()
    for h in range(2):
        g2.image.copy_(image[2 * h:2 * h + 2])
        g2.flow.copy_(flow[2 * h:2 * h + 2])
        g2.forward()
        g2.bwd['G'].run()
        torch.cuda.synchronize()
        acc += g2.gen_store.grad
        s_acc += g2.scalars[:4].double().cpu()
    cos = float(torch.dot(acc.double(), full.double()) / (acc.double().norm() * full.double().norm()))
    ratio = float(acc.norm() / full.norm())
    _note('dp split 1-cos (of 1e-4)', (1 - cos) / 1e-4)
    _note('dp split |norm-1| (of 1e-3)', abs(ratio - 1) / 1e-3)
    assert cos > 0.9999 and abs(ratio - 1) < 1e-3, (cos, ratio)
    _rel('dp split scalars', s_acc, s_full, 1e-6)

"""Gradients through ModelPWCNet.predict_from_img_pairs against torch.autograd through the CPU oracle (fp32), on the GPU, at 128x192 with
B = 2 (level 6 is 2x3): the fused warp + cost-volume backward and the transposed-conv backward alone, then the whole network, run-to-run
determinism, and the unchanged forward of calls without gradients."""
import pytest
import torch

from oracle import params as OP, pwcnet as OW, tf_ops as T
from unsupervised_detection_b200 import _lib
from unsupervised_detection_b200.engine import Act, Builder, ConvLayer, ParamStore, Plan, ACT_NONE
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import ModelPWCNet

pytestmark = pytest.mark.gpu
bf = lambda x: x.to(torch.bfloat16).float()
B, H, W = 2, 128, 192

# Bounds of the whole-network comparison.  Taken from the generator's 0.12 (bf16 activations through 17 layers); PWC-Net runs 18 shared
# feature layers, five DenseNet levels and their context networks, so the per-scope bound is looser.  Measured on an H100 SXM (400 W
# power limit) with these seeds: parameters 0.0736 (scopes ctxt 0.089, featpyr 0.079, predict_flow 0.055, upsample 0.143), lowest kernel
# cosine 0.948, img1 / img2 0.157 / 0.156.  The image bound started at 0.12 and is 0.25: the fp32 oracle's own image gradient moves by
# 0.130 / 0.134 when only its images and parameters are rounded to bf16 (printed by the test), because the warp's flow derivative jumps
# at sample-cell boundaries and every level's flow feeds the next level's warp.
GRAD_TOL, SCOPE_TOL, INPUT_TOL, COS_MIN = 0.12, 0.25, 0.25, 0.9


def _rel_l2(got, ref):
    e = sum(float(((g.detach().cpu().double() - r.detach().double()) ** 2).sum()) for g, r in zip(got, ref))
    n = sum(float((r.detach().double() ** 2).sum()) for r in ref)
    return (e / max(n, 1e-300)) ** 0.5


def _cos(a, b):
    a, b = a.detach().cpu().double().reshape(-1), b.detach().double().reshape(-1)
    return float((a @ b) / max(float(a.norm() * b.norm()), 1e-300))


def _pad8(x):
    b, h, w, c = x.shape
    out = torch.zeros(b, h, w, (c + 7) // 8 * 8, dtype=torch.bfloat16, device='cuda')
    out[..., :c] = x.to(torch.bfloat16).cuda()
    return out


def _costvol_case(h, w, C, seed, with_flow):
    g = torch.Generator().manual_seed(seed)
    c1, c2 = bf(torch.randn(B, h, w, C, generator=g)), bf(torch.randn(B, h, w, C, generator=g))
    up = bf(torch.randn(B, h, w, 81, generator=g))
    fs = 20.0 / 4 if with_flow else 1.0
    fl = None
    if with_flow:
        fl = torch.randn(B, h, w, 2, generator=g) * 3
        fl[:, ::3] = torch.round(fl[:, ::3])                          # integer sample positions (fs * fl exact): the inclusive clip rule
        fl[0, :2, :, 0] = -40.0                                         # rows past the bottom edge
        fl[1, :, :2, 1] = 60.0                                          # columns past the left edge
        fl[0, -2:, :, 0] = 50.0                                         # ... the top edge
        fl[1, :, -2:, 1] = -45.0                                        # ... the right edge
    ri = [c1.clone().requires_grad_(True), c2.clone().requires_grad_(True)] + ([fl.clone().requires_grad_(True)] if with_flow else [])
    warp = OW.dense_image_warp(ri[1], ri[2] * fs) if with_flow else ri[1]
    ref = torch.autograd.grad((OW.cost_volume(ri[0], warp) * up).sum(), ri)

    a1, a2 = _pad8(c1), _pad8(c2)
    dcorr = torch.zeros(B, h, w, 88, dtype=torch.bfloat16, device='cuda')
    dcorr[..., :81] = up.to(torch.bfloat16).cuda()
    d1, d2 = torch.zeros_like(a1), torch.zeros_like(a2)
    dfl = torch.zeros(B, h, w, 8, dtype=torch.bfloat16, device='cuda')
    flc = fl.cuda().contiguous() if with_flow else None
    gs = torch.empty(B * h * w * 81, device='cuda')
    ws = torch.empty(B * h * w * C, device='cuda')
    ds = torch.empty(B * h * w * C, dtype=torch.float64, device='cuda')

    def run(acc):
        _lib.call('cis_warp_costvol_bwd', a1.data_ptr(), a1.shape[-1], 0, a2.data_ptr(), a2.shape[-1], 0, flc.data_ptr() if with_flow else None,
                  fs, B, h, w, C, dcorr.data_ptr(), 88, 0, d1.data_ptr(), d1.shape[-1], 0, d2.data_ptr(), d2.shape[-1], 0, dfl.data_ptr(), 8, 0,
                  acc, gs.data_ptr(), ws.data_ptr(), ds.data_ptr(), torch.cuda.current_stream().cuda_stream)
    run(0)
    got = [d1[..., :C].float(), d2[..., :C].float()] + ([dfl[..., :2].float()] if with_flow else [])
    got = [t.clone() for t in got]
    run(7)                                                              # accumulate: every result doubles
    again = [d1[..., :C].float(), d2[..., :C].float()] + ([dfl[..., :2].float()] if with_flow else [])
    return ref, got, again


@pytest.mark.parametrize('h,w,C,with_flow', [(32, 48, 32, True), (2, 3, 196, False), (2, 3, 196, True)])
def test_warp_costvol_bwd_matches_autograd(h, w, C, with_flow):
    ref, got, again = _costvol_case(h, w, C, 21, with_flow)
    for i, (a, b, what) in enumerate(zip(got, ref, ('dc1', 'dc2', 'dflow'))):
        tol = (1e-2 if what == 'dflow' else 2 ** -7) * float(b.abs().max())
        err = float((a.cpu() - b).abs().max())
        print('MEASURED warp_costvol_bwd %dx%dx%d flow=%d %s max err / max %.2e' % (h, w, C, with_flow, what, err / float(b.abs().max())))
        assert err <= tol, what
        assert float((again[i].cpu() - 2 * a.cpu()).abs().max()) <= 2 * tol, what
    if with_flow:
        assert float((ref[2] == 0).float().mean()) > 0.05                 # the clamped branches are exercised


def _transposed_case(cin, h, w, g_off, seed):
    """One transposed conv through a one-layer Builder, its output gradient in channels [g_off, g_off + 2) of an 8-channel chunk."""
    g = torch.Generator().manual_seed(seed)
    dev = 'cuda'
    st = ParamStore(dev)
    L = ConvLayer(st, 'up', 4, cin, 2, act=ACT_NONE, tag='P', transposed=True)
    st.finalize(False)
    st.grad = torch.zeros_like(st.flat)
    wt = torch.randn(4, 4, 2, cin, generator=g) * (2.0 / (16 * cin)) ** 0.5
    bias = torch.randn(2, generator=g) * 0.1
    st.load({'up/kernel': wt, 'up/bias': bias})
    x = bf(torch.randn(2, h, w, cin, generator=g))
    up = bf(torch.randn(2, 2 * h, 2 * w, 2, generator=g))
    bld = Builder(dev)
    src = bld.new_act(2, h, w, cin, name='x', dep={'P'})
    src.buf[..., :cin] = x.to(torch.bfloat16).cuda()
    obuf, gbuf = (torch.zeros(2, 2 * h, 2 * w, 8, dtype=torch.bfloat16, device=dev) for _ in range(2))
    out = Act(2, 2 * h, 2 * w, 2, dev, buf=obuf, c_off=g_off, chanmap=[0, 1], name='y')
    out.grad_buf = gbuf
    bld.conv_transpose(L, src, out=out)
    bp = bld.build_backward('P', [out])
    fin, pack = Plan('fin'), Plan('pack')
    L.plan_finalize(fin, 'P')
    L.plan_pack(pack, dgrad=True)
    pack.run()
    bld.fwd.run()
    gbuf[..., g_off:g_off + 2] = up.to(torch.bfloat16).cuda()
    bp.run()
    fin.run()
    torch.cuda.synchronize()
    ri = [x.clone().requires_grad_(True), wt.clone().requires_grad_(True), bias.clone().requires_grad_(True)]
    y = T.conv2d_transpose_k4s2(*ri)
    assert float((obuf[..., g_off:g_off + 2].float().cpu() - y.detach()).abs().max()) <= 2e-2 * float(y.abs().max())
    ref = torch.autograd.grad((y * up).sum(), ri)
    got = [src.get_grad().float()[..., :cin], st.view('up/kernel', 'grad'), st.view('up/bias', 'grad')]
    return got, ref


@pytest.mark.parametrize('cin,h,w,g_off', [(2, 8, 12, 0), (529, 2, 3, 2), (661, 4, 6, 2)])
def test_transposed_conv_backward_matches_autograd(cin, h, w, g_off):
    got, ref = _transposed_case(cin, h, w, g_off, 5)
    for a, b, what in zip(got, ref, ('dx', 'dW', 'db')):
        assert a.shape == b.shape, what
        rel = _rel_l2([a], [b])
        print('MEASURED transposed conv Cin %d %s rel L2 %.4f' % (cin, what, rel))
        assert rel <= 2e-2, what


def _inputs(seed):
    g = torch.Generator().manual_seed(seed)
    img1 = torch.rand(B, H, W, 3, generator=g) - 0.5
    lo = torch.randn(B, 2, 3, 4, generator=g) * 4
    disp = torch.nn.functional.interpolate(lo, size=(H, W), mode='bicubic', align_corners=False).permute(0, 2, 3, 1).contiguous()
    img2 = (OW.dense_image_warp(img1, disp) + 0.02 * torch.randn(B, H, W, 3, generator=g)).clamp(-0.5, 0.5)
    up = torch.randn(B, H, W, 2, generator=g)
    return img1, img2, up


def _params():
    p = OP.make_params(11, jitter=0.05, nets=('pwcnet',))
    names = [n for n in p if n.startswith('pwcnet/')]
    for n in names:
        p[n].requires_grad_(True)
    return p, names


def _ours(img1, img2, p, names, up):
    x = [img1.cuda().requires_grad_(True), img2.cuda().requires_grad_(True)]
    out = ModelPWCNet.predict_from_img_pairs(x[0], x[1], params=p)
    return out, torch.autograd.grad((out * up.cuda()).sum(), x + [p[n] for n in names])


def test_pwcnet_gradients_match_oracle():
    p, names = _params()
    img1, img2, up = _inputs(0)
    ri = [img1.clone().requires_grad_(True), img2.clone().requires_grad_(True)]
    ref_out = OW.predict_from_img_pairs(ri[0], ri[1], p)
    ref = torch.autograd.grad((ref_out * up).sum(), ri + [p[n] for n in names])
    out, got = _ours(img1, img2, p, names, up)
    print('MEASURED pwcnet flow rel L2 %.4f' % _rel_l2([out], [ref_out]))
    # conditioning of the reference itself: the same fp32 oracle with bf16-rounded images and parameters (the operands the kernels see)
    pb = {n: bf(t.detach()).requires_grad_(True) for n, t in p.items()}
    rb = [bf(img1).requires_grad_(True), bf(img2).requires_grad_(True)]
    refb = torch.autograd.grad((OW.predict_from_img_pairs(rb[0], rb[1], pb) * up).sum(), rb + [pb[n] for n in names])
    print('MEASURED oracle bf16-operand sensitivity: params rel L2 %.4f, img1 %.4f, img2 %.4f'
          % (_rel_l2(refb[2:], ref[2:]), _rel_l2(refb[:1], ref[:1]), _rel_l2(refb[1:2], ref[1:2])))
    rel = _rel_l2(got[2:], ref[2:])
    ins = [_rel_l2(got[i:i + 1], ref[i:i + 1]) for i in range(2)]
    print('MEASURED pwcnet params rel L2 %.4f, img1 %.4f, img2 %.4f' % (rel, ins[0], ins[1]))
    scopes = {}
    for n, a, b in zip(names, got[2:], ref[2:]):
        scopes.setdefault(n.split('/')[1], []).append((a, b))
    for sc, ab in sorted(scopes.items()):
        r = _rel_l2([a for a, _ in ab], [b for _, b in ab])
        print('MEASURED pwcnet scope %s rel L2 %.4f' % (sc, r))
        assert r <= SCOPE_TOL, sc
    cos = {n: _cos(a, b) for n, a, b in zip(names, got[2:], ref[2:]) if n.endswith('/kernel')}
    worst = min(cos, key=cos.get)
    print('MEASURED pwcnet lowest kernel cosine %.4f (%s)' % (cos[worst], worst))
    assert rel <= GRAD_TOL
    assert all(v <= INPUT_TOL for v in ins), ins
    assert cos[worst] >= COS_MIN, worst


def test_pwcnet_backward_is_deterministic_and_forward_unchanged():
    p, names = _params()
    img1, img2, up = _inputs(0)
    out_a, a = _ours(img1, img2, p, names, up)
    out_b, b = _ours(img1, img2, p, names, up)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    with torch.no_grad():
        plain = ModelPWCNet.predict_from_img_pairs(img1.cuda(), img2.cuda(), params=p)     # the forward-only runner
    assert torch.equal(plain, out_a.detach()) and torch.equal(out_a, out_b)

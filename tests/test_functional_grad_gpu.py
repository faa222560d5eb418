"""Gradients of the function-level API (models/functional.py) against torch.autograd through the CPU oracle, on the GPU, at 64x96:
charbonnier_loss, cost_volume, dense_image_warp, generator_net and recover_net one by one, then the generator and recover steps of
adversarial_learner.py:99-194 written in plain PyTorch from the functional calls, and run-to-run determinism."""
import pytest
import torch

from oracle import nets as ON, pwcnet as OW, losses as OL, params as OP
from unsupervised_detection_b200.models.nets import generator_net, recover_net
from unsupervised_detection_b200.models.utils.loss_utils import charbonnier_loss
from unsupervised_detection_b200.models.PWCNet.core_costvol import cost_volume
from unsupervised_detection_b200.models.PWCNet.core_warp import dense_image_warp

pytestmark = pytest.mark.gpu
bf = lambda x: x.to(torch.bfloat16).float()
H, W = 64, 96

# relative L2 of the whole gradient vector of a scope (bf16 activations through 17 / 32 layers).  Measured on an H100 SXM (700 W power
# limit) with these seeds: generator_net 0.0082, generator step 0.0281; recover_net 0.0218, recover step 0.0164.  The 256x448 step-graph
# bounds of test_parity_bench_sizes_gpu.py (0.12 / 0.02) were the starting point; R is raised to about twice the value measured at
# 64x96 (the step graph measured 0.0046 at 256x448).
GRAD_TOL = {'G': 0.12, 'R': 0.04}
INPUT_TOL = 0.05          # relative L2 of an input gradient (bf16 gradient Acts); measured 0.0063 (generator), 0.030-0.033 (recover)


def _rel_l2(got, ref):
    e = sum(float(((g.detach().cpu().double() - r.detach().double()) ** 2).sum()) for g, r in zip(got, ref))
    n = sum(float((r.detach().double() ** 2).sum()) for r in ref)
    return (e / max(n, 1e-300)) ** 0.5


def _params(scope, seed=11):
    p = OP.make_params(seed, jitter=0.05, nets=('MaskNet', 'FlownetS'))
    names = [n for n in p if n.startswith(scope + '/')]
    for n in names:
        p[n].requires_grad_(True)
    return p, names


def test_charbonnier_loss_gradients_match_oracle():
    g = torch.Generator().manual_seed(3)
    for mc in (1, 2):
        for cbn in (0.5, 1.0, 0.3):
            gt, pr = torch.randn(2, H, W, 2, generator=g), torch.randn(2, H, W, 2, generator=g)
            mask = torch.rand(2, H, W, mc, generator=g)
            up = torch.randn(2, generator=g)
            ref_in = [t.clone().requires_grad_(True) for t in (gt, pr, mask)]
            ref = torch.autograd.grad((OL.charbonnier_loss(*ref_in, cbn) * up).sum(), ref_in)
            got_in = [t.cuda().requires_grad_(True) for t in (gt, pr, mask)]
            got = torch.autograd.grad((charbonnier_loss(*got_in, cbn) * up.cuda()).sum(), got_in)
            for a, b, what in zip(got, ref, ('dgt', 'dpred', 'dmask')):
                assert torch.allclose(a.cpu(), b, rtol=1e-4, atol=1e-5 * float(b.abs().max())), (mc, cbn, what)


@pytest.mark.parametrize('shape', [(2, H, W, 37), (1, 5, 7, 20)])      # the second map is smaller than the 9x9 window
def test_cost_volume_gradients_match_oracle(shape):
    g = torch.Generator().manual_seed(4)
    c1, c2 = bf(torch.randn(*shape, generator=g)), bf(torch.randn(*shape, generator=g))
    up = torch.randn(*shape[:3], 81, generator=g)
    ri = [c1.clone().requires_grad_(True), c2.clone().requires_grad_(True)]
    ref = torch.autograd.grad((OW.cost_volume(*ri) * up).sum(), ri)
    gi = [c1.cuda().requires_grad_(True), c2.cuda().requires_grad_(True)]
    got = torch.autograd.grad((cost_volume(*gi) * up.cuda()).sum(), gi)
    for a, b in zip(got, ref):
        assert a.shape == b.shape
        assert float((a.cpu() - b).abs().max()) <= 2 ** -7 * float(b.abs().max())


def _warp_inputs(seed):
    g = torch.Generator().manual_seed(seed)
    img = bf(torch.randn(2, H, W, 5, generator=g))
    fl = torch.randn(2, H, W, 2, generator=g) * 30                       # samples far past every edge
    fl[:, ::3] = torch.round(fl[:, ::3])                                  # integer positions: alpha exactly 0 or 1 (inclusive clip)
    fl[0, :8, :, 0] = -80.0                                               # whole rows past the bottom edge
    fl[1, :, :8, 1] = 120.0                                               # whole columns past the left edge
    up = torch.randn(2, H, W, 5, generator=g)
    return img, fl, up


def test_dense_image_warp_gradients_match_oracle():
    img, fl, up = _warp_inputs(5)
    ri = [img.clone().requires_grad_(True), fl.clone().requires_grad_(True)]
    ref = torch.autograd.grad((OW.dense_image_warp(*ri) * up).sum(), ri)
    gi = [img.cuda().requires_grad_(True), fl.cuda().requires_grad_(True)]
    got = torch.autograd.grad((dense_image_warp(*gi) * up.cuda()).sum(), gi)
    for a, b, what in zip(got, ref, ('dimage', 'dflow')):
        assert float((a.cpu() - b).abs().max()) <= 1e-5 * float(b.abs().max()), what
    assert float((ref[1] == 0).float().mean()) > 0.05                     # the clamped branches are exercised


def _gen_inputs(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(2, H, W, 3, generator=g) - 0.5, torch.randn(2, H, W, 2, generator=g), torch.randn(2, H, W, 1, generator=g)


def _rec_inputs(seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(2, H, W, 3, generator=g) - 0.5
    m = torch.rand(2, H, W, 1, generator=g)
    fm = torch.randn(2, H, W, 2, generator=g) * 0.3 * (1 - m)
    return img, fm, m, torch.randn(2, H, W, 2, generator=g) * 0.01


def test_generator_net_gradients_match_oracle():
    p, names = _params('MaskNet')
    img, flw, up = _gen_inputs(0)
    ri = [img.clone().requires_grad_(True), flw.clone().requires_grad_(True)]
    ref = torch.autograd.grad((ON.generator_net(*ri, p) * up).sum(), ri + [p[n] for n in names])
    gi = [img.cuda().requires_grad_(True), flw.cuda().requires_grad_(True)]
    got = torch.autograd.grad((generator_net(*gi, 'MaskNet/', params=p) * up.cuda()).sum(), gi + [p[n] for n in names])
    rel = _rel_l2(got[2:], ref[2:])
    print('MEASURED generator_net params rel L2 %.4f, image %.4f, flow %.4f'
          % (rel, _rel_l2(got[:1], ref[:1]), _rel_l2(got[1:2], ref[1:2])))
    assert rel <= GRAD_TOL['G']
    assert _rel_l2(got[:1], ref[:1]) <= INPUT_TOL and _rel_l2(got[1:2], ref[1:2]) <= INPUT_TOL


def test_recover_net_gradients_match_oracle():
    p, names = _params('FlownetS')
    img, fm, m, up = _rec_inputs(1)
    ri = [t.clone().requires_grad_(True) for t in (img, fm, m)]
    ref = torch.autograd.grad((ON.recover_net(*ri, p) * up).sum(), ri + [p[n] for n in names])
    gi = [t.cuda().requires_grad_(True) for t in (img, fm, m)]
    got = torch.autograd.grad((recover_net(*gi, 'FlownetS/', params=p) * up.cuda()).sum(), gi + [p[n] for n in names])
    rel = _rel_l2(got[3:], ref[3:])
    ins = [_rel_l2(got[i:i + 1], ref[i:i + 1]) for i in range(3)]
    print('MEASURED recover_net params rel L2 %.4f, img1 / flow_masked / mask %s' % (rel, ['%.4f' % v for v in ins]))
    assert rel <= GRAD_TOL['R']
    assert all(v <= INPUT_TOL for v in ins), ins


def _step_losses(image, flow, p, gen, rec, charb, pre, cbn=0.5, eps=75.0):
    """adversarial_learner.py:99-194: generator and recover losses from the function-level calls."""
    B = image.shape[0]
    m = gen(image, pre(flow), p)
    mc = 1.0 - m
    pred = rec(image, flow * (1.0 - m), m, p)
    pred_c = rec(image, flow * (1.0 - mc), mc, p)
    pred_i = rec(image, torch.zeros_like(flow), torch.ones_like(m), p)       # the image-only call
    rec_l = charb(flow, pred, m, cbn)
    rec_c = charb(flow, pred_c, mc, cbn)
    prior = charb(flow, pred_i, torch.ones_like(flow), cbn)
    den = charb(flow, pred_i, m, cbn) + eps
    den_c = charb(flow, pred_i, mc, cbn) + eps
    generator_loss = (1.0 - rec_l / den).sum() / B + (1.0 - rec_c / den_c).sum() / B
    recover_loss = (rec_l.sum() + rec_c.sum() + prior.sum()) / float(image.shape[1] * image.shape[2] * B)
    return generator_loss, recover_loss


def _ours(image, flow, p):
    return _step_losses(image.cuda(), flow.cuda(), p, lambda i, f, q: generator_net(i, f, 'MaskNet/', params=q),
                        lambda i, f, m, q: recover_net(i, f, m, 'FlownetS/', params=q), charbonnier_loss, OL.preprocess_flow_batch)


def _oracle(image, flow, p):
    return _step_losses(image, flow, p, ON.generator_net, ON.recover_net, OL.charbonnier_loss, OL.preprocess_flow_batch)


@pytest.mark.parametrize('scope,which', [('MaskNet', 0), ('FlownetS', 1)])
def test_adversarial_step_from_functional_calls_matches_oracle(scope, which):
    """The generator step (scope MaskNet, generator loss) and the recover step (FlownetS, recover loss), one backward each."""
    g = torch.Generator().manual_seed(7)
    image = torch.rand(2, H, W, 3, generator=g) - 0.5
    lo = torch.randn(2, 2, 4, 6, generator=g)
    flow = (torch.nn.functional.interpolate(lo, size=(H, W), mode='bicubic') * 0.3).permute(0, 2, 3, 1).contiguous()
    p, names = _params(scope, seed=3)
    ref_l = _oracle(image, flow, p)
    ref = torch.autograd.grad(ref_l[which], [p[n] for n in names])
    got_l = _ours(image, flow, p)
    got = torch.autograd.grad(got_l[which], [p[n] for n in names])
    # the oracle's own composition agrees with its adversarial_losses (the same loss, written the same way as above)
    L = OL.adversarial_losses(image, flow, p)
    assert abs(float(L['generator' if which == 0 else 'recover']) - float(ref_l[which])) <= 1e-5 * abs(float(ref_l[which])) + 1e-7
    rel = _rel_l2(got, ref)
    print('MEASURED %s step: loss %.6f vs %.6f, params rel L2 %.4f' % (scope, float(got_l[which]), float(ref_l[which]), rel))
    assert rel <= GRAD_TOL['G' if which == 0 else 'R']


def test_backward_passes_are_deterministic():
    p, gnames = _params('MaskNet')
    img, flw, up = _gen_inputs(0)

    def gen_grads():
        x = [img.cuda().requires_grad_(True), flw.cuda().requires_grad_(True)]
        return torch.autograd.grad((generator_net(*x, params=p) * up.cuda()).sum(), x + [p[n] for n in gnames])
    pr, rnames = _params('FlownetS')
    rimg, fm, m, rup = _rec_inputs(1)

    def rec_grads():
        x = [t.cuda().requires_grad_(True) for t in (rimg, fm, m)]
        return torch.autograd.grad((recover_net(*x, params=pr) * rup.cuda()).sum(), x + [pr[n] for n in rnames])
    gc = torch.Generator().manual_seed(4)
    c1, c2 = torch.randn(2, 12, 20, 37, generator=gc).cuda(), torch.randn(2, 12, 20, 37, generator=gc).cuda()
    cup = torch.randn(2, 12, 20, 81, generator=gc).cuda()

    def cv_grads():
        x = [c1.clone().requires_grad_(True), c2.clone().requires_grad_(True)]
        return torch.autograd.grad((cost_volume(*x) * cup).sum(), x)
    for f in (gen_grads, rec_grads, cv_grads):
        a, b = f(), f()
        assert all(torch.equal(u, v) for u, v in zip(a, b)), f.__name__
    wimg, wfl, wup = _warp_inputs(5)

    def warp_grads():
        x = [wimg.cuda().requires_grad_(True), wfl.cuda().requires_grad_(True)]
        return torch.autograd.grad((dense_image_warp(*x) * wup.cuda()).sum(), x)
    a, b = warp_grads(), warp_grads()
    assert torch.equal(a[1], b[1])
    assert float((a[0] - b[0]).abs().max()) <= 1e-6 * float(a[0].abs().max())

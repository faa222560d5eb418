"""Layer primitives of convolution_utils.py and preprocess_flow_batch against the fp64 oracle on the GPU: every cell of the supported set
(forward, input and parameter gradients), the four resize modes (forward and backward, run-to-run determinism), the flow standardisation,
and two compositions -- the generator rebuilt from the primitives, and one recover decoder step."""
import math

import pytest
import torch

import resize_ref
from oracle import losses as OL, nets as ON, params as OP, tf_ops as T
from unsupervised_detection_b200.models import functional as F
from unsupervised_detection_b200.models.utils import convolution_utils as CU
from unsupervised_detection_b200.models.utils.flow_utils import preprocess_flow_batch

pytestmark = pytest.mark.gpu
H, W = 37, 53

# relative L2 against the oracle's fp64 autograd (bf16 activations and packed weights, fp32 accumulation and outputs).  Measured on an
# H100 SXM (700 W power limit) over every cell below: output <= 3.3e-3; gradients <= 4.3e-3 through ELU (gen_conv) and <= 5.1e-2
# through leaky_relu (conv).  The leaky bound is looser because leaky_relu's derivative jumps from 1 to 0.2 at 0: rounding the input
# and the weights to bf16 moves pre-activations near 0 across it, and each such pixel passes 1 instead of 0.2 (or the reverse) of its
# gradient.  Rounding only the input and the weights of an fp64 conv to bf16 gives 2.5e-2 for a 3x3 20->16 leaky layer (3.1e-3 with
# ELU, whose derivative is continuous); the recover net, made of leaky layers, shows the same in test_functional_grad_gpu.py.
OUT_TOL, GRAD_TOL_ELU, GRAD_TOL_LEAKY = 1e-2, 2e-2, 6e-2
GRAD_TOL_G = 0.12                  # test_functional_grad_gpu.py GRAD_TOL['G']: the whole MaskNet gradient through 17 bf16 layers


def _rel_l2(got, ref):
    got, ref = got.detach().cpu().double(), ref.detach().double()
    return float((got - ref).norm() / max(float(ref.norm()), 1e-300))


def _layer_params(g, name, k, cin, cout, bn):
    a = math.sqrt(6.0 / (k * k * (cin + cout)))
    jit = lambda: (torch.rand(cout, generator=g, dtype=torch.float64) * 2 - 1) * 0.05
    w = (torch.rand(k, k, cin, cout, generator=g, dtype=torch.float64) * 2 - 1) * a
    if bn:
        return {name + '/kernel': w, name + '/bias': jit(), name + '/gamma': 1.0 + jit(), name + '/beta': jit()}
    return {name + '/weights': w, name + '/biases': jit()}


def _leaf(t):
    """fp64 leaf for the oracle's autograd; kernels get the memory layout of an OIHW tensor, so the permuted weight torch's CPU conv
    sees is contiguous (its backward rejects a non-contiguous weight of one output channel)."""
    if t.dim() == 4:
        t = t.permute(3, 2, 0, 1).contiguous().permute(2, 3, 1, 0)
    return t.detach().clone(memory_format=torch.preserve_format).requires_grad_(True)


def _oracle_layer(x, p, name, k, stride, rate, bn, act):
    if bn:
        y = T.conv2d_same(x, p[name + '/kernel'], stride, rate, p[name + '/bias'])
        return act(T.batch_norm_inference(y, p[name + '/gamma'], p[name + '/beta']))
    return act(T.conv2d_same(x, p[name + '/weights'], stride, rate, p[name + '/biases']))


CELLS = ([(k, s, 1, bn) for k in range(1, 8) for s in (1, 2) for bn in (True, False)] +
         [(3, 1, r, bn) for r in (2, 3, 4, 8, 9, 16) for bn in (True, False)])


@pytest.mark.parametrize('cin,cout', [(3, 1), (20, 16), (64, 200)])
@pytest.mark.parametrize('k,stride,rate,bn', CELLS)
def test_layer_cell_matches_oracle(k, stride, rate, bn, cin, cout):
    g = torch.Generator().manual_seed(1000 * k + 100 * stride + rate + cin + cout)
    name = 'Net/layer'
    p = _layer_params(g, name, k, cin, cout, bn)
    x = torch.randn(2, H, W, cin, generator=g, dtype=torch.float64)
    oh, ow = -(-H // stride), -(-W // stride)
    # upstream gradient with a non-zero mean: with a zero-mean one the bias / gamma / beta gradients of a one-channel layer are single
    # sums that nearly cancel, and their relative error measures that cancellation rather than the kernels
    up = torch.randn(2, oh, ow, cout, generator=g, dtype=torch.float64) + 0.5
    names = sorted(p)
    act = (T.elu, CU.elu) if bn else (T.leaky_relu, CU.leaky_relu)
    ri = [x.clone().requires_grad_(True)] + [_leaf(p[n]) for n in names]
    ref_y = _oracle_layer(ri[0], dict(zip(names, ri[1:])), name, k, stride, rate, bn, act[0])
    ref = torch.autograd.grad((ref_y * up).sum(), ri)
    gi = [x.float().cuda().requires_grad_(True)] + [p[n].float().cuda().requires_grad_(True) for n in names]
    gp = dict(zip(names, gi[1:]))
    y = _run_cell(gi[0], k, cin, cout, stride, rate, bn, act[1], name, gp)
    got = torch.autograd.grad((y * up.float().cuda()).sum(), gi)
    with torch.no_grad():                                   # the forward-only plan computes the same output
        assert torch.equal(_run_cell(gi[0], k, cin, cout, stride, rate, bn, act[1], name, gp), y.detach())
    rel_out = _rel_l2(y, ref_y)
    rel_grads = {n: _rel_l2(a, b) for n, a, b in zip(['x'] + names, got, ref)}
    print('MEASURED cell k%d s%d r%d bn%d %d->%d out %.2e grads %s' % (k, stride, rate, bn, cin, cout, rel_out,
                                                                      ' '.join('%s %.2e' % kv for kv in rel_grads.items())))
    assert rel_out <= OUT_TOL
    assert max(rel_grads.values()) <= (GRAD_TOL_ELU if bn else GRAD_TOL_LEAKY), rel_grads


def _run_cell(x, k, cin, cout, stride, rate, bn, act, name, p):
    """gen_conv for the BN cells, conv for the others; conv() takes no rate, so the dilated cells without BN call the layer helper
    behind both with conv's parameters."""
    if bn:
        return CU.gen_conv(x, cout, k, stride, rate, name=name, activation=act, params=p)
    if rate == 1:
        return CU.conv(x, name, [k, k, cin, cout], stride, activation=act, params=p)
    return F._layer('conv', x, 'conv', k, cout, stride, rate, 'SAME', act, name, params=p)


# ------------------------------------------------------------------------------------------------------------- resizes
RESIZE_CASES = [((5, 7), (11, 13)), ((37, 53), (16, 20)), ((12, 16), (7, 5)), ((6, 8), (1, 1)), ((1, 5), (4, 9)), ((33, 17), (33, 40)),
                ((16, 24), (32, 48))]


def _oracle_resize(x, size, method, ac):
    if method == 'nearest':
        return (T.resize_nn_align_corners if ac else T.resize_nn_legacy)(x, *size)
    return resize_ref.resize_bilinear(x, size[0], size[1], ac)


@pytest.mark.parametrize('src,size', RESIZE_CASES)
@pytest.mark.parametrize('method', ['bilinear', 'nearest'])
@pytest.mark.parametrize('ac', [False, True])
@pytest.mark.parametrize('C', [3, 64])
def test_resize_matches_oracle_and_is_deterministic(src, size, method, ac, C):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, src[0], src[1], C, generator=g)
    up = torch.randn(2, size[0], size[1], C, generator=g, dtype=torch.float64)
    fn = CU.resize_bilinear if method == 'bilinear' else CU.resize_nearest_neighbor
    got = fn(x.cuda(), size, align_corners=ac).cpu()
    ref = _oracle_resize(x, size, method, ac)
    if method == 'nearest':
        assert torch.equal(got, ref)
    else:
        assert float((got - ref).abs().max()) <= 1e-6 * float(ref.abs().max())
    rx = x.double().requires_grad_(True)
    (dref,) = torch.autograd.grad((_oracle_resize(rx, size, method, ac) * up).sum(), [rx])
    grads = []
    for _ in range(2):
        gx = x.cuda().requires_grad_(True)
        (d,) = torch.autograd.grad((fn(gx, size, align_corners=ac) * up.float().cuda()).sum(), [gx])
        grads.append(d.cpu())
    assert torch.equal(grads[0], grads[1])
    assert float((grads[0].double() - dref).abs().max()) <= 1e-5 * float(dref.abs().max()) + 1e-6


def test_resize_helper_sizes():
    x = torch.randn(1, 10, 14, 4).cuda()
    assert tuple(CU.resize(x).shape) == (1, 20, 28, 4)
    assert tuple(CU.resize(x, scale=0.5, func=CU.resize_nearest_neighbor).shape) == (1, 5, 7, 4)
    got, ref = CU.resize(x, to_shape=[20, 28]).cpu(), resize_ref.resize_bilinear(x.cpu(), 20, 28, True)
    assert float((got - ref).abs().max()) <= 1e-6 * float(ref.abs().max())


# ------------------------------------------------------------------------------------------------------- flow standardisation
@pytest.mark.parametrize('shape', [(3, 64, 96, 2), (2, 37, 53, 2), (1, 384, 640, 2)])
def test_preprocess_flow_batch_matches_oracle(shape):
    g = torch.Generator().manual_seed(5)
    f = torch.randn(*shape, generator=g) * torch.tensor([3.0, 0.5]) + torch.tensor([1.5, -4.0])
    up = torch.randn(*shape, generator=g, dtype=torch.float64)
    rf = f.double().requires_grad_(True)
    ref = OL.preprocess_flow_batch(rf)
    (dref,) = torch.autograd.grad((ref * up).sum(), [rf])
    outs, grads = [], []
    for _ in range(2):
        gf = f.cuda().requires_grad_(True)
        y = preprocess_flow_batch(gf)
        (d,) = torch.autograd.grad((y * up.float().cuda()).sum(), [gf])
        outs.append(y.detach().cpu())
        grads.append(d.cpu())
    assert torch.equal(outs[0], outs[1]) and torch.equal(grads[0], grads[1])
    with torch.no_grad():
        assert torch.equal(preprocess_flow_batch(f.cuda()).cpu(), outs[0])
    print('MEASURED preprocess_flow_batch %s out %.2e grad %.2e' % (shape, _rel_l2(outs[0], ref), _rel_l2(grads[0], dref)))
    assert _rel_l2(outs[0], ref) <= 1e-6          # measured <= 2.8e-7 (H100 SXM, 700 W), gradient <= 6.7e-8
    assert _rel_l2(grads[0], dref) <= 1e-4


# -------------------------------------------------------------------------------------------------------------- compositions
def _generator_from_primitives(img, flw, p):
    """models/nets.py:4-42 written with the layer primitives, the generator's input standardisation in front."""
    gc = lambda x, c, k, s, n, r=1, **kw: CU.gen_conv(x, c, k, s, r, name='MaskNet/' + n, params=p, **kw)
    x = torch.cat((img, preprocess_flow_batch(flw)), 3)
    x_0 = gc(x, 32, 5, 1, 'conv1')
    x = gc(x_0, 64, 3, 2, 'conv2_downsample')
    x_1 = gc(x, 64, 3, 1, 'conv3')
    x = gc(x_1, 128, 3, 2, 'conv4_downsample')
    x = gc(x, 128, 3, 1, 'conv5')
    x_2 = gc(x, 128, 3, 1, 'conv6')
    x = gc(x_2, 128, 3, 1, 'conv7_atrous', 2)
    x = gc(x, 128, 3, 1, 'conv8_atrous', 4)
    x = gc(x, 128, 3, 1, 'conv9_atrous', 8)
    x = gc(x, 128, 3, 1, 'conv10_atrous', 16)
    x = gc(x, 128, 3, 1, 'conv11') + x_2
    x = gc(x, 128, 3, 1, 'conv12')
    x = CU.gen_deconv(x, 64, name='MaskNet/conv13_upsample', params=p)
    x = gc(x, 64, 3, 1, 'conv14') + x_1
    x = CU.gen_deconv(x, 32, name='MaskNet/conv15_upsample', params=p) + x_0
    x = gc(x, 16, 3, 1, 'conv16')
    x = gc(x, 2, 3, 1, 'conv17', activation=CU.identity)
    return torch.softmax(x / 10.0, dim=-1)[..., 0:1]


def test_generator_rebuilt_from_primitives_matches_oracle():
    p = OP.make_params(11, jitter=0.05, nets=('MaskNet',))
    names = sorted(p)
    g = torch.Generator().manual_seed(0)
    img = torch.rand(2, 64, 96, 3, generator=g) - 0.5
    flw = torch.randn(2, 64, 96, 2, generator=g) * 2.0 + 0.5
    up = torch.randn(2, 64, 96, 1, generator=g)
    rp = {n: p[n].clone().requires_grad_(True) for n in names}
    ref = ON.generator_net(img, OL.preprocess_flow_batch(flw), rp)
    dref = torch.autograd.grad((ref * up).sum(), [rp[n] for n in names])
    gp = {n: p[n].cuda().requires_grad_(True) for n in names}
    got = _generator_from_primitives(img.cuda(), flw.cuda(), gp)
    dgot = torch.autograd.grad((got * up.cuda()).sum(), [gp[n] for n in names])
    got = got.detach().cpu()
    assert float((got - ref).abs().mean()) < 2e-3 and float((got - ref).abs().max()) < 3e-2    # test_generator_net_matches_oracle
    e = sum(float(((a.cpu().double() - b.double()) ** 2).sum()) for a, b in zip(dgot, dref))
    rel = (e / sum(float((b.double() ** 2).sum()) for b in dref)) ** 0.5
    print('MEASURED generator from primitives: mask mean-abs %.2e max %.2e, MaskNet grads rel L2 %.4f'
          % (float((got - ref).abs().mean()), float((got - ref).abs().max()), rel))
    assert rel <= GRAD_TOL_G                      # measured 0.0082, mask mean-abs 8.6e-5, max 4.1e-4 (H100 SXM, 700 W)


def test_recover_decoder_step_matches_oracle():
    """deconv5 = deconv(concat(aconv6, bconv6), size of bconv51) and flow5 = conv(concat(deconv5, bconv51, aconv51)) of nets.py:78-82
    at the 64x96 pyramid (conv6 1x2, conv51 2x3), f = 0.25."""
    p = OP.make_params(11, jitter=0.05, nets=('FlownetS',))
    names = ['FlownetS/deconv5/weights', 'FlownetS/deconv5/biases', 'FlownetS/flow5/weights', 'FlownetS/flow5/biases']
    g = torch.Generator().manual_seed(3)
    c6 = torch.randn(2, 1, 2, 256, generator=g)
    c51 = torch.randn(2, 2, 3, 256, generator=g)
    up = torch.randn(2, 2, 3, 2, generator=g)
    rx = [c6.double().requires_grad_(True), c51.double().requires_grad_(True)] + [_leaf(p[n].double()) for n in names]
    rp = dict(zip(names, rx[2:]))
    d5 = ON.deconv(rx[0], rp, 'FlownetS', 'deconv5', (2, 3))
    ref = ON.conv(torch.cat([d5, rx[1]], 3), rp, 'FlownetS', 'flow5', 1, activation=lambda t: t)
    dref = torch.autograd.grad((ref * up.double()).sum(), rx)
    gx = [c6.cuda().requires_grad_(True), c51.cuda().requires_grad_(True)] + [p[n].cuda().requires_grad_(True) for n in names]
    gp = dict(zip(names, gx[2:]))
    d5 = CU.deconv(gx[0], [2, 3], 'FlownetS/deconv5', [4, 4, 256, 128], params=gp)
    got = CU.conv(torch.cat([d5, gx[1]], 3), 'FlownetS/flow5', [3, 3, 384, 2], 1, activation=CU.identity, params=gp)
    dgot = torch.autograd.grad((got * up.cuda()).sum(), gx)
    rels = [_rel_l2(a, b) for a, b in zip(dgot, dref)]
    print('MEASURED recover decoder step: out %.2e grads %s' % (_rel_l2(got, ref), ' '.join('%.2e' % r for r in rels)))
    assert _rel_l2(got, ref) <= OUT_TOL
    assert max(rels) <= GRAD_TOL_LEAKY          # deconv5 is a leaky layer; measured out 2.8e-3, gradients <= 3.2e-2

"""Shared helpers for the conv-engine parity tests: run one layer through the product engine (libcis_b200.so) and
through a plain torch fp32 reference fed with the SAME bf16-rounded operands."""
import torch
import torch.nn.functional as F

from unsupervised_detection_b200 import engine as E
from unsupervised_detection_b200._lib import ACT_NONE, ACT_ELU, ACT_LEAKY
from oracle import tf_ops as T


def bf(x):
    return x.to(torch.bfloat16).float()


def ref_act(y, act, alpha):
    if act == ACT_ELU:
        return F.elu(y)
    if act == ACT_LEAKY:
        return F.leaky_relu(y, alpha)
    return y


def run_conv_case(N, H, W, cins, cout, k, stride=1, dil=1, act=ACT_NONE, alpha=0.2, bn=False, seed=0, post_add=False, backward=True,
                  n_mod_last=0, dev='cuda', bn_cap=None):
    """Returns dict of max-abs errors (and reference scales) for forward / dgrad / wgrad / bias grad."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    store = E.ParamStore(dev)
    cin = sum(cins)
    layer = E.ConvLayer(store, 'L', k, cin, cout, stride, dil, act, alpha, tag='R', bn=bn, bn_cap=bn_cap)
    store.finalize(True)
    w = bf(torch.randn(k, k, cin, cout, generator=g) * (1.0 / (k * k * cin) ** 0.5))
    b = torch.randn(cout, generator=g) * 0.1
    params = {'L/kernel': w, 'L/bias': b}
    if bn:
        params['L/gamma'] = 1.0 + 0.2 * torch.randn(cout, generator=g)
        params['L/beta'] = 0.1 * torch.randn(cout, generator=g)
    store.load(params)
    B = E.Builder(dev)
    srcs, xs = [], []
    for i, c in enumerate(cins):
        nm = n_mod_last if (i == len(cins) - 1 and n_mod_last) else 0
        n_i = nm if nm else N
        a = B.new_act(n_i, H, W, c, name='x%d' % i, dep={'R'}, n_mod=nm)
        x = bf(torch.randn(n_i, H, W, c, generator=g))
        a.buf[..., :c] = x.to(dev).to(torch.bfloat16)
        srcs.append(a)
        xs.append(x)
    OH, OW = -(-H // stride), -(-W // stride)
    pa = None
    res = None
    if post_add:
        pa = B.new_act(N, OH, OW, cout, name='res', dep={'R'})
        res = bf(torch.randn(N, OH, OW, cout, generator=g))
        pa.buf[..., :cout] = res.to(dev).to(torch.bfloat16)
    pack = E.Plan('pack')
    out = B.conv(layer, srcs, post_add=pa)
    # reference (fp32 on the same device)
    xcat = torch.cat([x.to(dev) if not s.n_mod else x.to(dev).repeat(N // s.n_mod, 1, 1, 1) for x, s in zip(xs, srcs)], 3).requires_grad_(True)
    wd = w.to(dev).clone().requires_grad_(True)
    bd = b.to(dev).clone().requires_grad_(True)
    if bn:
        gam = params['L/gamma'].to(dev).clone().requires_grad_(True)
        bet = params['L/beta'].to(dev).clone().requires_grad_(True)
        # the engine folds BN into bf16 weights: reference uses the same folded+rounded weights for forward checks
        s_ = 1.0 / (1.0 + 1e-3) ** 0.5
        w_eff = (wd * gam * s_)
        w_used = w_eff + (bf(w_eff.detach()) - w_eff.detach())   # straight-through rounding
        b_used = bd * gam * s_ + bet
    else:
        w_used, b_used = wd, bd
    y = T.conv2d_same(xcat, w_used, stride, dil, b_used)
    y = ref_act(y, act, alpha)
    if post_add:
        y = y + res.to(dev)
    layer.plan_pack(pack, dgrad=False)
    pack.run()
    B.fwd.run()
    torch.cuda.synchronize()
    got = out.float()
    r = dict(fwd_err=float((got - y.detach()).abs().max()), fwd_ref=float(y.detach().abs().max()))
    if not backward:
        return r
    gy = bf(torch.randn(N, OH, OW, cout, generator=g)).to(dev)
    out.get_grad().buf[..., :cout] = gy.to(torch.bfloat16)
    bp = B.build_backward('R', [out])
    pre = E.Plan('pre')
    layer.plan_pack(pre, dgrad=True)
    store.grad.zero_()
    pre.run()
    bp.run()
    fin = E.Plan('fin')
    layer.plan_finalize(fin, 'R')
    fin.run()
    torch.cuda.synchronize()
    grads = torch.autograd.grad(y, [xcat, wd, bd] + ([gam, bet] if bn else []), gy)
    off = 0
    dx_err, dx_ref = 0.0, 0.0
    for s, x in zip(srcs, xs):
        ref = grads[0][..., off:off + s.C]
        if s.n_mod:
            ref = ref.reshape(N // s.n_mod, s.n_mod, H, W, s.C).sum(0)
        gotx = s.grad.float()
        dx_err = max(dx_err, float((gotx - ref).abs().max()))
        dx_ref = max(dx_ref, float(ref.abs().max()))
        off += s.C
    r.update(dx_err=dx_err, dx_ref=dx_ref)
    dw = store.view('L/kernel', 'grad')
    r.update(dw_err=float((dw - grads[1]).abs().max()), dw_ref=float(grads[1].abs().max()))
    db = store.view('L/bias', 'grad')
    r.update(db_err=float((db - grads[2]).abs().max()), db_ref=float(grads[2].abs().max()))
    if bn:
        r.update(dgamma_err=float((store.view('L/gamma', 'grad') - grads[3]).abs().max()), dgamma_ref=float(grads[3].abs().max()),
                 dbeta_err=float((store.view('L/beta', 'grad') - grads[4]).abs().max()), dbeta_ref=float(grads[4].abs().max()))
    return r

"""Gradients of the function-level API (models/functional.py) without a GPU: the backward plans of the generator / recover runners are
BUILT on CPU tensors and inspected, the autograd plumbing (runner pool, parameter gradients) runs with the plan replay stubbed out, and
the kernel calls of the thin wrappers' backward are recorded.  The numerical checks live in test_functional_grad_gpu.py."""
import collections

import pytest
import torch

from unsupervised_detection_b200 import engine, params_init
from unsupervised_detection_b200.models import functional as F


def _names(plan):
    return [op[2] for op in plan.ops if op[0] is not None]


@pytest.fixture
def stubbed(monkeypatch):
    """Plans are built for real but never replayed; kernel calls of the thin wrappers are recorded."""
    calls = []
    monkeypatch.setattr(engine.Plan, 'run', lambda self, stream=None, lane_key=0: None)
    monkeypatch.setattr(F._lib, 'call', lambda name, *a: calls.append((name, a)))
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_stream', lambda: 0)
    monkeypatch.setattr(F, '_RUNNERS', {})
    monkeypatch.setattr(F, '_POOLS', {})
    return calls


def test_generator_backward_plan_reaches_conv1_data_gradient():
    r = F._GeneratorRunner(2, 32, 48, 'cpu', 'MaskNet')
    assert r.bwd is None
    r.ensure_backward()
    n = collections.Counter(_names(r.bwd))
    assert n['cis_conv_wgrad'] == 17 and n['cis_mask_bwd'] == 1
    assert _names(r.bwd)[0] == 'cis_mask_bwd'
    seed = r.bwd.ops[0][1]
    assert seed[0] is None and seed[3] is None and seed[4:6] == (2, 32 * 48)          # no flow, no recover-input chain
    assert r.gen_in.grad_written.get('G') and r.gen_in.grad is not None                # conv1's data gradient is emitted
    casts = [op[1] for op in r.bwd.ops if op[2] == 'cis_cast_bf16_to_f32']
    assert [(c[3], c[4]) for c in casts] == [(0, 3), (3, 2)]                           # image = channels 0-2, flow = 3-4
    assert all(c[0] == r.gen_in.grad.ptr for c in casts)
    assert n['cis_param_multi'] >= 2                                                    # un-pack + BN chain, batched
    assert r.store.grad.shape == r.store.flat.shape
    # the pack plan now also builds the data-gradient operands
    assert sum(1 for x in _names(r.pack) if x.startswith('cis_pack_weights')) > 17


def test_recover_backward_plan_reaches_both_inputs():
    r = F._RecoverRunner(1, 64, 96, 'cpu', 'FlownetS', 0.25)
    assert r.bwd is None
    r.ensure_backward()
    names = _names(r.bwd)
    assert collections.Counter(names)['cis_conv_wgrad'] == 32
    assert names[0] == 'cis_resize_f32_bwd_to_bf16'
    seed = r.bwd.ops[0][1]
    assert seed[1:7] == (1, 64, 96, 2, 32, 48) and seed[7] == r.net.flow1.grad.ptr
    assert r.img8.grad_written.get('R') and r.flow_in.grad_written.get('R')
    tail = [(op[2], op[1]) for op in r.bwd.ops[-3:]]
    assert tail[0][0] == 'cis_cast_bf16_to_f32' and tail[0][1][0] == r.img8.grad.ptr and tail[0][1][3:5] == (0, 3)
    assert tail[1][0] == 'cis_cast_bf16_to_f32' and tail[1][1][0] == r.flow_in.grad.ptr and tail[1][1][3:5] == (0, 2)
    assert tail[2][0] == 'cis_cast_bf16_to_f32_scaled' and tail[2][1][3:6] == (3, 1, -1.0)    # mask enters as 1 - mask


def test_forward_plan_is_unchanged_by_the_backward_plan():
    a = F._GeneratorRunner(1, 32, 48, 'cpu', 'MaskNet')
    b = F._GeneratorRunner(1, 32, 48, 'cpu', 'MaskNet')
    b.ensure_backward()
    assert _names(a.bld.fwd) == _names(b.bld.fwd)


def test_call_without_gradients_builds_no_backward_plan(stubbed):
    p = params_init.init_generator()
    out = F.generator_net(torch.zeros(1, 32, 48, 3), torch.zeros(1, 32, 48, 2), params=p)
    assert out.grad_fn is None and not out.requires_grad
    (r,) = F._RUNNERS.values()
    assert r.bwd is None and not F._POOLS
    pr = params_init.init_recover()
    out = F.recover_net(torch.zeros(1, 32, 48, 3), torch.zeros(1, 32, 48, 2), torch.zeros(1, 32, 48, 1), params=pr)
    assert out.grad_fn is None and all(r.bwd is None for r in F._RUNNERS.values()) and not F._POOLS
    x = torch.zeros(1, 32, 48, 3, requires_grad=True)
    with torch.no_grad():
        F.generator_net(x, torch.zeros(1, 32, 48, 2), params=p)
    assert not F._POOLS


def test_outstanding_gradient_calls_use_separate_runners(stubbed):
    p = {k: v.clone().requires_grad_(True) for k, v in params_init.init_recover().items()}
    img = torch.rand(1, 32, 48, 3)
    fm = torch.zeros(1, 32, 48, 2, requires_grad=True)
    m = torch.rand(1, 32, 48, 1, requires_grad=True)
    outs = [F.recover_net(img, fm, m, params=p) for _ in range(3)]
    leases = [o.grad_fn.lease for o in outs]
    runners = [l.runner for l in leases]
    assert len({id(r) for r in runners}) == 3                                          # three instances of one shape
    (free,) = F._POOLS.values()
    assert free == [] and all(r.bwd is not None for r in runners)
    sum(o.sum() for o in outs).backward()
    assert len(free) == 3 and all(l.runner is None for l in leases)                    # all returned after their backward
    assert fm.grad.shape == fm.shape and m.grad.shape == m.shape and img.grad is None
    assert all(p[n].grad is not None and p[n].grad.shape == p[n].shape for n in p if n.startswith('FlownetS/'))
    again = F.recover_net(img, fm, m, params=p)                                         # reuses a pooled instance, builds nothing new
    assert len(free) == 2 and any(again.grad_fn.lease.runner is r for r in runners)
    del again                                                                           # released with its autograd context
    assert len(free) == 3


def test_backward_refuses_a_rerun_runner(stubbed):
    p = params_init.init_generator()
    x = torch.zeros(1, 32, 48, 3, requires_grad=True)
    out = F.generator_net(x, torch.zeros(1, 32, 48, 2), params=p)
    out.grad_fn.lease.runner.runs += 1
    with pytest.raises(RuntimeError, match='re-run'):
        out.sum().backward()


def test_thin_wrappers_record_their_backward_kernels(stubbed):
    calls = stubbed
    gt, pr = torch.randn(2, 6, 5, 2, requires_grad=True), torch.randn(2, 6, 5, 2, requires_grad=True)
    mask = torch.rand(2, 6, 5, 1, requires_grad=True)
    F.charbonnier_loss(gt, pr, mask, cbn=0.3).sum().backward()
    name, a = calls[-1]
    assert name == 'cis_charbonnier_bwd' and a[3:8] == (2, 30, 2, 1, 0.3) and all(x is not None for x in a[9:12])
    assert gt.grad.shape == gt.shape and mask.grad.shape == mask.shape
    F.charbonnier_loss(gt.detach(), pr, torch.ones(2, 6, 5, 2)).sum().backward()
    name, a = calls[-1]
    assert a[6] == 2 and a[9] is not None and a[10] is None and a[11] is None        # only dpred wanted
    n0 = len(calls)
    F.charbonnier_loss(gt.detach(), pr.detach(), mask.detach())
    assert [c[0] for c in calls[n0:]] == ['cis_charbonnier_sum']                       # no gradient: forward only

    c1 = torch.randn(1, 6, 10, 196, requires_grad=True)
    wp = torch.randn(1, 6, 10, 196, requires_grad=True)
    F.cost_volume(c1, wp).sum().backward()
    name, a = calls[-1]
    assert name == 'cis_cost_volume_bwd' and a[1] == 200 and a[4] == 200 and a[7:11] == (1, 6, 10, 196)
    assert c1.grad.shape == c1.shape and wp.grad.shape == wp.shape

    img = torch.randn(2, 4, 4, 5, requires_grad=True)
    fl = torch.zeros(2, 4, 4, 2, requires_grad=True)
    F.dense_image_warp(img, fl).sum().backward()
    name, a = calls[-1]
    assert name == 'cis_dense_image_warp_bwd' and a[1] == 8 and a[4:9] == (1.0, 2, 4, 4, 5)
    assert a[10] is not None and a[11] is not None and a[12] is not None              # dimage, fp64 scratch, dflow
    assert img.grad.shape == img.shape and fl.grad.shape == fl.shape
    F.dense_image_warp(img.detach(), fl).sum().backward()
    assert calls[-1][1][10] is None and calls[-1][1][11] is None                       # flow only: no scatter, no scratch

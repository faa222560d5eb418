"""Gradients through ModelPWCNet.predict_from_img_pairs without a GPU: the backward plan of a trainable PWC-Net runner is BUILT on CPU
tensors and inspected, and the autograd plumbing runs with the plan replay stubbed out.  The numerical checks live in
test_pwc_grad_gpu.py."""
import collections

import pytest
import torch

from oracle import params as OP
from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.models import functional as F
from unsupervised_detection_b200.models.PWCNet import model_pwcnet as MP

B, H, W = 2, 128, 192


def _names(plan):
    return [op[2] for op in plan.ops if op[0] is not None]


def _ops(plan, name):
    return [op[1] for op in plan.ops if op[2] == name]


@pytest.fixture(scope='module')
def runner():
    r = F._PWCRunner(B, H, W, 'cpu', 'pwcnet', trainable=True)
    r.ensure_backward()
    return r


def _unpack_jobs(r):
    """Every cis_unpack_wgrad of the finalize step (batched or single) as (dw pointer, nsplit, layout)."""
    from unsupervised_detection_b200._lib import CisParamJob, JOB_UNPACK
    out = []
    for fn, a, name, _, _ in r.bwd.ops:
        if name == 'cis_unpack_wgrad':
            out.append((a[5], a[4], a[10]))
        elif name == 'cis_param_multi':
            tab = next(t for t in r.bwd.keep if isinstance(t, torch.Tensor) and t.data_ptr() == a[0])
            jobs = (CisParamJob * a[1]).from_buffer_copy(bytes(tab.numpy()))
            out += [(j.p[2], j.i[2], j.i[5]) for j in jobs if j.kind == JOB_UNPACK]
    return out


def test_every_pwcnet_layer_has_a_weight_gradient(runner):
    r = runner
    s = r.store
    jobs = _unpack_jobs(r)
    dws = collections.Counter(p for p, _, _ in jobs)
    for L in r.layers:
        base = s.ptr(L.wkey, 'grad')
        assert L.dgrad_used or L.tr_dgrad is not None, L.name                       # data gradient emitted
        if L.transposed:
            assert dws[base] == 4, L.name                                             # one job per output parity
            assert all(lay == 1 | (L.cin << 8) for p, _, lay in jobs if p == base)  # [kh,kw,Cout,Cin] slot: n stride Cin
        else:
            assert dws[base] == 1, L.name
            if L.cout > 128:                                                          # channels >= 128 in a launch of their own
                assert dws[base + 4 * 128] == 1, L.name


def test_feature_pyramid_slices_cover_both_frames(runner):
    r = runner
    wg = [op[1][0]._obj for op in r.bwd.ops if op[2] == 'cis_conv_wgrad']
    for L in r.layers:
        if '/featpyr/' not in L.name:
            continue
        assert L.ncalls == 2
        mine = [w for w in wg if w.dwp in range(L.dwp.data_ptr(), L.dwp.data_ptr() + 4 * L.dwp.numel())]
        assert len(mine) == 2, L.name
        per = mine[0].splits
        assert mine[1].splits == per and L.wg_splits['P'] == 2 * per
        offs = sorted(w.dwp - L.dwp.data_ptr() for w in mine)
        assert offs == [0, 4 * per * min(L.cout, 128) * L.wg_K_pad]                  # second call's slices follow the first's
        assert L.col_blocks['P'] % 2 == 0 and L.colpart.numel() >= 2 * 592 * L.cout


def test_one_warp_costvol_backward_per_level(runner):
    r = runner
    cv = _ops(r.bwd, 'cis_warp_costvol_bwd')
    assert len(cv) == 5
    levels = {a[9]: a for a in cv}                      # keyed by the map height
    for l in range(MP.FLOW_PRED_LVL, MP.PYR_LVLS + 1):
        a = levels[H >> l]
        assert a[11] == MP.NUM_CHANN[l]
        assert (a[6] is None) == (l == MP.PYR_LVLS)     # flow only below level 6
        assert a[12] == r.net.level_grad[l].data_ptr() and a[14] == MP.CORR_OFF
        if l != MP.PYR_LVLS:
            assert a[15] == a[12] and a[17] == MP.C1_OFF                        # dc1 into the c1 slice of dE[l]
            assert a[21] == a[12] and a[23] == MP.C1_OFF + MP.NUM_CHANN[l]      # d(up_flow) into its tail slice
            assert a[24] & 5 == 5                                               # both accumulate into the zeroed dE[l]


def test_seed_and_input_casts(runner):
    r = runner
    names = [n for n in _names(r.bwd) if n != 'cis_zero']                              # the level gradients are zeroed first
    assert names[0] == 'cis_resize_f32_bwd_to_bf16_scaled' and names.count('cis_resize_f32_bwd_to_bf16_scaled') == 1
    seed = _ops(r.bwd, 'cis_resize_f32_bwd_to_bf16_scaled')[0]
    fg = r.net.flows_bf[MP.FLOW_PRED_LVL].grad
    assert seed[1:7] == (B, H, W, 2, H // 4, W // 4) and seed[7] == fg.ptr and seed[9] == 4.0
    zeroed = {op[1][0] for op in r.bwd.ops if op[2] == 'cis_zero'}
    assert {g.data_ptr() for g in r.net.level_grad.values()} <= zeroed
    casts = _ops(r.bwd, 'cis_cast_bf16_to_f32')
    assert [(c[0], c[3], c[4]) for c in casts] == [(r.i1.grad.ptr, 0, 3), (r.i2.grad.ptr, 0, 3)]
    assert [c[5] for c in casts] == [r.dimg1.data_ptr(), r.dimg2.data_ptr()]


def test_forward_plan_does_not_depend_on_training():
    a = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet')
    b = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True)
    c = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True)
    c.ensure_backward()
    assert _names(a.bld.fwd) == _names(b.bld.fwd) == _names(c.bld.fwd)
    assert not a.bld.tape and all(not L.tag for L in a.layers)
    conv = lambda r: [bytes(op[1][0]._obj)[:8 * 4] for op in r.bld.fwd.ops if op[2] == 'cis_conv_igemm']   # N, H, W, OH, OW, strides, taps
    assert conv(a) == conv(b) == conv(c)


def test_step_graph_keeps_pwcnet_frozen():
    from unsupervised_detection_b200.step_graph import CISGraph
    g = CISGraph(128, 192, 1, device='cpu', with_pwc=True)
    assert not g.pwc.trainable and all(L.tag == '' for L in g.pwc.all_layers())
    for L in g.pwc.all_layers():
        assert L.wg_kmap is None and L.dwp is None and L.tr_dgrad is None and L.dgrad_packs is None and L.ncalls == 0
    # no backward launch of the recover / generator steps reads a PWC-Net operand or level buffer
    pwc = {t.data_ptr() for t in g.pwc.level_buf.values()}
    for L in g.pwc.all_layers():
        pwc |= {t.data_ptr() for pk in [L.fwd_pack] + (L.tr_packs or []) if pk is not None for t in (pk.w, pk.wt) if t is not None}
    assert set(g.bwd) == {'R', 'G'}
    for plan in g.bwd.values():
        for op in plan.ops:
            if op[2] in ('cis_conv_igemm', 'cis_conv_wgrad'):
                d = op[1][0]._obj
                ptrs = {d.src[i].ptr for i in range(d.nsrc)} | {getattr(d, 'wpack', None)}
                assert not (ptrs & pwc), op[2]


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(engine.Plan, 'run', lambda self, stream=None, lane_key=0: None)
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_RUNNERS', {})
    monkeypatch.setattr(F, '_POOLS', {})


def _params(grad):
    p = OP.make_params(11, jitter=0.05, nets=('pwcnet',))
    return {k: v.requires_grad_(grad) for k, v in p.items()}


def test_call_without_gradients_builds_no_backward_plan(stubbed):
    p = _params(False)
    out = F.predict_from_img_pairs(torch.zeros(1, 128, 192, 3), torch.zeros(1, 128, 192, 3), params=p)
    assert out.grad_fn is None and not out.requires_grad
    (r,) = F._RUNNERS.values()
    assert r.bwd is None and not r.net.trainable and not F._POOLS
    with pytest.raises(ValueError, match='multiples of 64'):
        F.predict_from_img_pairs(torch.zeros(1, 100, 192, 3), torch.zeros(1, 100, 192, 3), params=p)


def test_gradient_calls_lease_runners_and_fill_parameter_grads(stubbed):
    p = _params(True)
    img1 = torch.rand(1, 128, 192, 3, requires_grad=True)
    img2 = torch.rand(1, 128, 192, 3)
    outs = [F.predict_from_img_pairs(img1, img2, params=p) for _ in range(2)]
    runners = [o.grad_fn.lease.runner for o in outs]
    assert runners[0] is not runners[1] and all(r.net.trainable and r.bwd is not None for r in runners)
    (free,) = F._POOLS.values()
    (outs[0] + outs[1]).sum().backward()
    assert len(free) == 2
    assert img1.grad.shape == img1.shape and img2.grad is None
    names = [n for n in p if n.startswith('pwcnet/')]
    assert names and all(p[n].grad is not None and p[n].grad.shape == p[n].shape for n in names)
    tr = [n for n in names if '/upsample/' in n and n.endswith('/kernel')]
    assert tr and all(p[n].grad.shape[2:] == (2, p[n].shape[3]) for n in tr)        # [kh,kw,Cout,Cin]


def test_backward_refuses_a_rerun_runner(stubbed):
    p = _params(False)
    x = torch.zeros(1, 128, 192, 3, requires_grad=True)
    out = F.predict_from_img_pairs(x, torch.zeros(1, 128, 192, 3), params=p)
    out.grad_fn.lease.runner.runs += 1
    with pytest.raises(RuntimeError, match='re-run'):
        out.sum().backward()

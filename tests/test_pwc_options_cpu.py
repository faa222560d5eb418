"""PWC-Net options without a GPU (models/PWCNet/model_pwcnet.py: use_dense_cx, use_res_cx, search_range 1..4): parameter tables, level
layout, launch plans, the public ModelPWCNet(name, options) class and the option checks.  The numerical checks live in
test_pwc_options_gpu.py."""
import collections

import pytest
import torch

import plan_digest
import pwc_options_ref as REF
from oracle import params as OP
from unsupervised_detection_b200 import engine
from unsupervised_detection_b200.engine import ParamStore
from unsupervised_detection_b200.models import functional as F
from unsupervised_detection_b200.models.PWCNet import model_pwcnet as MP
from unsupervised_detection_b200.models.PWCNet.model_pwcnet import ModelPWCNet, PWCNetBuilder

SM = {'use_dense_cx': False, 'use_res_cx': True}
# parameter counts of the four networks, model_pwcnet.py:15-18 of the reference
COUNTS = {(True, True): 14079050, (True, False): 9374274, (False, True): 6774064, (False, False): 4705064}


def _builder(options=None):
    st = ParamStore('cpu')
    b = PWCNetBuilder(st, options=options)
    st.finalize(False)
    return b, st


def _names(plan):
    return [op[2] for op in plan.ops if op[0] is not None]


def _ops(plan, name):
    return [op[1] for op in plan.ops if op[2] == name]


def _convs(plan):
    return [op[1][0]._obj for op in plan.ops if op[2] == 'cis_conv_igemm']


@pytest.mark.parametrize('dense,res', sorted(COUNTS))
def test_parameter_counts_match_the_reference(dense, res):
    o = {'use_dense_cx': dense, 'use_res_cx': res}
    b, st = _builder(o)
    assert st.real_count() == COUNTS[dense, res]
    assert REF.param_count(o) == COUNTS[dense, res]
    # the builder's layers and the reference table agree layer by layer
    tab = {n: (k, ci, co, tr) for n, k, ci, co, tr in REF.pwc_layers(o)}
    assert {n: (L.k, L.cin, L.cout, L.transposed) for n, L in b.L.items()} == tab


def test_default_reference_tables_are_the_oracle():
    assert REF.pwc_layers() == OP.pwc_layers() and REF.default_tables_match_oracle()
    a, b = REF.make_params(5, jitter=0.05), OP.make_params(5, jitter=0.05, nets=('pwcnet',))
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('dense', [True, False])
def test_search_range_changes_the_corr_slice_and_its_readers(dense):
    b4, _ = _builder({'use_dense_cx': dense})
    b3, _ = _builder({'use_dense_cx': dense, 'search_range': 3})
    assert (b4.ndisp, b4.corr_pad, b4.c1_off) == (81, MP.CORR_PAD, MP.C1_OFF)
    assert (b3.ndisp, b3.corr_pad, b3.c1_off) == (49, 56, MP.CORR_OFF + 56)
    for l in range(2, 7):
        assert b4.level_pitch(l) - b3.level_pitch(l) == 32
    changed = {n for n in b4.L if b4.L[n].cin != b3.L[n].cin}
    assert all(b4.L[n].cin - b3.L[n].cin == 32 for n in changed)
    if dense:    # every estimator input, the flow head, the context net's first conv and up_feat read the correlation
        want = {'predict_flow/conv%d_%d' % (l, i) for l in range(2, 7) for i in range(5)}
        want |= {'predict_flow/flow%d' % l for l in range(2, 7)} | {'ctxt/dc_conv%d1' % l for l in range(2, 7)}
        want |= {'upsample/up_feat%d' % l for l in range(3, 7)}
    else:        # only conv{l}_0 reads it
        want = {'predict_flow/conv%d_0' % l for l in range(2, 7)}
    assert changed == want
    assert b3.L['predict_flow/conv6_0'].cin == 49 and b3.L['predict_flow/conv5_0'].cin == 49 + 128 + 4
    assert b3._chanmap(5, MP.A_TOTAL)[:56] == list(range(49)) + [-1] * 7


def test_dense_off_plan_reads_single_slices():
    r = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', options=SM)
    net = r.net
    assert net.options.use_dense_cx is False
    convs = _convs(r.bld.fwd)
    for l in range(2, 7):
        for i in range(1, 5):
            L = net.L['predict_flow/conv%d_%d' % (l, i)]
            assert L.cin == MP.DENSE[i - 1]
        assert net.L['predict_flow/flow%d' % l].cin == 32
        assert net.L['ctxt/dc_conv%d1' % l].cin == 32
        if l != 2:
            assert net.L['upsample/up_feat%d' % l].cin == 32
    # the estimator convs of one level: conv_0 reads [corr | c1 | up] from A_TOTAL, conv_i one 8-aligned slice act_{i-1}
    level_buf = {t.data_ptr(): l for l, t in net.level_buf.items()}
    by_level = collections.defaultdict(list)
    for d in convs:
        if d.nsrc == 1 and d.src[0].ptr in level_buf and d.out in level_buf and d.out_coff in MP.A_OFF:
            by_level[level_buf[d.src[0].ptr]].append(d)
    for l, ds in by_level.items():
        assert len(ds) == 5, l
        assert ds[0].src[0].c_off == MP.A_TOTAL
        for i, d in enumerate(ds[1:], start=1):
            assert (d.src[0].c_off, d.src[0].chunks, d.out_coff) == (MP.A_OFF[i - 1], MP.DENSE[i - 1] // 8, MP.A_OFF[i])


def test_residual_off_drops_the_context_net_above_the_prediction_level():
    lg = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet')
    nr = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', options={'use_res_cx': False})
    names = set(nr.net.L)
    for l in range(3, 7):
        assert not any(n.startswith('ctxt/dc_conv%d' % l) for n in names)
        assert nr.net.flows_bf[l].name == 'predict_flow/flow%d' % l
    assert {'ctxt/dc_conv2%d' % i for i in range(1, 8)} <= names       # refine_flow stays at the prediction level
    assert nr.net.flows_bf[2].name == 'ctxt/dc_conv27'
    n_lg, n_nr = collections.Counter(_names(lg.bld.fwd)), collections.Counter(_names(nr.bld.fwd))
    assert n_lg['cis_conv_igemm'] - n_nr['cis_conv_igemm'] == 4 * 7
    # the flow heads above level 2 write both the fp32 flow and the bf16 flow that up_flow reads
    flows = {nr.net.flows[l].data_ptr(): l for l in range(3, 7)}
    heads = [d for d in _convs(nr.bld.fwd) if d.outf in flows]
    assert len(heads) == 4 and all(d.out == nr.net.flows_bf[flows[d.outf]].ptr and not d.addf_pre for d in heads)


@pytest.mark.parametrize('options', [{'search_range': 3}, {'search_range': 1, 'use_dense_cx': False, 'use_res_cx': False}])
def test_costvol_launches_carry_the_range(options):
    r = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True, options=options)
    r.ensure_backward()
    rng = options['search_range']
    fwd, bwd = _ops(r.bld.fwd, 'cis_warp_costvol_r'), _ops(r.bwd, 'cis_warp_costvol_bwd_r')
    assert len(fwd) == len(bwd) == 5 and not _ops(r.bld.fwd, 'cis_warp_costvol') and not _ops(r.bwd, 'cis_warp_costvol_bwd')
    assert all(a[15] == rng and a[14] == MP.CORR_OFF for a in fwd)
    assert all(a[28] == rng and a[14] == MP.CORR_OFF for a in bwd)
    for a in bwd:
        l = {128 >> k: k for k in range(2, 7)}[a[9]]
        assert a[13] == r.net.level_pitch(l)
        if l != 6:
            assert a[17] == r.net.c1_off and a[23] == r.net.c1_off + MP.NUM_CHANN[l]
    gs = r.net.cv_scratch[0]
    assert gs.numel() == 32 * 48 * (2 * rng + 1) ** 2


def test_default_range_keeps_the_range_free_entry_points():
    r = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True, options={'search_range': 4})
    r.ensure_backward()
    assert len(_ops(r.bld.fwd, 'cis_warp_costvol')) == len(_ops(r.bwd, 'cis_warp_costvol_bwd')) == 5
    assert not any(n.endswith('_r') for n in _names(r.bld.fwd) + _names(r.bwd))


def test_none_and_an_explicit_copy_of_the_defaults_give_the_same_plans():
    from unsupervised_detection_b200.step_graph import CISGraph
    with plan_digest.filled_uninitialized():
        a = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True)
        b = F._PWCRunner(1, 128, 192, 'cpu', 'pwcnet', trainable=True, options=dict(MP._DEFAULT_PWCNET_TEST_OPTIONS))
        a.ensure_backward()
        b.ensure_backward()
        g1 = CISGraph(128, 192, 1, device='cpu', with_pwc=True)
        g2 = CISGraph(128, 192, 1, device='cpu', with_pwc=True, pwc_options=dict(MP._DEFAULT_PWCNET_TEST_OPTIONS))
    assert a.net.options == b.net.options == MP.normalize_options(None)
    assert plan_digest.digest(plan_digest.runner_plans(a)) == plan_digest.digest(plan_digest.runner_plans(b))
    assert plan_digest.digest([('fwd', g1.bld.fwd)]) == plan_digest.digest([('fwd', g2.bld.fwd)])


def test_step_graph_takes_the_options():
    from unsupervised_detection_b200.step_graph import CISGraph
    g = CISGraph(64, 96, 1, device='cpu', pwc_hw=(128, 192), pwc_options=SM)
    assert g.pwc.options.use_dense_cx is False and g.pwc_store.real_count() == COUNTS[False, True]
    assert not g.pwc.trainable and all(L.tag == '' for L in g.pwc.all_layers())


def test_model_pwcnet_takes_the_reference_signature():
    m = ModelPWCNet()
    assert m.name == 'pwcnet' and m.opts is MP._DEFAULT_PWCNET_TEST_OPTIONS and m.options == MP.normalize_options(None)
    assert set(MP._DEFAULT_PWCNET_TEST_OPTIONS) == {'verbose', 'ckpt_path', 'pyr_lvls', 'flow_pred_lvl', 'search_range', 'use_dense_cx',
                                                    'use_res_cx'}
    sm = ModelPWCNet('pwcnet', dict(MP._DEFAULT_PWCNET_TEST_OPTIONS, use_dense_cx=False, verbose=True, ckpt_path='x'))
    assert sm.options == MP.PWCOptions(6, 2, 4, False, True)
    with pytest.raises(TypeError, match='PWCNetBuilder'):
        ModelPWCNet(ParamStore('cpu'))


@pytest.mark.parametrize('bad', [{'pyr_lvls': 7}, {'flow_pred_lvl': 3}, {'search_range': 0}, {'search_range': 5}, {'search_range': 2.5}])
def test_out_of_scope_options_raise(bad):
    o = dict(MP._DEFAULT_PWCNET_TEST_OPTIONS, **bad)
    with pytest.raises(ValueError, match='supported'):
        ModelPWCNet(options=o)
    with pytest.raises(ValueError, match='supported'):
        PWCNetBuilder(ParamStore('cpu'), options=o)
    with pytest.raises(ValueError, match='supported'):
        F._PWCRunner(1, 64, 64, 'cpu', 'pwcnet', options=o)


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(engine.Plan, 'run', lambda self, stream=None, lane_key=0: None)
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_RUNNERS', {})
    monkeypatch.setattr(F, '_POOLS', {})


def test_both_call_forms_run_their_options(stubbed):
    x = torch.zeros(1, 128, 192, 3)
    p_lg, p_sm = REF.make_params(3), REF.make_params(3, options=SM)
    ModelPWCNet.predict_from_img_pairs(x, x, params=p_lg)                        # unbound: the default options
    ModelPWCNet(options=SM).predict_from_img_pairs(x, x, params=p_sm)           # the reference's form: the instance's options
    ModelPWCNet().predict_from_img_pairs(x, x, params=p_lg)                      # same options as the unbound call: same runner
    assert len(F._RUNNERS) == 2
    opts = sorted((r.net.options for r in F._RUNNERS.values()), key=lambda o: o.use_dense_cx)
    assert opts == [MP.PWCOptions(6, 2, 4, False, True), MP.normalize_options(None)]
    with pytest.raises(ValueError, match='shape mismatch'):                      # same variable names, the sm network's own shapes
        ModelPWCNet(options=SM).predict_from_img_pairs(x, x, params=p_lg)


def test_gradient_calls_lease_runners_per_option_set(stubbed):
    x = torch.zeros(1, 128, 192, 3, requires_grad=True)
    p = {k: v.requires_grad_(True) for k, v in REF.make_params(3, options=SM).items()}
    out = ModelPWCNet(options=SM).predict_from_img_pairs(x, torch.zeros(1, 128, 192, 3), params=p)
    r = out.grad_fn.lease.runner
    assert r.net.trainable and r.net.options.use_dense_cx is False
    (key,) = F._POOLS
    assert key[-1] == MP.PWCOptions(6, 2, 4, False, True)
    out.sum().backward()
    assert x.grad.shape == x.shape and all(p[n].grad is not None and p[n].grad.shape == p[n].shape for n in p)


def test_cost_volume_r_issues_the_range_entry_points(monkeypatch):
    calls = []
    monkeypatch.setattr(F._lib, 'call', lambda name, *a: calls.append((name, a)))
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_stream', lambda: 0)
    c1, wp = torch.randn(1, 6, 10, 196), torch.randn(1, 6, 10, 196)
    for fn in (lambda: F.cost_volume(c1, wp), lambda: F.cost_volume_r(c1, wp, 4)):       # range 4: exactly cost_volume's launch
        cv = fn()
        name, a = calls[-1]
        assert name == 'cis_warp_costvol' and cv.shape == (1, 6, 10, 81) and a[13:15] == (88, 0) and len(a) == 16
    cv = F.cost_volume_r(c1, wp, 3)                                              # ranges 1..3: the entry point with a range argument
    name, a = calls[-1]
    assert name == 'cis_warp_costvol_r' and cv.shape == (1, 6, 10, 49) and a[13:16] == (56, 0, 3) and a[8:12] == (1, 6, 10, 196)
    for bad in (0, 5, True):
        with pytest.raises(NotImplementedError):
            F.cost_volume_r(c1, wp, bad)
    with pytest.raises(NotImplementedError, match='cost_volume_r'):               # the reference-signature op keeps range 4
        F.cost_volume(c1, wp, search_range=3)
    from unsupervised_detection_b200.models.PWCNet.core_costvol import cost_volume_r
    assert cost_volume_r is F.cost_volume_r


def test_cost_volume_backward_entry_point_follows_the_range(monkeypatch):
    calls = []
    monkeypatch.setattr(F._lib, 'call', lambda name, *a: calls.append((name, a)))
    monkeypatch.setattr(F, '_check_cuda', lambda *t: None)
    monkeypatch.setattr(F, '_stream', lambda: 0)
    c1, wp = torch.randn(1, 6, 10, 20, requires_grad=True), torch.randn(1, 6, 10, 20, requires_grad=True)
    F.cost_volume_r(c1, wp, 2).sum().backward()
    name, a = calls[-1]
    assert name == 'cis_cost_volume_bwd_r' and a[7:11] == (1, 6, 10, 20) and a[-2] == 2
    gs = a[11]
    assert c1.grad.shape == c1.shape and wp.grad.shape == wp.shape and isinstance(gs, int)

"""Moving average of the weights, host side: --ema_decay / --use_ema, the shadow names of the checkpoints and their TF-bundle round trip,
ParamStore's shadow, and the launch plans of CISGraph, the boxes graph and FlowTrainGraph with averaging off (unchanged) and on (one
cis_ema_update after each optimiser launch, nothing else)."""
import math
import os
import re
import sys

import pytest
import torch
from absl import flags as absl_flags

import plan_digest
from unsupervised_detection_b200 import checkpoint as ckpt_io, ema_flags, params_init
from unsupervised_detection_b200.common_flags import FLAG_NAMES, FLAGS, Config
from unsupervised_detection_b200.engine import ParamStore
from unsupervised_detection_b200.flow_train_graph import FlowTrainGraph
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
from unsupervised_detection_b200.step_graph import CISGraph

OPTIMISERS = ('cis_clip_adam', 'cis_adam_l2')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(**kw):
    c = Config()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


# ------------------------------------------------------------------------------------------------ flags
@pytest.mark.parametrize('decay', [0.0, 1e-6, 0.5, 0.999, 0.9999])
def test_ema_decay_accepts_off_and_the_open_unit_interval(decay):
    ema_flags.check(_cfg(ema_decay=decay))


@pytest.mark.parametrize('decay', [-0.1, 1.0, 1.5, math.nan])
def test_ema_decay_outside_the_unit_interval_is_a_usage_error(decay):
    with pytest.raises(absl_flags.IllegalFlagValueError, match='ema_decay'):
        ema_flags.check(_cfg(ema_decay=decay))
    with pytest.raises(ValueError, match='ema_decay'):
        CISGraph(64, 96, 1, device='cpu', with_pwc=False, ema_decay=decay)
    with pytest.raises(ValueError, match='ema_decay'):
        FlowTrainGraph(128, 128, 1, device='cpu', ema_decay=decay)


def test_flags_are_defined_once_outside_the_reference_surface():
    sys.path.insert(0, ROOT)
    import export_flow  # noqa: F401
    import pretrain_recover
    import test_generator  # noqa: F401  (the evaluation scripts take --use_ema through the learner's import of ema_flags)
    import test_generator_ensemble  # noqa: F401
    import train_flow
    assert len(FLAG_NAMES) == 31 and not {'ema_decay', 'use_ema'} & set(FLAG_NAMES)
    assert FLAGS['ema_decay'].default == 0.0 and FLAGS['use_ema'].default is False
    assert 'ema_decay' in pretrain_recover.PRETRAIN_FLAGS and 'ema_decay' in train_flow.TRAIN_FLOW_FLAGS


def test_training_scripts_take_the_decay_and_reject_a_bad_one(monkeypatch, tmp_path):
    sys.path.insert(0, ROOT)
    import pretrain_recover
    import train
    import train_flow
    seen = []
    args = ['--checkpoint_dir=%s' % tmp_path, '--dataset=FLYINGCHAIRS', '--root_dir=%s' % tmp_path]
    try:
        for mod in (train, pretrain_recover, train_flow):
            monkeypatch.setattr(mod, 'run', lambda config: seen.append(config.ema_decay))
            FLAGS.unparse_flags()
            mod.main(['x', '--ema_decay=0.999'] + args)
            FLAGS.unparse_flags()
            with pytest.raises(SystemExit, match='ema_decay'):
                mod.main(['x', '--ema_decay=1.0'] + args)
    finally:
        FLAGS.unparse_flags()
    assert seen == [0.999] * 3


# ------------------------------------------------------------------------------------------------ names and checkpoints
def test_shadow_names_are_tf_moving_average_names():
    assert ckpt_io.ema_name('FlownetS/conv1/weights') == 'FlownetS/conv1/weights/ExponentialMovingAverage'
    cases = {'MaskNet/conv3/gamma': 'MaskNet//batch_normalization_2/gamma',
             'MaskNet/conv13_upsample/kernel': 'MaskNet//conv13_upsample/conv13_upsample_conv/kernel',
             'FlownetS/conv1/weights': 'FlownetS//conv1/weights',
             'pwcnet/featpyr/conv1a/kernel': 'pwcnet/featpyr/conv1a/kernel'}
    for internal, tf in cases.items():
        assert ckpt_io.to_tf_name(internal) == tf
        assert ckpt_io.to_tf_name(ckpt_io.ema_name(internal)) == tf + '/ExponentialMovingAverage'
        assert ckpt_io.to_tf_name(ckpt_io.ema_name(internal), '/') == tf.replace('//', '/') + '/ExponentialMovingAverage'


def _params():
    p = params_init.init_generator()
    p.update(params_init.init_recover())
    return p


def _averaged_graph(decay=0.99, **kw):
    g = CISGraph(64, 96, 1, device='cpu', with_pwc=False, ema_decay=decay, **kw)
    g.load_params(_params())
    return g


def test_param_store_shadow_starts_from_the_loaded_weights_or_the_checkpoint():
    st = ParamStore('cpu')
    st.declare('a/kernel', (3, 1))          # padded to 4
    st.declare('a/bias', (2,))              # padded to 4
    st.finalize(True)
    st.add_shadow()
    st.load({'a/kernel': torch.tensor([[1.0], [2.0], [3.0]]), 'a/bias': torch.tensor([4.0, 5.0])})
    assert st.shadow.tolist() == [1, 2, 3, 0, 4, 5, 0, 0]
    st.load({'a/kernel': torch.zeros(3, 1), 'a/bias': torch.ones(2), 'a/kernel/ExponentialMovingAverage': torch.full((3, 1), 7.0)})
    assert st.flat.tolist() == [0, 0, 0, 0, 1, 1, 0, 0] and st.shadow.tolist() == [7, 7, 7, 0, 1, 1, 0, 0]
    with pytest.raises(ValueError, match='shape mismatch'):
        st.load({'a/kernel': torch.zeros(3), 'a/bias': torch.ones(2), 'a/bias/ExponentialMovingAverage': torch.ones(3)})
    out = st.export_all()
    assert sorted(out) == ['a/bias', 'a/bias/ExponentialMovingAverage', 'a/kernel', 'a/kernel/ExponentialMovingAverage']


def test_averaged_graph_exports_and_round_trips_its_shadows_through_a_tf_bundle(tmp_path):
    g = _averaged_graph()
    torch.manual_seed(0)
    for st in (g.gen_store, g.rec_store):
        for _, _, n, off, _ in st.entries:
            st.shadow[off:off + n] = torch.randn(n)
    assert g.pwc_store.shadow is None
    L = AdversarialLearner()
    L.rank, L.graph, L.global_step = 0, g, 12
    L.save(None, str(tmp_path), 3)
    prefix = str(tmp_path / 'model-3')
    names = L._names('MaskNet', 'FlownetS')
    avg = [ckpt_io.ema_name(n) for n in names]
    held = sorted(v[0] for v in ckpt_io.list_variables(prefix))
    assert held == sorted([ckpt_io.to_tf_name(n) for n in names + avg] + ['train_op/global_step'])
    for path in (prefix, prefix + '.pt'):
        got, gs = AdversarialLearner._read_ckpt(path, names + avg)
        assert gs == 12
        h = CISGraph(64, 96, 1, device='cpu', with_pwc=False, ema_decay=0.5)
        h.load_params(got)
        for a, b in ((g.gen_store, h.gen_store), (g.rec_store, h.rec_store)):
            assert torch.equal(a.flat, b.flat) and torch.equal(a.shadow, b.shadow)
    # averaging off: the same checkpoint loads its plain variables and ignores the averages
    h = CISGraph(64, 96, 1, device='cpu', with_pwc=False)
    h.load_params(AdversarialLearner._read_ckpt(prefix, names + avg)[0])
    assert torch.equal(h.rec_store.flat, g.rec_store.flat) and h.rec_store.shadow is None


def test_resume_restores_the_shadows_or_starts_them_from_the_weights(tmp_path, monkeypatch):
    g = _averaged_graph()
    for st, d in ((g.gen_store, 0.5), (g.rec_store, 0.25)):
        for _, _, n, off, _ in st.entries:
            st.shadow[off:off + n] += d
    L = AdversarialLearner()
    L.rank, L.graph = 0, g
    L.save(None, str(tmp_path / 'with'), 2)
    plain = CISGraph(64, 96, 1, device='cpu', with_pwc=False)
    plain.load_params(g.export_params())
    L.graph = plain
    L.save(None, str(tmp_path / 'without'), 2)
    for sub, with_avg in (('with', True), ('without', False)):
        R = AdversarialLearner()
        R.config = _cfg(resume_train=True, checkpoint_dir=str(tmp_path / sub), ema_decay=0.9)
        R.graph = h = CISGraph(64, 96, 1, device='cpu', with_pwc=False, ema_decay=0.9)
        monkeypatch.setattr(h, 'flow_source', 'input')
        R._init_params()
        for a, b in ((g.gen_store, h.gen_store), (g.rec_store, h.rec_store)):
            assert torch.equal(a.flat, b.flat)
            assert torch.equal(b.shadow, a.shadow if with_avg else a.flat)


def test_use_ema_reads_the_averages_and_names_the_file_without_them(tmp_path):
    g = _averaged_graph()
    g.gen_store.shadow.mul_(0.5)
    L = AdversarialLearner()
    L.rank, L.graph = 0, g
    L.save(None, str(tmp_path / 'with'), 'best')
    plain = CISGraph(64, 96, 1, device='cpu', with_pwc=False)
    plain.load_params(_params())
    L.graph = plain
    L.save(None, str(tmp_path / 'without'), 'best')
    for suffix in ('', '.pt'):
        E = AdversarialLearner()
        E.config = _cfg(use_ema=True)
        E.graph = h = CISGraph(64, 96, 1, device='cpu', with_pwc=False, train=False)
        E.restore(str(tmp_path / 'with' / 'model.best') + suffix)
        assert torch.equal(h.gen_store.flat, g.gen_store.shadow)
        path = str(tmp_path / 'without' / 'model.best') + suffix
        with pytest.raises(KeyError, match=re.escape(path) + '.*MaskNet/conv1/kernel/ExponentialMovingAverage'):
            E.restore(path)
        E.config = _cfg(use_ema=False)
        E.restore(path)
        assert torch.equal(h.gen_store.flat, plain.gen_store.flat)


# ------------------------------------------------------------------------------------------------ launch plans
def _lines(plan):
    return [ln for ln in plan_digest.digest([(plan.name, plan)]) if not ln.startswith('storage ')]


def _cis_plans(g):
    return dict(plan_digest.graph_plans(g))


def _train_plans(g):
    return {p: getattr(g, p) for p in ('aug', 'fwd', 'bwd', 'adam', 'pack')}


SMALL = dict(pwc_hw=(128, 192))
CASES = {
    'cis': (lambda **kw: CISGraph(64, 96, 1, device='cpu', **SMALL, **kw), _cis_plans, {'R': 'adamR', 'G': 'adamG'}),
    'boxes': (lambda **kw: CISGraph(64, 96, 2, device='cpu', masks='boxes', box=(6, 32, 9, 48), **SMALL, **kw), _cis_plans,
              {'R': 'adamR'}),
    'flow': (lambda **kw: FlowTrainGraph(128, 128, 1, device='cpu', **kw), _train_plans, {'P': 'adam'}),
    'flow_unsup': (lambda **kw: FlowTrainGraph(128, 128, 1, device='cpu', loss='unsupervised', **kw), _train_plans, {'P': 'adam'}),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_plans_unchanged_with_averaging_off(case):
    make, plans, _ = CASES[case]
    with plan_digest.filled_uninitialized():
        a, b = make(), make(ema_decay=0.0)
        da, db = plan_digest.digest(list(plans(a).items())), plan_digest.digest(list(plans(b).items()))
    assert da == db
    assert not any('cis_ema_update' in ln for ln in da)


@pytest.mark.parametrize('case', sorted(CASES))
def test_averaging_adds_one_update_after_each_optimiser_launch(case):
    make, plans, adam = CASES[case]
    off, on = make(), make(ema_decay=0.999)
    po, pn = plans(off), plans(on)
    assert sorted(po) == sorted(pn)
    for name in po:
        lo, ln = _lines(po[name]), _lines(pn[name])
        if name not in adam.values():
            assert lo == ln, name
            continue
        names = [op[2] for op in pn[name].ops]
        k = next(i for i, n in enumerate(names) if n in OPTIMISERS)
        assert names == [op[2] for op in po[name].ops][:k + 1] + ['cis_ema_update'] + [op[2] for op in po[name].ops][k + 1:]
        assert ln[:k + 2] + ln[k + 3:] == lo
    for mode, name in adam.items():
        st = on.store(mode) if hasattr(on, 'rec_store') else on.store
        op = next(op for op in pn[name].ops if op[2] == 'cis_ema_update')
        assert op[1][:4] == (st.shadow.data_ptr(), st.flat.data_ptr(), st.size, 0.999)
        assert op[1][4] == on.step_state.data_ptr()
        assert torch.equal(st.shadow, st.flat)
    # only the trained stores are averaged
    if case == 'boxes':
        assert on.gen_store.shadow is None
    if case in ('cis', 'boxes'):
        assert on.pwc_store.shadow is None

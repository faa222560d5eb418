"""PWC-Net training without a GPU: the fp64 restatement of the multi-scale loss against hand-computed cases, the training graph's launch
lists (one loss forward and backward, no conv1a data gradient, one cis_adam_l2 whose segments are exactly the kernels), the unchanged
launch plans of every other graph, the usage errors of train_flow.py, and the pwcnet-<epoch> bundle's variables."""
import collections
import hashlib
import math
import os
import sys

import pytest
import torch

import flow_loss_ref as FR
from chairs_tree import make_chairs_tree
from unsupervised_detection_b200.flow_train_graph import ALPHAS, LEVELS, FlowTrainGraph, check_size

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONDENSE = {'use_dense_cx': False, 'use_res_cx': False, 'search_range': 2}
# sha256 of the file `python tests/plan_digest.py OUT` writes: every launch of the step graphs and the functional runners.  The same on
# the parent of the commit that added PWC-Net training, which changed none of them.
PLAN_DIGEST_SHA256 = '485298eebe0fad4ee7f40a1b5c26a97b5dba40d0252d9db2d4b42453b85c305d'


# ------------------------------------------------------------------------------------------------ the loss restated
def test_target_is_the_legacy_resize_over_2_pow_l_not_an_average():
    gt = torch.zeros(1, 3, 1, 2, dtype=torch.float64)
    gt[0, :, 0, 0] = torch.tensor([0.0, 1.0, 4.0])          # rows y^2
    gt[0, :, 0, 1] = torch.tensor([2.0, 2.0, 2.0])
    # 3 -> 2 rows: source rows 0 and 1.5 (lo 1, hi 2, frac 0.5) -> (0, 2.5); a 2x2 mean would give 0.5 for the first row
    g = FR.level_target(gt, 2, 1, 1)
    assert torch.equal(g[0, :, 0, 0], torch.tensor([0.0, 1.25], dtype=torch.float64))
    assert torch.equal(g[0, :, 0, 1], torch.tensor([1.0, 1.0], dtype=torch.float64))
    g = FR.level_target(gt, 2, 1, 2, s0=2.0, s1=0.5)          # vector scales per channel, / 4
    assert torch.equal(g[0, :, 0, 0], torch.tensor([0.0, 1.25], dtype=torch.float64))
    assert torch.equal(g[0, :, 0, 1], torch.tensor([0.25, 0.25], dtype=torch.float64))


def test_rho_values_and_the_zero_difference_gradient():
    d = torch.tensor([[3.0, 4.0], [0.0, 0.0], [3.0, -4.0]], dtype=torch.float64, requires_grad=True)
    r = FR.rho(d)
    assert r.tolist() == [5.0, 0.0, 5.0]
    (g,) = torch.autograd.grad(r.sum(), d)
    assert torch.isfinite(g).all() and g[1].tolist() == [0.0, 0.0]
    assert torch.allclose(g[0], torch.tensor([0.6, 0.8], dtype=torch.float64))
    rr = FR.rho(d, robust=True)
    assert abs(float(rr[0].detach()) - 7.01 ** 0.4) < 1e-15 and abs(float(rr[1].detach()) - 0.01 ** 0.4) < 1e-15
    (g,) = torch.autograd.grad(rr.sum(), d)
    k = 0.4 * 7.01 ** -0.6
    assert torch.allclose(g[2], torch.tensor([k, -k], dtype=torch.float64)) and g[1].tolist() == [0.0, 0.0]


def test_flow_loss_weights_levels_and_divides_by_the_global_batch():
    B, H, W = 2, 64, 128
    gt = torch.zeros(B, H, W, 2, dtype=torch.float64)
    flows = [torch.zeros(B, H >> l, W >> l, 2, dtype=torch.float64) for l in LEVELS]
    flows[0][0, 0, 0] = torch.tensor([3.0, 4.0])           # level 6, sample 0: one pixel off by 5
    flows[4][1, 5, 7] = torch.tensor([0.0, -2.0])          # level 2, sample 1: one pixel off by 2
    s = FR.level_sums(flows, gt)
    assert s.tolist() == [[5.0, 0, 0, 0, 0], [0, 0, 0, 0, 2.0]]
    total, terms = FR.flow_loss(flows, gt, global_batch=4)
    assert abs(float(terms[0]) - 0.32 * 5 / 4) < 1e-15 and abs(float(terms[4]) - 0.005 * 2 / 4) < 1e-15
    assert abs(float(total) - (0.32 * 5 + 0.005 * 2) / 4) < 1e-15
    p = {'pwcnet/a/kernel': torch.full((2, 2), 2.0, dtype=torch.float64), 'pwcnet/a/bias': torch.full((3,), 9.0, dtype=torch.float64)}
    assert abs(float(FR.l2_term(p, 4e-4)) - 0.5 * 4e-4 * 16.0) < 1e-18


def test_adam_l2_restatement_decays_kernels_only():
    p = {'x/kernel': torch.tensor([1.0, -2.0], dtype=torch.float64), 'x/bias': torch.tensor([1.0], dtype=torch.float64)}
    g = {'x/kernel': torch.zeros(2, dtype=torch.float64), 'x/bias': torch.zeros(1, dtype=torch.float64)}
    FR.adam_l2_step(p, g, {}, {}, 1, lr=0.1, decay=0.5)
    assert p['x/bias'].tolist() == [1.0]                     # zero gradient, no decay: unchanged
    # first step: m / sqrt(v) = sign(g') -> w - lr * sign(w) (up to eps)
    assert torch.allclose(p['x/kernel'], torch.tensor([0.9, -1.9], dtype=torch.float64), atol=1e-7)


# ------------------------------------------------------------------------------------------------ the training graph's launch lists
def _counts(plan):
    return collections.Counter(op[2] for op in plan.ops)


@pytest.mark.parametrize('options', [None, NONDENSE])
def test_training_graph_launches(options):
    g = FlowTrainGraph(128, 128, 2, options=options, device="cpu", global_batch=4)
    plans = {'fwd': g.fwd, 'bwd': g.bwd, 'adam': g.adam, 'pack': g.pack}
    total = collections.Counter()
    for p in plans.values():
        total += _counts(p)
    assert _counts(g.fwd)['cis_flow_multiscale_loss'] == 1 and _counts(g.bwd)['cis_flow_multiscale_loss_bwd'] == 1
    assert total['cis_flow_multiscale_loss'] == 1 and total['cis_flow_multiscale_loss_bwd'] == 1 and total['cis_adam_l2'] == 1
    assert [op[2] for op in g.adam.ops] == ['cis_adam_l2']
    # the loss backward comes right after zeroing the five level gradients, before the reverse tape
    names = [op[2] for op in g.bwd.ops]
    assert names[:6] == ['cis_zero'] * 5 + ['cis_flow_multiscale_loss_bwd']
    # no conv1a data gradient: the image Acts carry no dependency and no backward launch writes or reads their gradient
    for a in g.img_acts:
        assert a.grad is None and not a.grad_written and not a.dep
    # the loss reads the five refined flows and seeds the five bf16 flow gradients, weighted alpha_l / global batch
    pyr = g.pyr
    for i, l in enumerate(LEVELS):
        assert pyr.flow[i] == g.pwc.flows[l].data_ptr() and pyr.grad[i] == g.pwc.flows_bf[l].get_grad().ptr
        assert pyr.weight[i] == pytest.approx(ALPHAS[i] / 4, rel=1e-7) and pyr.accumulate[i] == 0
    # cis_adam_l2's segments: exactly the variables named */kernel, biases excluded
    args = g.adam.ops[0][1]
    assert args[5] == g._seg.data_ptr() and args[6] == len(g.kernel_seg)
    seg = g._seg.view(-1, 2).tolist()
    want = [[off, off + n] for name, _, n, off, _ in g.store.entries if name.endswith('/kernel')]
    assert seg == want and len(seg) == sum(1 for e in g.store.entries if e[0].endswith('/kernel'))
    covered = set()
    for a, b in seg:
        covered.update(range(a, b))
    for name, _, n, off, _ in g.store.entries:
        inside = sum(1 for i in range(off, off + n) if i in covered)
        assert inside == (n if name.endswith('/kernel') else 0), name
    assert g.adam.ops[0][1][7] == pytest.approx(4e-4)


def test_training_graph_input_resize_and_sizes():
    g = FlowTrainGraph(128, 192, 1, device='cpu', in_hw=(384, 640), loss='robust')
    assert _counts(g.fwd)['cis_resize_bilinear_f32'] == 3                # the two frames to 128x192, the final x4
    op = [o for o in g.fwd.ops if o[2] == 'cis_flow_multiscale_loss'][0]
    assert op[1][1:12] == (g.gt.data_ptr(), 1, 128, 192, 384, 640, 128 / 384, 192 / 640, 1, 0.01, 0.4)
    for H, W in ((96, 128), (128, 100), (0, 128), (64, 128)):
        with pytest.raises(ValueError):
            check_size(H, W)
        with pytest.raises(ValueError):
            FlowTrainGraph(H, W, 1, device='cpu')
    with pytest.raises(ValueError):
        FlowTrainGraph(128, 128, 1, device="cpu", loss="l1")


@pytest.mark.timeout(1200)
def test_other_graphs_plans_unchanged(tmp_path):
    import plan_digest
    out = tmp_path / 'digest.txt'
    plan_digest.main(str(out))
    assert hashlib.sha256(out.read_bytes()).hexdigest() == PLAN_DIGEST_SHA256


def test_learning_rate_schedule():
    from unsupervised_detection_b200.models.flow_learner import learning_rate_at
    assert [learning_rate_at(t, 1.0, [2, 4]) for t in range(1, 7)] == [1.0, 1.0, 0.5, 0.5, 0.25, 0.25]
    assert learning_rate_at(10, 1e-4, []) == 1e-4


# ------------------------------------------------------------------------------------------------ train_flow.py
def test_train_flow_usage_errors(monkeypatch, tmp_path):
    sys.path.insert(0, ROOT)
    import train_flow as TF
    from unsupervised_detection_b200.common_flags import FLAGS, FLAG_NAMES
    assert len(FLAG_NAMES) == 31 and not set(TF.TRAIN_FLOW_FLAGS) & set(FLAG_NAMES)
    split = make_chairs_tree(tmp_path / 'split', n=2, labels=[1, 2])
    nosplit = make_chairs_tree(tmp_path / 'nosplit', n=2)
    seen = []
    monkeypatch.setattr(TF, 'run', lambda cfg: seen.append((cfg.flow_loss, cfg.learning_rate, list(cfg.lr_boundaries), cfg.validate)))
    ck = '--checkpoint_dir=%s' % (tmp_path / 'ck')

    def main(*args):
        FLAGS.unparse_flags()
        TF.main(['train_flow.py'] + list(args))
    try:
        main(ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit)
        main(ck, '--dataset=FLYINGCHAIRS', '--root_dir=' + split, '--validate', '--flow_loss=robust', '--learning_rate=1e-5',
             '--lr_boundaries=100,200', '--img_height=384', '--img_width=640')
        assert seen == [('multiscale', 1e-4, [], False), ('robust', 1e-5, ['100', '200'], True)]
        bad = [['--dataset=DAVIS2016', '--root_dir=' + nosplit],                        # not Flying Chairs
               ['--dataset=SYNTHETIC'],
               ['--checkpoint_dir=', '--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit],  # no --checkpoint_dir
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--validate'],        # --validate without a split file
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--img_height=100'],  # sizes not multiples of 64
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--img_width=300'],
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--flow_loss=l1'],
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--lr_boundaries=200,100'],
               ['--dataset=FLYINGCHAIRS', '--root_dir=' + nosplit, '--learning_rate=0']]
        for b in bad:
            with pytest.raises(SystemExit):
                main(ck, *b)
    finally:
        FLAGS.unparse_flags()
    assert len(seen) == 2


# ------------------------------------------------------------------------------------------------ the saved checkpoint
@pytest.mark.parametrize('options', [None, NONDENSE, {'use_dense_cx': True, 'use_res_cx': False, 'search_range': 3}])
def test_saved_bundle_holds_exactly_the_trained_option_sets_variables(tmp_path, options):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import inspect_ckpt
    from unsupervised_detection_b200 import checkpoint as ckpt_io
    from unsupervised_detection_b200.models.flow_learner import FlowLearner
    from unsupervised_detection_b200.params_init import init_pwcnet
    L = object.__new__(FlowLearner)
    L.graph = FlowTrainGraph(128, 128, 1, options=options, device="cpu")
    p = init_pwcnet(L.graph.store.entries)
    L.graph.load_params(p)
    L.save_flow(str(tmp_path), 3)
    for suf in ('.index', '.data-00000-of-00001', '.pt'):
        assert (tmp_path / ('pwcnet-3' + suf)).is_file()
    assert ckpt_io.latest_checkpoint(str(tmp_path)).endswith('pwcnet-3')
    rows = ckpt_io.list_variables(str(tmp_path / 'pwcnet-3'))
    shapes = {n: tuple(int(d) for d in s) for n, s, _ in rows}
    assert all(n.startswith('pwcnet/') for n in shapes)                # no global_step, no other scope, no Adam slots
    opts, msg = inspect_ckpt.detect_pwc_options(shapes)
    want = dict(search_range=4, use_dense_cx=True, use_res_cx=True)
    want.update(options or {})
    assert opts == want, msg
    assert sorted(shapes) == sorted(inspect_ckpt.pwcnet_variable_names(opts))
    got, _ = FlowLearner._read_ckpt(str(tmp_path / 'pwcnet-3'), list(p))
    assert all(torch.equal(got[k], p[k]) for k in p)
    assert math.isclose(float(torch.load(str(tmp_path / 'pwcnet-3.pt'))['params']['pwcnet/featpyr/conv1a/kernel'].sum()),
                        float(p['pwcnet/featpyr/conv1a/kernel'].sum()))

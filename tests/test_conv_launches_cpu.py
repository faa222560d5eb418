"""Coverage of the per-launch conv checks (tests/conv_launch_ref.py) on the CPU: the benchmarked graphs are BUILT on CPU tensors (nothing
is launched), every cis_conv_igemm / cis_conv_wgrad op of their plans must be attributed to exactly one check, and the checked set must
contain the launch configurations the toy-shape tests never reach -- so a planner change that silently stops exercising one of them
shows up here."""
import collections

import pytest

import conv_launch_ref as R
from unsupervised_detection_b200.models import functional as FN
from unsupervised_detection_b200.step_graph import CISGraph


@pytest.fixture(scope='module')
def config2():
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        g = CISGraph(256, 448, 4, device='cpu')
    return g, rec


@pytest.fixture(scope='module')
def pwc_runner():
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        r = FN._PWCRunner(2, 384, 640, 'cpu', 'pwcnet', trainable=True)
        r.ensure_backward()
    return r, rec


def _attributed(rec, plans):
    """Every conv op of `plans` maps to one check, every op of such a check is in the same plan, in order, each op in one check only."""
    seen = collections.Counter()
    checks = []
    for plan in plans:
        pos = {id(op): i for i, op in enumerate(plan.ops)}
        for op in R.conv_ops(plan):
            ck = rec.by_op.get(id(op))
            assert ck is not None, ('unattributed', op[2], plan.name)
            seen[id(op)] += 1
            if ck.ops[0] is op:
                idx = [pos.get(id(o)) for o in ck.ops]
                assert None not in idx and idx == sorted(idx), ck
                checks.append(ck)
    assert all(v == 1 for v in seen.values())
    return checks


def _features(checks):
    f = set()
    for ck in checks:
        for d in ck.descs():
            if ck.kind == 'wgrad':
                f.add(('wgrad.tma', d.tma))
                f.add(('wgrad.nwg', d.nwg))
                f.add(('wgrad.split', d.splits > 1))
                if d.tma == 2:
                    f.add(('wgrad.nh', d.nh))
                if any(b.data_ptr() <= d.dwp < b.data_ptr() + 4 * b.numel() for b in ck.layer.dwp_hi.values()):
                    f.add('wgrad.cout_hi')
                continue
            if ck.kind == 'dgrad' and d.nsub == 4 and d.add_pre:
                f.add(('dgrad.nsub4_add_pre.BN', d.BN))
            if ck.kind == 'dgrad' and d.n_tiles >= 3:
                f.add('dgrad.n_tiles>=3')
            if d.halo and d.splits > 2:
                f.add('halo.splits>2')
            if not d.halo and d.splits > 1:
                f.add('gather.splitk')
            if d.nwg == 2:
                f.add('nwg2')
                if d.add_post:
                    f.add('add_post.nwg2')
            if d.halo and d.dil > 1:
                f.add(('dil', d.dil))
            if any(d.src[i].n_mod for i in range(d.nsrc)):
                f.add(('n_mod', d.nsrc, max(d.splits, 1)))
            if d.addf_pre:
                f.add('addf_pre' + ('.outf' if d.outf else ''))
            if d.add_post:
                f.add('add_post')
            if d.mode == 1:
                f.add('mode1')
            if d.nsub > 1 and d.outf:
                f.add('parity_group.outf')
    return f


def test_config2_every_conv_launch_is_attributed_once(config2):
    g, rec = config2
    checks = _attributed(rec, [g.fwd, g.bwd['R'], g.bwd['G']])
    kinds = collections.Counter(ck.kind for ck in checks)
    assert kinds['fwd'] > 50 and kinds['dgrad'] > 30 and kinds['wgrad'] == 17 + 32
    nops = sum(len(R.conv_ops(p)) for p in (g.fwd, g.bwd['R'], g.bwd['G']))
    assert nops == sum(len(ck.ops) for ck in checks) == 276        # the census of the benchmarked step


def test_config2_covers_the_launch_configurations_of_the_step(config2):
    g, rec = config2
    f = _features(_attributed(rec, [g.fwd, g.bwd['R'], g.bwd['G']]))
    for bn in (16, 32, 64, 128):
        assert ('dgrad.nsub4_add_pre.BN', bn) in f
    for want in ('dgrad.n_tiles>=3', 'halo.splits>2', 'nwg2', 'gather.splitk', 'addf_pre.outf', 'add_post', 'add_post.nwg2', 'mode1',
                 'parity_group.outf'):
        assert want in f, want
    for dil in (2, 4, 8):
        assert ('dil', dil) in f
    assert {('n_mod', 4, 1), ('n_mod', 4, 4), ('n_mod', 3, 6)} <= f          # (sources, split-K factor) of batch-broadcast concats
    assert {('wgrad.tma', t) for t in (0, 1, 2)} <= f
    assert {('wgrad.nh', n) for n in (16, 32, 64)} <= f
    assert {('wgrad.nwg', 1), ('wgrad.nwg', 2), ('wgrad.split', True), ('wgrad.split', False)} <= f


def test_pwc_runner_every_conv_launch_is_attributed_once(pwc_runner):
    r, rec = pwc_runner
    checks = _attributed(rec, [r.bld.fwd, r.bwd])
    f = _features(checks)
    assert 'wgrad.cout_hi' in f                                                  # Cout > 128: launches of their own (dwp_hi)
    tr = [ck for ck in checks if ck.layer.transposed]
    assert {ck.kind for ck in tr} == {'fwd', 'dgrad', 'wgrad'}
    assert sum(1 for ck in tr if ck.kind == 'wgrad') == 4 * sum(1 for ck in tr if ck.kind == 'dgrad')   # four parity weight gradients
    # the siamese feature pyramid: two calls per layer, each with its own weight-gradient launch
    calls = collections.defaultdict(set)
    for ck in checks:
        if ck.kind == 'wgrad' and 'featpyr' in ck.layer.name:
            calls[ck.layer.name].add(ck.call)
    assert len(calls) == 18 and all(v == {0, 1} for v in calls.values())

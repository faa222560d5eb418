"""Coverage of the per-launch conv checks (tests/conv_launch_ref.py) on the CPU: the benchmarked graphs are BUILT on CPU tensors (nothing
is launched), every cis_conv_igemm / cis_conv_wgrad op of their plans must be attributed to exactly one check, and the checked set must
contain the launch configurations the toy-shape tests never reach -- so a planner change that silently stops exercising one of them
shows up here."""
import collections

import pytest

import conv_launch_ref as R
from launch_suites import attributed, build, features


@pytest.fixture(scope='module')
def config2():
    g, rec, _ = build('config2', 'cpu')
    return g, rec


@pytest.fixture(scope='module')
def pwc_runner():
    r, rec, _ = build('pwc_runner', 'cpu')
    return r, rec


def test_config2_every_conv_launch_is_attributed_once(config2):
    g, rec = config2
    checks = attributed(rec, [g.fwd, g.bwd['R'], g.bwd['G']])
    kinds = collections.Counter(ck.kind for ck in checks)
    assert kinds['fwd'] > 50 and kinds['dgrad'] > 30 and kinds['wgrad'] == 17 + 32
    nops = sum(len(R.conv_ops(p)) for p in (g.fwd, g.bwd['R'], g.bwd['G']))
    assert nops == sum(len(ck.ops) for ck in checks) == 276        # the census of the benchmarked step


def test_config2_covers_the_launch_configurations_of_the_step(config2):
    g, rec = config2
    f = features(attributed(rec, [g.fwd, g.bwd['R'], g.bwd['G']]))
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
    checks = attributed(rec, [r.bld.fwd, r.bwd])
    f = features(checks)
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

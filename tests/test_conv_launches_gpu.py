"""Every convolution launch of the benchmarked train step, at its benchmarked shape and launch plan, against an fp64 reference of the
same launch (tests/conv_launch_ref.py: attribution, replay, per-element bound and its derivation).

  config 2   the train graph at 256x448, batch 4, PWC-Net at 384x640: fwd, then bwd['R'] and bwd['G'] with their weight gradients
  PWC-Net    _PWCRunner(2, 384, 640, trainable=True): Cout > 128 weight gradients, the transposed convs' parity weight gradients and
             data gradient, two calls per pyramid layer
  defaults   the reference's default geometry 192x384, batch 16: other tile counts, split factors and MT choices

Each graph is replayed once, with its glue launches checked in the same replay (launch_suites.walk_graph, shared with
tests/test_glue_launches_gpu.py), so a failing launch of either kind fails the graph's test here.  A failing launch is named with its
descriptor.  One summary line per launch kind (count, worst bound ratio, descriptor-side candidates of the persistent kernel) is printed
(pytest -s shows it)."""
import pytest

from launch_suites import assert_within_bounds, walk_graph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


@pytest.mark.parametrize('phase', ['fwd', 'bwd_R', 'bwd_G'])
def test_config2_every_conv_launch(phase):
    assert_within_bounds(walk_graph('config2'), phase)


def test_config2_checks_every_launch_kind():
    r = walk_graph('config2')
    for lab in ('fwd.halo', 'fwd.gather', 'fwd.tr_parity', 'dgrad.halo', 'dgrad.gather', 'dgrad.parity_group', 'wgrad.tma0', 'wgrad.tma1',
                'wgrad.tma2', 'bias_grad'):
        assert r['summary'][lab]['count'] > 0, lab
    assert r['conv'] == 276


def test_config2_bn_fold():
    bn_fold = walk_graph('config2')['bn_fold']
    assert bn_fold <= 1.0, bn_fold


def test_negative_controls_are_rejected():
    """The bound has teeth: for the first launch of each kind, a reference without the centre tap of the weights, and an output with one
    16 x 8 tile of one channel scaled by 1 + 2^-5, are rejected.  These act on the reference and the copied result only."""
    c = walk_graph('config2')['controls']
    for kind in ('fwd.halo', 'fwd.gather', 'dgrad.parity_group', 'wgrad.tma0', 'wgrad.tma1', 'wgrad.tma2', 'tile'):
        assert kind in c, (kind, c)
        assert c[kind] > 1.0, (kind, c)


def test_pwc_runner_every_conv_launch():
    """_PWCRunner(trainable=True) forward and backward at 384x640."""
    r = walk_graph('pwc_runner')
    s = r['summary']
    assert s['wgrad.tr']['count'] == 4 * s['dgrad.tr']['count'] > 0
    assert_within_bounds(r)


def test_defaults_192x384_batch16_every_conv_launch():
    """The reference's default geometry (common_flags.py: 192x384, batch 16) with the flow given directly: fwd, bwd['R'], bwd['G']."""
    assert_within_bounds(walk_graph('defaults'))

"""Every convolution launch of the benchmarked train step, at its benchmarked shape and launch plan, against an fp64 reference of the
same launch (tests/conv_launch_ref.py: attribution, replay, per-element bound and its derivation).

  config 2   the train graph at 256x448, batch 4, PWC-Net at 384x640: fwd, then bwd['R'] and bwd['G'] with their weight gradients
  PWC-Net    _PWCRunner(2, 384, 640, trainable=True): Cout > 128 weight gradients, the transposed convs' parity weight gradients and
             data gradient, two calls per pyramid layer
  defaults   the reference's default geometry 192x384, batch 16: other tile counts, split factors and MT choices

A failing launch is named with its descriptor.  One summary line per launch kind (count, worst bound ratio, descriptor-side candidates
of the persistent kernel) is printed (pytest -s shows it)."""
import pytest
import torch

import conv_launch_ref as R
from oracle import params as OP
from unsupervised_detection_b200.models import functional as FN
from unsupervised_detection_b200.step_graph import CISGraph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def _report(key, walker, rec, plans):
    cand = R.count_persist(rec, plans)
    for lab, v in walker.summary().items():
        print('%-22s %-20s count %4d  worst bound ratio %.3g  persistent-kernel candidates %d'
              % (key, lab, v['count'], v['worst'], cand[lab][1] if lab in cand else 0))
    if walker.controls is not None:
        print('%-22s negative controls (ratio > 1 = rejected): %s' % (key, walker.controls))


def _graph_inputs(g, B, ph, pw, seed):
    gen = torch.Generator().manual_seed(seed)
    img1 = R.smooth(B, ph, pw, 3, 0.25, gen).clamp(-0.5, 0.5)
    img2 = torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, ph, pw, 3, generator=gen)
    g.img1.copy_(img1)
    g.img2.copy_(img2)


@pytest.fixture(scope='module')
def config2():
    """Config 2 with the parameters and smooth inputs of test_parity_bench_sizes_gpu.cfg2, every conv launch checked."""
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        g = CISGraph(256, 448, 4, with_pwc=True, train=True)
    g.load_params(OP.make_params(seed=1, jitter=0.1))
    for pl in (g.pack_pwc, g.pack_gen, g.pack_rec):
        pl.run()
    _graph_inputs(g, 4, 384, 640, 7)
    w = R.Walker(rec, controls=True)
    out = {}
    for phase, plan in (('fwd', g.fwd), ('bwd_R', g.bwd['R']), ('bwd_G', g.bwd['G'])):
        n = len(w.failures)
        w.run(plan)
        out[phase] = w.failures[n:]
    out['bn_fold'] = R.check_bn_fold(g.gen.all_layers())
    _report('config2_256x448_b4', w, rec, [g.fwd, g.bwd['R'], g.bwd['G']])
    return dict(w=w, rec=rec, g=g, **out)


@pytest.mark.parametrize('phase', ['fwd', 'bwd_R', 'bwd_G'])
def test_config2_every_conv_launch(config2, phase):
    assert not config2[phase], '\n'.join(config2[phase][:20])


def test_config2_checks_every_launch_kind(config2):
    s = config2['w'].summary()
    for lab in ('fwd.halo', 'fwd.gather', 'fwd.tr_parity', 'dgrad.halo', 'dgrad.gather', 'dgrad.parity_group', 'wgrad.tma0', 'wgrad.tma1',
                'wgrad.tma2', 'bias_grad'):
        assert s[lab]['count'] > 0, lab
    assert config2['w'].checked == 276


def test_config2_bn_fold(config2):
    assert config2['bn_fold'] <= 1.0, config2['bn_fold']


def test_negative_controls_are_rejected(config2):
    """The bound has teeth: for the first launch of each kind, a reference without the centre tap of the weights, and an output with one
    16 x 8 tile of one channel scaled by 1 + 2^-5, are rejected.  These act on the reference and the copied result only."""
    c = config2['w'].controls
    for kind in ('fwd.halo', 'fwd.gather', 'dgrad.parity_group', 'wgrad.tma0', 'wgrad.tma1', 'wgrad.tma2', 'tile'):
        assert kind in c, (kind, c)
        assert c[kind] > 1.0, (kind, c)


def test_pwc_runner_every_conv_launch():
    """_PWCRunner(trainable=True) forward and backward at 384x640."""
    B, H, W = 2, 384, 640
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        r = FN._PWCRunner(B, H, W, 'cuda', 'pwcnet', trainable=True)
        r.ensure_backward()
    p = OP.make_params(seed=1, jitter=0.1)
    r.reload(p)
    gen = torch.Generator().manual_seed(13)
    img1 = R.smooth(B, H, W, 3, 0.25, gen).clamp(-0.5, 0.5)
    r.img1.copy_(img1)
    r.img2.copy_(torch.roll(img1, shifts=(2, 3), dims=(1, 2)) + 0.01 * torch.randn(B, H, W, 3, generator=gen))
    r.dflow_out.copy_(R.smooth(B, H, W, 2, 1.0, gen))
    w = R.Walker(rec)
    w.run(r.bld.fwd)
    w.run(r.bwd)
    _report('pwc_runner_384x640_b2', w, rec, [r.bld.fwd, r.bwd])
    s = w.summary()
    assert s['wgrad.tr']['count'] == 4 * s['dgrad.tr']['count'] > 0
    assert not w.failures, '\n'.join(w.failures[:20])


def test_defaults_192x384_batch16_every_conv_launch():
    """The reference's default geometry (common_flags.py: 192x384, batch 16) with the flow given directly: fwd, bwd['R'], bwd['G']."""
    B, H, W = 16, 192, 384
    mp = pytest.MonkeyPatch()
    with R.recorded(mp) as rec:
        g = CISGraph(H, W, B, with_pwc=False, train=True)
    g.load_params(OP.make_params(seed=4, jitter=0.1, nets=('MaskNet', 'FlownetS')))
    for pl in (g.pack_gen, g.pack_rec):
        pl.run()
    gen = torch.Generator().manual_seed(3)
    g.image.copy_(torch.rand(B, H, W, 3, generator=gen) - 0.5)
    g.flow.copy_(R.smooth(B, H, W, 2, 0.3, gen))
    w = R.Walker(rec)
    for plan in (g.fwd, g.bwd['R'], g.bwd['G']):
        w.run(plan)
    _report('defaults_192x384_b16', w, rec, [g.fwd, g.bwd['R'], g.bwd['G']])
    assert not w.failures, '\n'.join(w.failures[:20])
